"""CPU tests: the Gaussian beam (pic_add_gaussian_beam, Simulation.add_beam_species).  The beam oracle
(tests/beam_oracle.py) on the numpy generator: statistics, weights, cuts and bounds, images, the boosted-frame map,
focusing.  The host build of the CUDA body (tests/host_harness) against the oracle bit for bit, one box and bricks.
Config 4 with its beam through the C++ driver on the host, one rank and four z slabs, against the oracle."""
import ctypes as C
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest

import beam_oracle as bo
from test_gpu_beam import GEOM, beam_cases, brick_bounds, compare_deck, make_beam_deck, union_equals_single_box
from warpx_b200 import abi, workloads

INF = math.inf
QE, CL = workloads.Q_E, workloads.C
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def hh():
    from host_harness import harness
    return harness


def _lab(npart=1000, **kw):
    base = dict(x_m=(1.e-6, -2.e-6, 3.e-6), rms=(1.e-6, 2.e-6, 3.e-6), q_tot=-1.e-12, u_m=(0.5, -1.0, 20.0),
                u_th=(0.1, 0.2, 0.3), seed=42)
    base.update(kw)
    return abi.make_gaussian_beam(npart=npart, **base)


def _oracle(beam, charge=-QE, t0=0.0, geom=None):
    n = bo.ndraws(beam)
    g = workloads.beam_normals(beam.seed, 0, n)
    if geom is None:
        return bo.creation_list(beam, charge, g, t0)
    return bo.gaussian_beam(beam, charge, g, geom.prob_lo, geom.prob_hi, geom.periodic, t0)


def test_gaussian_beam_struct_mirrors_header():
    """abi.pic_gaussian_beam: size and every field offset == what the C compiler lays out."""
    fields = [f for f, _ in abi.pic_gaussian_beam._fields_]
    code = '#include <stdio.h>\n#include <stddef.h>\n#include "pic_b200.h"\nint main(){printf("%zu", sizeof(pic_gaussian_beam));' + \
        "".join('printf(" %%zu", offsetof(pic_gaussian_beam, %s));' % f for f in fields) + "return 0;}\n"
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "s.c"), os.path.join(d, "s")
        open(src, "w").write(code)
        subprocess.run(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe], check=True)
        got = [int(v) for v in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(abi.pic_gaussian_beam)] + [getattr(abi.pic_gaussian_beam, f).offset for f in fields]


def test_normals_reference_extends_philox_normal():
    """beam_normals uses philox_normal's construction: block 2i of draw i gives philox_normal's three numbers of
    particle 2i; the raw words are numpy's Philox stream."""
    g = workloads.beam_normals(7, 5, 100)
    p = workloads.philox_normal(7, 10, 200)
    assert np.array_equal(g[:, 0:3], p[0::2]) and np.array_equal(g[:, 4:7], p[1::2])
    bg = np.random.Philox(key=7)
    assert np.array_equal(workloads.philox_blocks(7, 0, 3).ravel(), bg.random_raw(12))


def test_lab_beam_statistics_and_weights():
    """10^6 draws, no cuts or bounds: mean and rms of x, y, z, ux, uy, uz within 5 sigma of the parameters; the
    weights sum to q_tot / charge to 1e-12."""
    b = _lab(npart=1000000)
    P = _oracle(b)
    assert len(P["x"]) == 1000000 and np.array_equal(P["id"], np.arange(1000000))
    n = 1000000
    for k, mean, rms in (("x", 1.e-6, 1.e-6), ("y", -2.e-6, 2.e-6), ("z", 3.e-6, 3.e-6), ("ux", .5 * CL, .1 * CL),
                         ("uy", -1.0 * CL, .2 * CL), ("uz", 20. * CL, .3 * CL)):
        assert abs(np.mean(P[k]) - mean) <= 5 * rms / math.sqrt(n), k
        assert abs(np.std(P[k]) - rms) <= 5 * rms / math.sqrt(2 * n), k
    assert math.fsum(P["w"]) == pytest.approx(-1.e-12 / -QE, rel=1e-12)


@pytest.mark.parametrize("npart,order", [(1000, 4), (1001, 4), (1003, 8), (1000, 8)])
def test_symmetrized_weights_and_count(npart, order):
    """npart // order draws (the reference's integer division), order images each; the weights still sum to q_tot /
    charge to 1e-12."""
    P = _oracle(_lab(npart=npart, do_symmetrize=True, symmetrization_order=order))
    assert len(P["x"]) == (npart // order) * order
    assert np.all(P["w"] == P["w"][0])
    assert math.fsum(P["w"]) == pytest.approx(-1.e-12 / -QE, rel=1e-12)


def test_cuts_and_bounds():
    """With cuts and bounds, no particle lies beyond its cut or outside bound_lo / bound_hi (half-open, like
    insideBounds); both remove some."""
    cut, blo, bhi = (1.0, 1.5, 2.0), (-INF, -5.e-6, 0.0), (1.5e-6, INF, INF)
    b = _lab(npart=100000, cut=cut, bound_lo=blo, bound_hi=bhi)
    P = _oracle(b)
    assert 1000 < len(P["x"]) < 50000
    xm, rms = (1.e-6, -2.e-6, 3.e-6), (1.e-6, 2.e-6, 3.e-6)
    for d, k in enumerate("xyz"):
        assert np.all(np.abs(P[k] - xm[d]) <= cut[d] * rms[d]), k
        assert np.all((P[k] >= blo[d]) & (P[k] < bhi[d])), k


@pytest.mark.parametrize("order", [4, 8])
def test_symmetrization_images_are_exact_mirrors(order):
    """The images of each draw, in the reference's order (x,y) (x,-y) (-x,y) (-x,-y) [(y,x) (-y,x) (y,-x) (-y,-x)],
    with u alike and z, uz shared: exact mirrors, weight / order."""
    P = _oracle(_lab(npart=400, do_symmetrize=True, symmetrization_order=order))
    x, y, ux, uy = (P[k].reshape(-1, order) for k in ("x", "y", "ux", "uy"))
    x0, y0, ux0, uy0 = x[:, 0], y[:, 0], ux[:, 0], uy[:, 0]
    want = [(x0, y0), (x0, -y0), (-x0, y0), (-x0, -y0), (y0, x0), (-y0, x0), (y0, -x0), (-y0, -x0)][:order]
    wantu = [(ux0, uy0), (ux0, -uy0), (-ux0, uy0), (-ux0, -uy0), (uy0, ux0), (-uy0, ux0), (uy0, -ux0), (-uy0, -ux0)][:order]
    for j in range(order):
        assert np.array_equal(x[:, j], want[j][0]) and np.array_equal(y[:, j], want[j][1]), j
        assert np.array_equal(ux[:, j], wantu[j][0]) and np.array_equal(uy[:, j], wantu[j][1]), j
    for k in ("z", "uz"):
        a = P[k].reshape(-1, order)
        assert np.all(a == a[:, :1]), k
    assert np.all(P["w"] == (-1.e-12 / ((400 // order) * -QE)) / order)


@pytest.mark.parametrize("t0", [0.0, 2.5e-13])
def test_boost_map_known_answer(t0):
    """MapParticletoBoostedFrame at t_lab = 0: z' = z / (gamma_b (1 - beta_b vz/c)) + t0 v'z, x' = x,
    u'z = gamma_b (uz - beta_b c gamma), gamma' = gamma_b (gamma - beta_b uz / c), to 1e-13 relative; a particle at
    rest in the lab gets u'z = -gamma_b beta_b c exactly."""
    gb = 10.0
    bb = abi.beta_of_gamma(gb)
    # u_z ~ c: no cancellation in uz - beta_b c gamma, so both sides are good to a few ulp
    kw = dict(npart=5000, x_m=(0.0, 0.0, -20.e-6), u_m=(0.5, -1.0, 0.7))
    lab = _oracle(_lab(**kw))
    P = _oracle(_lab(gamma_boost=gb, **kw), t0=t0)
    gam = np.sqrt(1 + (lab["ux"] ** 2 + lab["uy"] ** 2 + lab["uz"] ** 2) / CL ** 2)
    vz = lab["uz"] / gam
    for k in ("x", "y", "ux", "uy", "w"):
        assert np.array_equal(P[k], lab[k]), k
    uzp = gb * (lab["uz"] - bb * CL * gam)
    assert np.max(np.abs(P["uz"] - uzp) / np.abs(uzp)) <= 1e-13
    gp = np.sqrt(1 + (P["ux"] ** 2 + P["uy"] ** 2 + P["uz"] ** 2) / CL ** 2)
    assert np.max(np.abs(gp - gb * (gam - bb * lab["uz"] / CL)) / gp) <= 1e-13
    zp = lab["z"] / (gb * (1 - bb * vz / CL)) + t0 * P["uz"] / gp
    assert np.max(np.abs(P["z"] - zp) / np.abs(zp)) <= 1e-13
    rest = _oracle(_lab(npart=10, u_m=(0.0, 0.0, 0.0), u_th=(0.0, 0.0, 0.0), gamma_boost=gb))
    assert np.all(rest["uz"] == -gb * bb * CL)


def test_focusing_puts_the_drawn_size_at_the_focus():
    """Each focused particle, moved ballistically with its lab velocity to the focal plane (z = z_m + focal_distance
    along the bulk momentum, here z), lands on its drawn transverse position to round-off: x_rms is the size at the
    focus.  Needs u_th transverse > 0 (otherwise focusing moves nothing)."""
    f = 40.e-6
    drawn = _oracle(_lab(npart=5000, u_m=(0.0, 0.0, 5.0), u_th=(0.3, 0.3, 0.1)))
    P = _oracle(_lab(npart=5000, u_m=(0.0, 0.0, 5.0), u_th=(0.3, 0.3, 0.1), focal_distance=f))
    assert np.max(np.abs(P["x"] - drawn["x"])) > 1e-7                 # focusing moved them
    gam = np.sqrt(1 + (P["ux"] ** 2 + P["uy"] ** 2 + P["uz"] ** 2) / CL ** 2)
    t = (3.e-6 + f - P["z"]) / (P["uz"] / gam)
    for k, uk in (("x", "ux"), ("y", "uy")):
        at_focus = P[k] + P[uk] / gam * t
        assert np.max(np.abs(at_focus - drawn[k])) <= 1e-9 * 2.e-6, k
    assert np.array_equal(P["z"], drawn["z"])      # the bulk momentum is along z: z is not displaced


# ---------------------------------------------------------------------------------------------
def _host_beam(L, beam, geom=GEOM, own_lo=(-INF,) * 3, own_hi=(INF,) * 3, t0=0.0, capacity=None, np0=0):
    lo, hi = abi.dbl3(own_lo), abi.dbl3(own_hi)
    n = L.pic_add_gaussian_beam(C.byref(beam), -QE, C.byref(geom), lo, hi, None, 0, t0, None)
    assert n >= 0, L.pic_last_error()
    cap = np0 + n if capacity is None else capacity
    arr = {k: np.full(max(cap, 1), 7.0) for k in bo.NAMES}
    ids = np.full(max(cap, 1), 99, dtype=np.int64)
    soa = abi.pic_soa()
    for k in bo.NAMES:
        setattr(soa, k, arr[k].ctypes.data)
    soa.idcpu, soa.np = ids.ctypes.data, np0
    got = L.pic_add_gaussian_beam(C.byref(beam), -QE, C.byref(geom), lo, hi, C.byref(soa), cap, t0, None)
    out = {k: arr[k][np0:np0 + max(got, 0)] for k in bo.NAMES}
    out["id"] = ids[np0:np0 + max(got, 0)]
    return n, got, out, arr, ids


def _host_normals(L, seed, nd):
    g = np.zeros(8 * nd)
    assert L.pic_gaussian_beam_normals(seed, 0, nd, g.ctypes.data, None) == 0
    return g.reshape(nd, 8)


def test_host_generator_matches_numpy(hh):
    """Host build of the generator: Philox words bit for bit, normals to a few ulp of the numpy reference."""
    L = hh.lib()
    for first, n in ((0, 1000), ((1 << 40) - 7, 33)):
        raw = np.zeros(4 * n, dtype=np.uint64)
        assert L.pic_philox4x64(987654321, first, n, raw.ctypes.data, None) == 0
        assert np.array_equal(raw.reshape(n, 4), workloads.philox_blocks(987654321, first, n))
    ref = workloads.beam_normals(11, 0, 20000)
    assert np.max(np.abs(_host_normals(L, 11, 20000) - ref)) <= 1e-14 * np.max(np.abs(ref))


def test_host_body_matches_oracle(hh):
    """The CUDA body built for the host, every beam case of the GPU test: bit for bit the oracle fed with the same
    normals, ids included; count-only call == count; appended after p->np."""
    L = hh.lib()
    for name, beam, t0 in beam_cases():
        n, got, out, arr, ids = _host_beam(L, beam, t0=t0, np0=5)
        assert got == n > 0, name
        want = bo.gaussian_beam(beam, -QE, _host_normals(L, beam.seed, bo.ndraws(beam)), GEOM.prob_lo, GEOM.prob_hi,
                                GEOM.periodic, t0)
        for k in want:
            assert np.array_equal(out[k], want[k]), (name, k)
        assert np.all(arr["x"][:5] == 7.0) and np.all(ids[:5] == 99)


def test_domain_drop_and_periodic_wrap(hh):
    """InitData's Redistribute: beyond the non-periodic z faces particles are dropped (their ids leave gaps), along
    the periodic x, y axes they are wrapped into the domain."""
    L = hh.lib()
    geom = abi.make_geom((8, 8, 8), (-4.e-6, -4.e-6, -4.e-6), (4.e-6, 4.e-6, 4.e-6), periodic=(1, 1, 0))
    beam = _lab(npart=3000, x_m=(3.e-6, -3.e-6, 3.e-6), rms=(2.e-6, 2.e-6, 2.e-6))
    n, got, out, _, _ = _host_beam(L, beam, geom=geom)
    full = bo.creation_list(beam, -QE, _host_normals(L, beam.seed, 3000))
    assert 0 < n < 3000 and np.all(np.diff(out["id"]) > 0) and out["id"][-1] > n
    assert np.all((out["x"] >= -4.e-6) & (out["x"] <= 4.e-6) & (out["y"] >= -4.e-6) & (out["y"] <= 4.e-6))
    assert np.all((out["z"] >= -4.e-6) & (out["z"] <= 4.e-6))
    kept = np.abs(full["z"] - 0.0) <= 4.e-6
    assert np.array_equal(out["id"], full["id"][kept])
    assert np.any(out["x"] != full["x"][kept])


def test_host_preconditions_leave_particles_untouched(hh):
    """npart < 1, rms < 0, a symmetrization order other than 4 or 8, a bad boost, focusing without a bulk momentum and
    too small a capacity are refused with -1 and pic_last_error before anything is written."""
    L = hh.lib()
    bad = [dict(npart=0), dict(rms=(1.e-6, -1.e-6, 1.e-6)), dict(do_symmetrize=True, symmetrization_order=6),
           dict(npart=3, do_symmetrize=True, symmetrization_order=4), dict(u_m=(0.0, 0.0, 0.0), focal_distance=1.e-6)]
    for kw in bad:
        beam = _lab(**kw)
        arr = np.full(100, 7.0)
        soa = abi.pic_soa()
        for k in bo.NAMES:
            setattr(soa, k, arr.ctypes.data)
        soa.idcpu, soa.np = None, 0
        assert L.pic_add_gaussian_beam(C.byref(beam), -QE, C.byref(GEOM), abi.dbl3((-INF,) * 3), abi.dbl3((INF,) * 3),
                                       C.byref(soa), 100, 0.0, None) == -1, kw
        assert L.pic_last_error(), kw
        assert np.all(arr == 7.0), kw
    beam = _lab()
    beam.gamma_boost, beam.beta_boost = 10.0, 1.5
    n, got, out, arr, ids = _host_beam(L, _lab(), capacity=10)
    assert got == -1 and b"capacity" in L.pic_last_error() and np.all(arr["x"] == 7.0) and np.all(ids == 99)
    assert L.pic_add_gaussian_beam(C.byref(beam), -QE, C.byref(GEOM), abi.dbl3((-INF,) * 3), abi.dbl3((INF,) * 3),
                                   None, 0, 0.0, None) == -1
    with pytest.raises(NotImplementedError):
        abi.make_gaussian_beam((0, 0, 0), (1, 1, 1), 10, 1.0, do_backward_propagation=True)


@pytest.mark.parametrize("nb", [(1, 1, 4), (2, 2, 1)])
def test_host_bricks_union_equals_single_box(hh, nb):
    """4 z slabs and 2x2x1 bricks: the union of what each brick keeps is the single box, bit for bit, ids included."""
    L = hh.lib()
    for name, beam, t0 in beam_cases():
        union_equals_single_box(lambda lo, hi: _host_beam(L, beam, GEOM, lo, hi, t0)[2], GEOM, nb)
    assert brick_bounds(GEOM, (1, 1, 4), 0)[0] == [-INF, -INF, -INF]


# ---------------------------------------------------------------------------------------------
def _small_deck():
    wl = workloads.laser_acceleration_boosted_3d(n_cell=(12, 12, 48), density=1.e22, use_fdtd_nci_corr=True, beam=True)
    dx = [(wl["prob_hi"][d] - wl["prob_lo"][d]) / wl["n_cell"][d] for d in range(3)]
    # six cells of vacuum above the antenna, as in tests/test_host_engine.py (the coarse grid's guard-cell tie at the wall)
    wl["prob_lo"] = wl["prob_lo"][:2] + (wl["prob_lo"][2] + 6 * dx[2],)
    wl["prob_hi"] = wl["prob_hi"][:2] + (wl["prob_hi"][2] + 6 * dx[2],)
    return wl


def test_workload_default_is_unchanged_and_beam_is_the_decks():
    assert workloads.laser_acceleration_boosted_3d() == {k: v for k, v in
                                                         workloads.laser_acceleration_boosted_3d(beam=True).items()
                                                         if k != "beams"}
    assert "beams" not in workloads.laser_acceleration_boosted_3d()
    (b,) = workloads.laser_acceleration_boosted_3d(beam=True)["beams"]
    assert b["npart"] == 1000 and b["q_tot"] == -1.e-14 and b["rms"] == (1.e-6, 1.e-6, .2e-6)
    assert b["x_m"][2] == -20.e-6 and b["u_m"] == (0.0, 0.0, 2.e5) and b["u_th"] == (.2, .2, 20.)
    assert b["q"] == -QE and b["m"] == workloads.M_E


def test_boosted_deck_with_beam_on_the_host_matches_oracle(orc, hh):
    """Config 4 with electrons, ions and the witness beam in the very small: 14 steps of the C++ driver on the host
    against the oracle (the bars of test_host_engine's boosted deck: fields 1e-9 of each vector's scale, particles by
    id 1e-9); the beam keeps every particle."""
    import torch
    HS = hh.host_simulation_class()
    wl = _small_deck()
    sim, osim, obeams = make_beam_deck(HS, orc, wl, 12 * 12 * 100, torch, hh.host_library(), device="cpu")
    assert sim.species[2].np == len(obeams[0]["x"]) == 1000
    for chunk, sync in ((9, False), (5, True)):
        sim.Evolve(chunk, synchronize_last=sync)
        osim.evolve(chunk, synchronize_last=sync)
    compare_deck(sim, osim, obeams, ftol=1e-9, ptol=1e-9)
    assert sim.species[2].np == 1000


def test_boosted_deck_with_beam_on_z_slabs_matches_oracle(orc, hh):
    """The same deck on four thread ranks (z slabs, NCCL stand-in): each rank creates its slab's share of the beam; the
    union of fields and of the three species by id against the single-box oracle (test_boosted_frame_z_slabs_match_oracle's
    bars)."""
    import torch
    from test_host_multirank import _gather_fields
    HS = hh.host_simulation_class()
    world, nsteps = 4, 12
    wl = _small_deck()
    wl["n_cell"] = (12, 12, 96)
    # centre the beam on the face between slabs 1 and 2: z' ~ gamma_b (1 + beta_b) z_lab for a beam at ~c
    gb = wl["gamma_boost"]
    z_face = wl["prob_lo"][2] + 48 * (wl["prob_hi"][2] - wl["prob_lo"][2]) / 96
    wl["beams"][0]["x_m"] = (0.0, 0.0, z_face / (gb * (1 + abi.beta_of_gamma(gb))))

    def rank_fn(rank, dist):
        sim, _, _ = make_beam_deck(HS, None, wl, 12 * 12 * 200, torch, hh.host_library(), device="cpu",
                                   nb=(1, 1, world), dist=dist)
        n0 = sim.species[2].np
        sim.Evolve(nsteps)
        return dict(fields={c: sim.field_numpy(c) for c in range(9)}, box=(sim.box_lo, sim.box_hi), n0=n0,
                    parts=[sim.species_numpy(i, sort_by_id=False) for i in (0, 1, 2)], dz=sim.dx[2])

    res = hh.run_ranks(world, rank_fn)
    assert sum(res[r]["n0"] > 0 for r in range(world)) >= 2, "the beam must straddle slabs"
    L = hh.host_library()
    osim = __import__("test_oracle").make_lwfa_oracle(orc, wl)
    beam = abi.make_gaussian_beam(**{k: v for k, v in wl["beams"][0].items() if k not in ("name", "q", "m")},
                                  gamma_boost=wl["gamma_boost"])
    P = bo.add_beam(osim, -QE, workloads.M_E, beam, _host_normals(L, beam.seed, bo.ndraws(beam)))
    osim.evolve(nsteps)
    err, scale = _gather_fields(res, osim, world)
    for group in ((0, 1, 2), (3, 4, 5), (6, 7, 8)):
        s = max(scale[c] for c in group)
        for c in group:
            assert err[c] <= 1e-9 * s, abi.COMP_NAMES[c]
    for isp in (0, 1, 2):
        B = osim.particles(isp)
        ids = np.concatenate([res[r]["parts"][isp]["id"] for r in range(world)])
        order = np.argsort(ids)
        want = np.arange(len(B["x"])) if isp < 2 else P["id"]
        assert len(B["x"]) > 0 and np.array_equal(ids[order], want), isp
        for k in ("x", "y", "z"):
            a = np.concatenate([res[r]["parts"][isp][k] for r in range(world)])[order]
            assert np.max(np.abs(a - B[k])) / res[0]["dz"] <= 1e-9, (isp, k)
        for k in ("ux", "uy", "uz"):
            a = np.concatenate([res[r]["parts"][isp][k] for r in range(world)])[order]
            scale = max(10.0, float(np.max(np.abs(B[k]))) / CL) * CL
            assert np.max(np.abs(a - B[k])) / scale <= 1e-9, (isp, k)
