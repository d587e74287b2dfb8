"""GPU tests (-m gpu): Gaussian beams created on the device (pic_add_gaussian_beam, Simulation.add_beam_species) against
the numpy reference of the generator (warpx_b200.workloads.beam_normals) and the beam oracle (tests/beam_oracle.py):
the generator's words bit for bit, the particles of one box and of bricks, config 4's boosted deck with its witness
beam through the C++ driver, and Gauss's law with a relativistic beam in a periodic plasma.
tests/host_harness/run_beam_tests_on_host.py runs these functions against the host build of the library."""
import ctypes as C
import math

import numpy as np
import pytest

import beam_oracle as bo
from helpers import gauss_drift, rel_linf, simulation_gauss
from warpx_b200 import abi, workloads

pytestmark = pytest.mark.gpu
INF = math.inf
GEOM = abi.make_geom((16, 16, 128), (-128.e-6, -128.e-6, -800.e-6), (128.e-6, 128.e-6, 0.0), periodic=(1, 1, 0))


def beam_cases():
    """(name, beam, t0): lab frame and boosted frame, images, cuts and bounds, focusing."""
    d = dict(x_m=(0.0, 0.0, -20.e-6), rms=(1.e-6, 1.e-6, .2e-6), q_tot=-1.e-14, u_m=(0.0, 0.0, 2.e5), u_th=(.2, .2, 20.))
    lab = dict(d, x_m=(0.0, 0.0, -400.e-6), rms=(20.e-6, 30.e-6, 50.e-6), u_m=(1.0, -2.0, 10.0), u_th=(.5, .5, 2.))
    return [
        ("lab", abi.make_gaussian_beam(npart=20000, seed=1, **lab), 0.0),
        ("lab_cut_bounds_sym4", abi.make_gaussian_beam(npart=20003, seed=2, cut=(1.5, 2.0, 2.5), bound_lo=(-INF, -40.e-6, -INF),
                                                       bound_hi=(30.e-6, INF, -380.e-6), do_symmetrize=True, **lab), 0.0),
        ("lab_focus_sym8", abi.make_gaussian_beam(npart=16000, seed=3, focal_distance=50.e-6, do_symmetrize=True,
                                                  symmetrization_order=8, **lab), 0.0),
        ("boosted", abi.make_gaussian_beam(npart=20000, seed=4, gamma_boost=10.0, **d), 0.0),
        ("boosted_t0_sym8_focus", abi.make_gaussian_beam(npart=8000, seed=5, gamma_boost=10.0, do_symmetrize=True,
                                                         symmetrization_order=8, focal_distance=1.e-3, **d), 3.7e-14),
    ]


def _device_soa(t, n):
    buf = t.zeros((7, max(n, 1)), dtype=t.float64, device="cuda")
    ids = t.zeros(max(n, 1), dtype=t.int64, device="cuda")
    soa = abi.pic_soa()
    for k, name in enumerate(bo.NAMES):
        setattr(soa, name, buf[k].data_ptr())
    soa.idcpu, soa.np = ids.data_ptr(), 0
    return soa, buf, ids


def device_beam(t, L, beam, charge, geom, own_lo=(-INF,) * 3, own_hi=(INF,) * 3, t0=0.0):
    """pic_add_gaussian_beam into fresh device arrays -> numpy dict (creation order) with ids."""
    stream = t.cuda.current_stream().cuda_stream
    lo, hi = abi.dbl3(own_lo), abi.dbl3(own_hi)
    n = L.pic_add_gaussian_beam(C.byref(beam), charge, C.byref(geom), lo, hi, None, 0, t0, stream)
    assert n >= 0, L.pic_last_error()
    soa, buf, ids = _device_soa(t, n)
    got = L.pic_add_gaussian_beam(C.byref(beam), charge, C.byref(geom), lo, hi, C.byref(soa), n, t0, stream)
    assert got == n, L.pic_last_error()
    t.cuda.synchronize()
    out = {k: buf[i, :n].cpu().numpy().copy() for i, k in enumerate(bo.NAMES)}
    out["id"] = ids[:n].cpu().numpy().copy()
    return out


def device_normals(t, L, seed, ndraw):
    g = t.zeros(8 * ndraw, dtype=t.float64, device="cuda")
    assert L.pic_gaussian_beam_normals(seed, 0, ndraw, g.data_ptr(), t.cuda.current_stream().cuda_stream) == 0
    t.cuda.synchronize()
    return g.cpu().numpy().reshape(ndraw, 8)


def test_device_generator_and_beam_match_reference(cuda):
    """The device's Philox4x64-10 words equal numpy's bit for bit (blocks near 0 and near 2^40); its normals equal the
    numpy reference's to a few ulp (log / sincos of CUDA vs the host's); every beam case equals the oracle fed with the
    numpy normals to 1e-14 of the spread of each coordinate, and the oracle fed with the device's own normals bit for
    bit, ids included."""
    from warpx_b200.lib import lib
    t, L = cuda, lib()
    stream = t.cuda.current_stream().cuda_stream
    for first, n in ((0, 4096), ((1 << 40) - 7, 333)):
        raw = t.zeros(4 * n, dtype=t.int64, device="cuda")
        assert L.pic_philox4x64(987654321, first, n, raw.data_ptr(), stream) == 0
        t.cuda.synchronize()
        assert np.array_equal(raw.cpu().numpy().view(np.uint64).reshape(n, 4), workloads.philox_blocks(987654321, first, n))
    g = device_normals(t, L, 11, 50000)
    ref = workloads.beam_normals(11, 0, 50000)
    assert np.max(np.abs(g - ref)) <= 1e-14 * np.max(np.abs(ref))
    for name, beam, t0 in beam_cases():
        nd = bo.ndraws(beam)
        got = device_beam(t, L, beam, -workloads.Q_E, GEOM, t0=t0)
        exact = bo.gaussian_beam(beam, -workloads.Q_E, device_normals(t, L, beam.seed, nd), GEOM.prob_lo, GEOM.prob_hi,
                                 GEOM.periodic, t0)
        for k in exact:
            assert np.array_equal(got[k], exact[k]), (name, k)
        want = bo.gaussian_beam(beam, -workloads.Q_E, workloads.beam_normals(beam.seed, 0, nd), GEOM.prob_lo,
                                GEOM.prob_hi, GEOM.periodic, t0)
        assert len(got["x"]) > 0 and np.array_equal(got["id"], want["id"]), name
        assert np.array_equal(got["w"], want["w"]), name
        for k in ("x", "y", "z", "ux", "uy", "uz"):     # 1e-14 of the spread, plus a few ulp where |mean| >> spread
            bar = 1e-14 * np.std(want[k]) + 4 * np.spacing(np.abs(want[k]))
            assert np.all(np.abs(got[k] - want[k]) <= bar), (name, k)


def brick_bounds(geom, nb, r):
    """[own_lo, own_hi) of brick r of an nb grid (+-inf at the domain's faces), as Simulation.add_beam_species forms it."""
    from warpx_b200 import parallel
    n = tuple(geom.n_cell)
    dec = parallel.Decomposition(n, nb, r)
    dx = [(geom.prob_hi[d] - geom.prob_lo[d]) / n[d] for d in range(3)]
    lo = [geom.prob_lo[d] + dx[d] * dec.box_lo[d] if dec.box_lo[d] > 0 else -INF for d in range(3)]
    hi = [geom.prob_lo[d] + dx[d] * (dec.box_hi[d] + 1) if dec.box_hi[d] < n[d] - 1 else INF for d in range(3)]
    return lo, hi


def union_equals_single_box(make, geom, nb):
    """Every particle of `make(own_lo, own_hi)` over the bricks of nb, sorted by id, == the single box, bit for bit."""
    one = make((-INF,) * 3, (INF,) * 3)
    parts = [make(*brick_bounds(geom, nb, r)) for r in range(nb[0] * nb[1] * nb[2])]
    assert sum(len(p["x"]) > 0 for p in parts) >= 2, "the beam must straddle bricks"
    cat = {k: np.concatenate([p[k] for p in parts]) for k in one}
    order = np.argsort(cat["id"], kind="stable")
    for k in one:
        assert np.array_equal(cat[k][order], one[k]), k


@pytest.mark.parametrize("nb", [(1, 1, 4), (2, 2, 1)])
def test_device_beam_on_bricks_equals_single_box(cuda, nb):
    """4 z slabs and 2x2x1 bricks: each brick keeps [own_lo, own_hi); the union is the single box, ids included."""
    from warpx_b200.lib import lib
    L = lib()
    for name, beam, t0 in beam_cases():        # every beam is centred on a brick face (x = y = 0, z = -400 um)
        union_equals_single_box(lambda lo, hi: device_beam(cuda, L, beam, -workloads.Q_E, GEOM, lo, hi, t0), GEOM, nb)


# ---------------------------------------------------------------------------------------------
def make_beam_deck(Simulation, orc, wl, capacity, t, L, device="cuda", nb=None, dist=None):
    """Config 4 with its beam: the Simulation (C++ driver) and, when orc is given, the single-box oracle with the beam
    the oracle restates from the normals the library L reports (the same draws, so the two start bit-identical).
    t / device: where L's memory lives."""
    from test_oracle import make_lwfa_oracle, _nci_lines
    from warpx_b200.engine import max_dt, nci_godfrey_stencils
    dx = [(wl["prob_hi"][d] - wl["prob_lo"][d]) / wl["n_cell"][d] for d in range(3)]
    nci = nci_godfrey_stencils(L, _nci_lines(), workloads.C * wl["cfl"] * max_dt(wl["solver"], dx) / dx[2])
    sim = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=wl["nox"], cfl=wl["cfl"], dist=dist, nb=nb,
                     solver=wl["solver"], pusher=wl["pusher"], use_filter=wl["use_filter"], sort_interval=4,
                     boundaries=abi.make_boundaries(wl["field_lo"], wl["field_hi"]),
                     moving_window=(wl["moving_window_dir"], wl["moving_window_v"]),
                     gamma_boost=wl["gamma_boost"], nci_stencils=nci)
    for s in wl["species"]:
        sim.add_plasma_species(s["name"], s["q"], s["m"],
                               abi.make_injector(s["ppc"], s["bound_lo"], s["bound_hi"], s["density"],
                                                 s["do_continuous_injection"]), capacity)
    beams = []
    for b in wl["beams"]:
        beam = abi.make_gaussian_beam(**{k: v for k, v in b.items() if k not in ("name", "q", "m")})
        sim.add_beam_species(b["name"], b["q"], b["m"], beam, capacity=2 * b["npart"])   # sets the boost
        beams.append((b, beam))
    for la in wl["lasers"]:
        sim.add_laser(abi.make_laser(la["position"], la["direction"], la["polarization"], la["wavelength"],
                                     la["e_max"], la["waist"], la["duration"], la["t_peak"], la["focal_distance"]))
    osim, obeams = None, []
    if orc is not None:
        osim = make_lwfa_oracle(orc, wl)
        for b, beam in beams:
            nd = bo.ndraws(beam)
            g = t.zeros(8 * nd, dtype=t.float64, device=device)
            assert L.pic_gaussian_beam_normals(beam.seed, 0, nd, g.data_ptr(), None) == 0
            if device == "cuda":
                t.cuda.synchronize()
            obeams.append(bo.add_beam(osim, b["q"], b["m"], beam, g.cpu().numpy().reshape(nd, 8)))
    return sim, osim, obeams


def compare_deck(sim, osim, obeams, ftol, ptol, nplasma=2):
    """Fields against the scale of each vector; every particle of every species by id; the antenna.  Returns the
    deviation of each field component and particle coordinate on its scale."""
    dev = {}
    for group in ((0, 1, 2), (3, 4, 5), (6, 7, 8)):
        want = [osim.fab(c)[1] for c in group]
        scale = max(float(np.max(np.abs(w))) for w in want)
        assert scale > 0
        for c, w in zip(group, want):
            d, a = sim.field_numpy(c)
            e = float(np.max(np.abs(a[d.valid_slices()] - w[d.valid_slices()])))
            assert e <= ftol * scale, abi.COMP_NAMES[c]
            dev[abi.COMP_NAMES[c]] = e / scale
    for isp in range(nplasma + len(obeams)):
        A = sim.species_numpy(isp, sort_by_id=True)
        B = osim.particles(isp)
        ids = np.arange(len(B["x"])) if isp < nplasma else obeams[isp - nplasma]["id"]
        assert len(B["x"]) > 0 and np.array_equal(A["id"], ids), isp
        assert np.array_equal(A["w"], B["w"]), isp
        for k in ("x", "y", "z"):
            dev[(isp, k)] = float(np.max(np.abs(A[k] - B[k]))) / sim.dx[2]
            assert dev[(isp, k)] <= ptol, (isp, k)
        for k in ("ux", "uy", "uz"):
            scale = max(10.0, float(np.max(np.abs(B[k]))) / workloads.C) * workloads.C
            dev[(isp, k)] = float(np.max(np.abs(A[k] - B[k]))) / scale
            assert dev[(isp, k)] <= ptol, (isp, k)
    LA, LB = sim.laser_numpy(0), osim.laser_particles(0)
    assert len(LA["x"]) == len(LB["x"]) > 0
    for k in ("x", "y", "z"):
        assert np.max(np.abs(LA[k] - LB[k])) / sim.dx[2] <= ptol, k
    return dev


def test_boosted_deck_with_beam_matches_oracle(orc, cuda):
    """BASELINE.json config 4 with its three species (workloads.laser_acceleration_boosted_3d(beam=True)): 40 steps
    through the C++ driver against the oracle in two chunks -- fields to 1e-8 of each vector's scale, every particle of
    the electrons, ions and beam by id to 1e-9, the antenna.  The beam keeps all its particles, and at gamma' ~ 1e4 its
    centroid moves by its mean boosted-frame velocity times the elapsed time, to 1e-6."""
    from warpx_b200.engine import Simulation
    from warpx_b200.lib import lib
    wl = workloads.laser_acceleration_boosted_3d(use_fdtd_nci_corr=True, beam=True)
    sim, osim, obeams = make_beam_deck(Simulation, orc, wl, 16 * 16 * 400, cuda, lib())
    beam0 = sim.species_numpy(2, sort_by_id=True)
    assert len(beam0["x"]) == len(obeams[0]["x"]) == wl["beams"][0]["npart"]
    for chunk, sync in ((23, False), (17, True)):
        sim.Evolve(chunk, synchronize_last=sync)
        osim.evolve(chunk, synchronize_last=sync)
    cuda.cuda.synchronize()
    assert sim.time == pytest.approx(osim.time(), rel=1e-15)
    dev = compare_deck(sim, osim, obeams, ftol=1e-8, ptol=1e-9)
    print("deviations from the oracle:", dev)
    beam = sim.species_numpy(2, sort_by_id=True)
    assert len(beam["x"]) == len(beam0["x"])
    gam = np.sqrt(1.0 + (beam0["ux"] ** 2 + beam0["uy"] ** 2 + beam0["uz"] ** 2) / workloads.C ** 2)
    expect = float(np.mean(beam0["uz"] / gam)) * sim.time
    moved = float(np.mean(beam["z"]) - np.mean(beam0["z"]))
    assert abs(moved - expect) <= 1e-6 * abs(expect), (moved, expect)


def test_periodic_plasma_with_beam_keeps_gauss_law(cuda):
    """A relativistic beam (u_m = (0, 0, 10), lab frame) in the periodic uniform plasma, 20 steps: Gauss's law over all
    species (rho from Simulation.rho_numpy) stays within test_gpu_gauss.py's 1e-11, so the beam deposits and crosses
    the periodic faces consistently; no beam particle is lost."""
    from warpx_b200.engine import Simulation
    wl = workloads.uniform_plasma_3d(n=32, ppc=(1, 1, 1), u_th=0.05, lx=5.0e-6)
    sim = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=3, sort_interval=4)
    s = wl["species"][0]
    sim.add_species(s["name"], s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    beam = abi.make_gaussian_beam(x_m=(0.0, 0.0, 1.e-6), rms=(.3e-6, .3e-6, .5e-6), npart=4000, q_tot=-2.e-15,
                                  u_m=(0.0, 0.0, 10.0), u_th=(.1, .1, .5), seed=17)
    sp = sim.add_beam_species("beam", -workloads.Q_E, workloads.M_E, beam, capacity=8000)
    assert sp.np == 4000
    G0, rho0 = simulation_gauss(sim)
    done = 0
    for step in (1, 4, 5, 12, 20):
        sim.Evolve(step - done, synchronize_last=False)
        done = step
        G, _ = simulation_gauss(sim)
        assert gauss_drift(G, G0, rho0) <= 1e-11, step
        assert sim.species[1].np == 4000
    B = sim.species_numpy(1, sort_by_id=True)
    assert np.array_equal(B["id"], np.arange(4000))
    assert rel_linf(np.array([np.mean(B["uz"])]), np.array([10.0 * workloads.C])) < 0.1
