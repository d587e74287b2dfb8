"""CPU tests of the pairwise Coulomb collisions: the product's kernel source (csrc/collision.cu, through the SIMT host
build of tests/host_harness) against the numpy restatement of tests/collision_oracle.py, the exact invariants of one
collision stage, the C++ driver's collision loop and its refusals."""
import numpy as np
import pytest

import collision_cases as cc
import collision_oracle as co
from warpx_b200 import abi, workloads

ME = workloads.M_E


@pytest.fixture(scope="module")
def host():
    import torch
    from host_harness import harness
    return harness.host_library(), torch


def counts(seed, mean=4.0, big=300):
    rng = np.random.default_rng(seed)
    n = rng.poisson(mean, size=(4, 5, 6))
    n[0, 0, 0:4] = (0, 1, 2, 3)
    n[1, 1, 1] = big                      # a cell for the block-per-cell path
    return n


def oracle_by_id(sp1, sp2, coll, dt, step):
    r1, r2 = co.collide({k: v.copy() for k, v in sp1.items()}, None if sp2 is None else {k: v.copy() for k, v in sp2.items()},
                        coll, cc.GEOM, dt, step)
    out = []
    for sp, r in ((sp1, r1), (sp2, r2)):
        if sp is None:
            continue
        o = dict(sp)
        o["ux"], o["uy"], o["uz"] = r
        out.append(cc.by_id(o))
    return out


def assert_close_u(got, want, rtol):
    scale = np.sqrt(want["ux"] ** 2 + want["uy"] ** 2 + want["uz"] ** 2).max()
    for k in ("ux", "uy", "uz"):
        err = np.abs(got[k] - want[k]).max() / scale
        assert err <= rtol, (k, err)


# dt spans the s12 branches: small angles with the redraw loop, the fitted A(s12), the exp form and isotropic
@pytest.mark.parametrize("dt", [1e-17, 3e-15, 3e-14, 1e-11])
@pytest.mark.parametrize("kind", ["ee_fixed", "ee_computed", "ei_unequal"])
@pytest.mark.parametrize("pending", [True, False])
def test_host_stage_matches_oracle(host, dt, kind, pending):
    L, t = host
    if kind == "ei_unequal":
        sp1 = cc.particle_set(1, cc.GEOM, counts(1), (0.01, 0.02, 0.01), weights="log")
        sp2 = cc.particle_set(2, cc.GEOM, counts(2, 2.0, 150), (0.004, 0.004, 0.004), u_m=(0.01, 0, 0), weights="log",
                              id_offset=10 ** 6)
        coll = cc.ei_spec(L=-1.0)
    else:
        sp1 = cc.particle_set(3, cc.GEOM, counts(3), (0.01, 0.02, 0.01))
        sp2 = None
        coll = cc.ee_spec(L=15.9 if kind == "ee_fixed" else -1.0)
    g1, g2, status = cc.run_stage(L, t, "cpu", sp1, sp2, coll, cc.GEOM, dt, 5, pending=pending)
    assert status == 0
    want = oracle_by_id(sp1, sp2, coll, dt, 5)
    for got, w, ini in zip((g1, g2), want, (sp1, sp2)):
        got = cc.by_id(got)
        assert np.array_equal(got["id"], w["id"])
        assert_close_u(got, w, 1e-13)        # numpy's and glibc's transcendentals differ by ulps
        changed = np.mean(got["ux"] != cc.by_id(ini)["ux"])
        assert changed > 0.3, changed
        for k in ("x", "y", "z", "w"):                 # only u changes
            assert np.array_equal(got[k], cc.by_id(ini)[k])


def test_host_stage_conserves_momentum_and_energy_and_keeps_lone_particles(host):
    L, t = host
    n = counts(4)
    sp = cc.particle_set(4, cc.GEOM, n, (0.05, 0.02, 0.03))
    got, _, _ = cc.run_stage(L, t, "cpu", sp, None, cc.ee_spec(L=-1.0), cc.GEOM, 3e-14, 0)
    before, after = cc.by_id(sp), cc.by_id(got)
    for k in ("ux", "uy", "uz"):
        p0, p1 = (ME * before["w"] * before[k]).sum(), (ME * after["w"] * after[k]).sum()
        scale = (ME * before["w"] * np.abs(before[k])).sum()
        assert abs(p1 - p0) <= 1e-13 * scale, k

    def energy(s):
        u2 = (s["ux"] ** 2 + s["uy"] ** 2 + s["uz"] ** 2) / workloads.C ** 2
        return (s["w"] * ME * workloads.C ** 2 * (u2 / (np.sqrt(1.0 + u2) + 1.0))).sum()
    assert abs(energy(after) - energy(before)) <= 1e-13 * energy(before)
    # the lone particle of cell (1, 0, 0) keeps its bits
    cell = co.cells_of(before, cc.GEOM)
    lone = cell == 1
    assert lone.sum() == 1
    for k in ("ux", "uy", "uz"):
        assert np.array_equal(after[k][lone], before[k][lone])


def test_host_stage_does_not_depend_on_storage_order(host):
    L, t = host
    sp1 = cc.particle_set(5, cc.GEOM, counts(5), (0.01, 0.02, 0.01), weights="log")
    sp2 = cc.particle_set(6, cc.GEOM, counts(6, 3.0, 90), (0.004, 0.004, 0.004), id_offset=10 ** 6)
    perm1 = np.random.default_rng(9).permutation(len(sp1["x"]))
    perm2 = np.random.default_rng(10).permutation(len(sp2["x"]))
    a1, a2, _ = cc.run_stage(L, t, "cpu", sp1, sp2, cc.ei_spec(), cc.GEOM, 3e-15, 2)
    b1, b2, _ = cc.run_stage(L, t, "cpu", {k: v[perm1] for k, v in sp1.items()}, {k: v[perm2] for k, v in sp2.items()},
                             cc.ei_spec(), cc.GEOM, 3e-15, 2, pending=False)
    for a, b in ((a1, b1), (a2, b2)):
        a, b = cc.by_id(a), cc.by_id(b)
        for k in a:
            assert np.array_equal(a[k], b[k]), k


def _host_sim(Sim, wl, solver, nox=1):
    return Sim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=nox, solver=solver, dt=wl["dt"], sort_interval=4)


def test_host_driver_loop_with_solver_none_matches_oracle(host):
    """A reduced xyz deck (2^3 cells of the deck's size, 40 particles per cell and species, collisions every 3 steps)
    through the C++ driver of the host build against the oracle's deck loop, over two Evolve calls."""
    from host_harness import harness
    wl = workloads.collision_xyz_3d(n=2, ppc=40)
    colls = [dict(c, ndt=3) for c in wl["collisions"]]
    Sim = harness.host_simulation_class()
    sim = _host_sim(Sim, wl, abi.SOLVER_NONE)
    for s in wl["species"]:
        sim.add_species(s["name"], s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    for c in colls:
        sim.add_collision(c["species"][0], c["species"][1], coulomb_log=c["coulomb_log"], ndt=c["ndt"], seed=c["seed"])
    sim.Evolve(4)
    sim.Evolve(3)
    geom = dict(n_cell=wl["n_cell"], prob_lo=wl["prob_lo"], prob_hi=wl["prob_hi"], box_lo=(0, 0, 0),
                box_hi=tuple(v - 1 for v in wl["n_cell"]))
    species = [dict(s, id=np.arange(len(s["x"]), dtype=np.int64)) for s in wl["species"]]
    co.deck_loop(species, colls, geom, wl["dt"], 7)
    for isp in range(2):
        got = sim.species_numpy(isp, sort_by_id=True)
        want = cc.by_id(species[isp])
        for k in ("ux", "uy", "uz"):
            err = np.abs(got[k] - want[k]).max() / workloads.C
            assert err <= 1e-12, (isp, k, err)
        assert np.array_equal(got["w"], want["w"])


def test_host_collision_refusals_leave_the_engine_untouched(host):
    from host_harness import harness
    Sim = harness.host_simulation_class()
    wl = workloads.collision_xyz_3d(n=2, ppc=4)
    with pytest.raises(ValueError, match="explicit dt"):
        Sim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=1, solver=abi.SOLVER_NONE)
    with pytest.raises(RuntimeError, match="filter"):
        Sim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=1, solver=abi.SOLVER_NONE, dt=wl["dt"], use_filter=True)
    sim = _host_sim(Sim, wl, abi.SOLVER_NONE)
    with pytest.raises(RuntimeError, match="none"):
        sim.add_laser(abi.make_laser((0, 0, 0), (0, 0, 1), (1, 0, 0), 8e-7, 1e12, 5e-6, 1e-14, 2e-14, 1e-4))
    s = wl["species"][0]
    sim.add_species(s["name"], s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    nobins = Sim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=1, solver=abi.SOLVER_NONE, dt=wl["dt"], use_bins=False)
    nobins.add_species(s["name"], s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    with pytest.raises(RuntimeError, match="no species"):
        sim.add_collision(0, 1)
    with pytest.raises(RuntimeError, match="no species"):
        sim.add_collision(-1, 0)
    with pytest.raises(RuntimeError, match="ndt"):
        sim.add_collision(0, 0, ndt=0)
    with pytest.raises(RuntimeError, match="no cell bins"):
        nobins.add_collision(0, 0)
    assert sim.collisions == [] and nobins.collisions == []
    before = sim.species_numpy(0, sort_by_id=True)
    sim.Evolve(2)                                   # nothing registered: no collision ran
    after = sim.species_numpy(0, sort_by_id=True)
    for k in ("ux", "uy", "uz"):
        assert np.array_equal(before[k], after[k])
    sim.add_collision(0, 0, coulomb_log=15.9)
    assert len(sim.collisions) == 1


def test_host_stage_refuses_particles_behind_the_bins(host):
    """particles appended after the last sort (np_binned < np) must be sorted before they collide"""
    L, t = host
    import ctypes as C
    sp = cc.particle_set(8, cc.GEOM, 3.0, (0.01, 0.01, 0.01))
    d = cc.DeviceSpecies(L, t, "cpu", sp, cc.GEOM)
    d.sort(True)
    d.bins.np_binned = d.n - 1
    status = t.zeros(1, dtype=t.int32)
    rc = L.pic_collide_pairwise_coulomb(C.byref(cc.collision_spec(cc.ee_spec())), C.byref(d.soa(0)), C.byref(d.bins), d.src,
                                        None, None, None, C.byref(d.g), 1e-15, 0, None, None, status.data_ptr(), None)
    assert rc != 0 and b"current bins" in L.pic_last_error()
    assert np.array_equal(d.numpy()["ux"], sp["ux"])
