"""GPU tests (-m gpu) of the pairwise Coulomb collisions (csrc/collision.cu, the C++ driver's collision stage and
algo.maxwell_solver = none):

  * the device stage against the numpy restatement (tests/collision_oracle.py) on seeded multi-cell sets -- Poisson
    counts, cells of 0, 1, 2, 3 and 1000 particles, cells without species 2, log-uniform weights, every s12 branch,
    through a pending permutation and on moved particles -- to 1e-13 of the largest |u|;
  * the device stage against what the reference's own headers compute (tests/golden/collision_reference.npz) to 1e-13
    of each cell's |u| scale, and cells of more than 2048 particles (the kernel's global-memory path) against the
    restatement;
  * two storage orders of the same particles give the same result per id, bit for bit;
  * the reference's acceptance tests on both collision decks at full size (analysis_collision_3d.py and
    analysis_collision_3d_isotropization.py), and the device loop against the oracle's loop on the xyz deck;
  * a restart from a checkpoint continues an xyz run bit for bit;
  * Gauss's law, the particle count and the weights by id at 128^3 x 8 ppc with Yee and electron-electron collisions
    every step (the extra sorts must neither drop nor duplicate a particle)."""
import numpy as np
import pytest

import collision_cases as cc
import collision_oracle as co
from warpx_b200 import abi, workloads

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(cuda):
    from warpx_b200.lib import lib
    return lib(), cuda, cuda.device("cuda", 0)


def counts(seed, mean, big):
    rng = np.random.default_rng(seed)
    n = rng.poisson(mean, size=(4, 5, 6))
    n[0, 0, 0:4] = (0, 1, 2, 3)
    n[1, 1, 1] = big
    return n


def cases(kind):
    if kind == "ei":
        sp1 = cc.particle_set(11, cc.GEOM, counts(11, 6.0, 1000), (0.01, 0.02, 0.01), weights="log")
        n2 = counts(12, 2.0, 300)
        n2[2, 2, 2] = 0                               # a cell without species 2
        sp2 = cc.particle_set(12, cc.GEOM, n2, (0.004, 0.004, 0.004), u_m=(0.01, 0, 0), weights="log", id_offset=10 ** 7)
        return sp1, sp2, cc.ei_spec(L=-1.0)
    sp1 = cc.particle_set(13, cc.GEOM, counts(13, 8.0, 1000), (0.01, 0.02, 0.01), weights="log" if kind == "ee_log" else "equal")
    return sp1, None, cc.ee_spec(L=15.9 if kind == "ee_fixed" else -1.0)


def run(dev, sp1, sp2, coll, dt, step, pending=True):
    L, t, d = dev
    return cc.run_stage(L, t, d, sp1, sp2, coll, cc.GEOM, dt, step, pending=pending, stream=t.cuda.current_stream().cuda_stream,
                        sync=t.cuda.synchronize)


@pytest.mark.parametrize("dt", [1e-17, 3e-15, 3e-14, 1e-11])
@pytest.mark.parametrize("kind", ["ee_fixed", "ee_log", "ei"])
@pytest.mark.parametrize("pending", [True, False])
def test_device_stage_matches_oracle(dev, dt, kind, pending):
    sp1, sp2, coll = cases(kind)
    g1, g2, status = run(dev, sp1, sp2, coll, dt, 3, pending)
    assert status == 0
    r1, r2 = co.collide({k: v.copy() for k, v in sp1.items()}, None if sp2 is None else {k: v.copy() for k, v in sp2.items()},
                        coll, cc.GEOM, dt, 3)
    for got, ini, r in ((g1, sp1, r1), (g2, sp2, r2)):
        if ini is None:
            continue
        want = dict(ini)
        want["ux"], want["uy"], want["uz"] = r
        got, want, ini = cc.by_id(got), cc.by_id(want), cc.by_id(ini)
        scale = np.sqrt(want["ux"] ** 2 + want["uy"] ** 2 + want["uz"] ** 2).max()
        for k in ("ux", "uy", "uz"):
            err = np.abs(got[k] - want[k]).max() / scale
            assert err <= 1e-13, (k, err)
        for k in ("x", "y", "z", "w", "id"):
            assert np.array_equal(got[k], ini[k]), k
        assert np.mean(got["ux"] != ini["ux"]) > 0.3


def test_device_stage_does_not_depend_on_storage_order(dev):
    sp1, sp2, coll = cases("ei")
    p1 = np.random.default_rng(1).permutation(len(sp1["x"]))
    p2 = np.random.default_rng(2).permutation(len(sp2["x"]))
    a1, a2, _ = run(dev, sp1, sp2, coll, 3e-15, 9)
    b1, b2, _ = run(dev, {k: v[p1] for k, v in sp1.items()}, {k: v[p2] for k, v in sp2.items()}, coll, 3e-15, 9, pending=False)
    for a, b in ((a1, b1), (a2, b2)):
        a, b = cc.by_id(a), cc.by_id(b)
        for k in a:
            assert np.array_equal(a[k], b[k]), k


def deck_sim(wl, solver=abi.SOLVER_NONE, collisions=None):
    from warpx_b200.engine import Simulation
    sim = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=1, solver=solver, dt=wl["dt"])
    for s in wl["species"]:
        sim.add_species(s["name"], s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    for c in (wl["collisions"] if collisions is None else collisions):
        sim.add_collision(c["species"][0], c["species"][1], coulomb_log=c["coulomb_log"], ndt=c["ndt"], seed=c["seed"])
    return sim


def test_xyz_deck_relaxes_the_drift_as_the_reference_analysis_expects(cuda):
    """analysis_collision_3d.py: mean over steps 0, 10, ..., 150 of |a exp(b j) - (<ux>_e - <ux>_i)/c| < 0.001."""
    wl = workloads.collision_xyz_3d()
    sim = deck_sim(wl)
    an = wl["analysis"]
    err = []
    for j in range(0, wl["max_step"] + 1, 10):
        if j:
            sim.Evolve(10)
        vxd = float(sim.species[0].array("ux").mean()) / workloads.C - float(sim.species[1].array("ux").mean()) / workloads.C
        err.append(abs(an["a"] * np.exp(an["b"] * j) - vxd))
    print("XYZ deck: mean |fit - drift| = %.3e (tolerance %g)" % (np.mean(err), an["tolerance"]))
    assert np.mean(err) < an["tolerance"]
    sim.close()


def test_iso_deck_isotropises_as_the_reference_analysis_expects(cuda):
    """analysis_collision_3d_isotropization.py: Tx and Ty after 100 steps within 5 % of the analytic relaxation."""
    import scipy.constants as sc
    wl = workloads.collision_iso_3d()
    sim = deck_sim(wl)
    sim.Evolve(wl["max_step"])
    an = wl["analysis"]
    e, m, dt = sc.e, sc.m_e, wl["dt"]
    T_par, T_per = an["T_par"] * e, an["T_per"] * e
    A = 1.0 - T_per / T_par
    mu = (e ** 4 * an["ne"] * an["coulomb_log"] / (8.0 * np.pi ** 1.5 * sc.epsilon_0 ** 2 * m ** 0.5 * T_par ** 1.5)
          * A ** (-2) * (-3.0 + (3.0 - A) * np.arctanh(A ** 0.5) / A ** 0.5))
    Tx0, Ty0 = T_par, T_per
    for _ in range(wl["max_step"] - 1):
        Tx0 = Tx0 + dt * mu * (Ty0 - Tx0) * 2.0
        Ty0 = Ty0 + dt * mu * (Tx0 - Ty0)
    me = workloads.M_E
    Tx = float((sim.species[0].array("ux") ** 2).mean()) * me / e
    Ty = float((sim.species[0].array("uy") ** 2).mean()) * me / e
    err = max(abs(Tx - Tx0 / e) / Tx, abs(Ty - Ty0 / e) / Ty)
    print("ISO deck: Tx %.4f eV (analytic %.4f), Ty %.4f eV (analytic %.4f), error %.3e" % (Tx, Tx0 / e, Ty, Ty0 / e, err))
    assert err < an["tolerance"]
    sim.close()


def test_device_xyz_loop_matches_oracle_loop(cuda):
    """The full-size xyz deck for 30 steps (three collision calls of each of the three collisions) against
    collision_oracle.deck_loop: 1e-10 in u/c per particle."""
    wl = workloads.collision_xyz_3d()
    sim = deck_sim(wl)
    sim.Evolve(30)
    geom = dict(n_cell=wl["n_cell"], prob_lo=wl["prob_lo"], prob_hi=wl["prob_hi"], box_lo=(0, 0, 0),
                box_hi=tuple(v - 1 for v in wl["n_cell"]))
    species = [dict(s, id=np.arange(len(s["x"]), dtype=np.int64)) for s in wl["species"]]
    co.deck_loop(species, wl["collisions"], geom, wl["dt"], 30)
    for isp in range(2):
        got, want = sim.species_numpy(isp, sort_by_id=True), cc.by_id(species[isp])
        err = max(np.abs(got[k] - want[k]).max() for k in ("ux", "uy", "uz")) / workloads.C
        print("XYZ loop vs oracle, species %d: max |du|/c = %.3e" % (isp, err))
        assert err <= 1e-10
    sim.close()


def test_restart_continues_an_xyz_run_bit_for_bit(cuda, tmp_path):
    from warpx_b200 import diagnostics
    from warpx_b200.engine import Simulation
    wl = workloads.collision_xyz_3d(ppc=50)
    colls = [dict(c, ndt=3) for c in wl["collisions"]]
    a = deck_sim(wl, collisions=colls)
    a.Evolve(20)
    a.Evolve(20)
    b = deck_sim(wl, collisions=colls)
    b.Evolve(20)
    root = diagnostics.write_checkpoint(b, str(tmp_path / "chk"))
    b.close()
    c = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=1, solver=abi.SOLVER_NONE, dt=wl["dt"])
    diagnostics.read_checkpoint(c, root)
    for col in colls:
        c.add_collision(col["species"][0], col["species"][1], coulomb_log=col["coulomb_log"], ndt=col["ndt"], seed=col["seed"])
    c.Evolve(20)
    for isp in range(2):
        x, y = a.species_numpy(isp, sort_by_id=True), c.species_numpy(isp, sort_by_id=True)
        for k in x:
            assert np.array_equal(x[k], y[k]), (isp, k)
    a.close()
    c.close()


def test_gauss_weights_and_count_with_yee_and_collisions_every_step(cuda):
    """The benchmark's plasma at 128^3 x 8 ppc, order 3, Yee, with electron-electron collisions every step (a sort
    before every collision): Gauss's law within 1e-11, the count and the weights by id kept (test_gpu_gauss.run_gauss)."""
    from test_gpu_gauss import bench_workload, make_sim, run_gauss
    sim = make_sim(bench_workload(128))
    sim.add_collision(0, 0, coulomb_log=-1.0, ndt=1, seed=5)
    sim.enable_stage_timing(True)
    try:
        run_gauss(sim, (1, 4, 5, 20), "collisions")
        assert sim.stage_ms()["collisions"][1] == 20
    finally:
        sim.close()


@pytest.mark.parametrize("name", sorted(cc.reference_cases()))
def test_device_stage_matches_reference_headers(dev, name):
    L, t, d = dev
    sp1, sp2, coll, geom, dt, step, u1, u2 = cc.reference_cases()[name]
    g1, g2, status = cc.run_stage(L, t, d, sp1, sp2, coll, geom, dt, step, stream=t.cuda.current_stream().cuda_stream,
                                  sync=t.cuda.synchronize)
    assert status == 0
    cc.assert_matches_reference(g1, sp1, u1, 1e-13, geom)
    if sp2 is not None:
        cc.assert_matches_reference(g2, sp2, u2, 1e-13, geom)


@pytest.mark.parametrize("kind", ["ee", "ei"])
def test_device_cells_beyond_shared_memory_match_oracle(dev, kind):
    from test_collision_reference import huge_cells
    sp1, sp2 = huge_cells()
    coll = cc.ee_spec(L=-1.0) if kind == "ee" else cc.ei_spec(L=-1.0)
    if kind == "ee":
        sp2 = None
    g1, g2, status = run(dev, sp1, sp2, coll, 3e-15, 6)
    assert status == 0
    r1, r2 = co.collide({k: v.copy() for k, v in sp1.items()}, None if sp2 is None else {k: v.copy() for k, v in sp2.items()},
                        coll, cc.GEOM, 3e-15, 6)
    for got, sp, r in ((g1, sp1, r1), (g2, sp2, r2)):
        if sp is not None:
            cc.assert_matches_reference(got, sp, r, 1e-13)
