"""CPU tests of proton-boron fusion (p + B11 -> 3 He4) and of the do_not_push / do_not_deposit species flags: the kernel
source (csrc/fusion.cu, csrc/engine.cu, through the SIMT host build of tests/host_harness) against the numpy restatement
of tests/proton_boron_oracle.py, the exact invariants of one stage, the C++ driver's use of both and its refusals."""
import numpy as np
import pytest

import fusion_cases as fc
import proton_boron_cases as pc
import proton_boron_oracle as po
from warpx_b200 import abi
from warpx_b200.engine import nuclear_fusion_type, species_charge_mass


@pytest.fixture(scope="module")
def host():
    import torch
    from host_harness import harness
    return harness.host_library(), torch


def counts(seed, mean=4.0, big=0):
    rng = np.random.default_rng(seed)
    n = rng.poisson(mean, size=(4, 5, 6))
    n[0, 0, 0:4] = (0, 1, 2, 3)
    if big:
        n[1, 1, 1] = big                  # a cell for the block-per-cell path
    return n


def case(boron_first=False, E_keV=300.0, mult=1e5, thr=1e300, target=0.002, weights="log", big=(300, 150)):
    f = pc.spec(boron_first, mult=mult, thr=thr, target=target)
    sp1 = fc.reactants(41, counts(41, 4.0, big[0]), f["m1"], E_keV, weights=weights)
    sp2 = fc.reactants(42, counts(42, 3.0, big[1]), f["m2"], E_keV, weights=weights, id_offset=10 ** 6)
    return f, sp1, sp2


# (dt, threshold): no events, probabilities ~0.2, and the threshold branch
@pytest.mark.parametrize("dt,thr", [(1e-18, 0.02), (1e-13, 1e300), (1e-9, 0.02)])
@pytest.mark.parametrize("boron_first", [False, True])
@pytest.mark.parametrize("pending", [True, False])
def test_host_stage_matches_oracle(host, dt, thr, boron_first, pending):
    L, t = host
    f, sp1, sp2 = case(boron_first, thr=thr)
    g1, g2, gA, status = pc.run_stage(L, t, "cpu", sp1, sp2, f, dt, 5, pending=pending)
    assert status == 0
    w1, w2, wA = po.fuse(sp1, sp2, f, pc.GEOM, dt, 5)
    fc.assert_matches(g1, w1, 1e-14, "reactant")
    fc.assert_matches(g2, w2, 1e-14, "reactant")
    fc.assert_matches(gA, wA, 1e-13, "product")
    if dt >= 1e-13:
        assert len(wA["x"]) > 0


def test_host_stage_large_cells_in_place(host):
    """cells above 2048 particles take the in-place canonical-order path; same result as the restatement"""
    L, t = host
    f, sp1, sp2 = case(big=(2500, 1500), mult=1e4)
    g1, g2, gA, status = pc.run_stage(L, t, "cpu", sp1, sp2, f, 1e-13, 2)
    assert status == 0
    w1, w2, wA = po.fuse(sp1, sp2, f, pc.GEOM, 1e-13, 2)
    fc.assert_matches(g1, w1, 1e-14, "reactant")
    fc.assert_matches(g2, w2, 1e-14, "reactant")
    fc.assert_matches(gA, wA, 1e-13, "product")
    assert len(wA["x"]) > 0


def test_host_stage_independent_of_storage_order(host):
    L, t = host
    f, sp1, sp2 = case()
    a1, a2, aA, _ = pc.run_stage(L, t, "cpu", sp1, sp2, f, 1e-13, 3)
    rng = np.random.default_rng(5)
    o1, o2 = rng.permutation(len(sp1["x"])), rng.permutation(len(sp2["x"]))
    b1, b2, bA, _ = pc.run_stage(L, t, "cpu", {k: v[o1] for k, v in sp1.items()}, {k: v[o2] for k, v in sp2.items()},
                                 f, 1e-13, 3)
    assert len(aA["x"]) > 0
    for k in aA:
        assert np.array_equal(aA[k], bA[k]), k
    for a, b in ((a1, b1), (a2, b2)):
        a, b = fc.by_id(a), fc.by_id(b)
        for k in a:
            assert np.array_equal(a[k], b[k]), k


def test_host_stage_conserves_weight_charge_momentum_energy(host):
    L, t = host
    # multiplier 1 and probabilities ~1: every event takes a whole macroparticle's weight, which the sums resolve
    f, sp1, sp2 = case(E_keV=500.0, mult=1.0)
    g1, g2, gA, _ = pc.run_stage(L, t, "cpu", sp1, sp2, f, 1e-5, 0)
    n = len(gA["x"])
    assert n > 0 and n % 6 == 0
    # weight: each reactant loses what the alphas gain over three (pending=True: the buffers keep the storage order)
    lost1, lost2 = (sp1["w"] - g1["w"]).sum(), (sp2["w"] - g2["w"]).sum()
    assert lost1 > 0 and abs(lost1 - lost2) <= 1e-12 * lost1
    assert abs(gA["w"].sum() / 3.0 - lost1) <= 1e-12 * lost1
    # charge: 1 + 5 elementary charges per reaction weight become 3 x 2
    qa = species_charge_mass("helium4")[0]
    assert abs(gA["w"].sum() * qa - lost1 * (f["q1"] + f["q2"])) <= 1e-12 * lost1 * (f["q1"] + f["q2"])
    # per event: momentum and energy of the two reactants go to the three alphas, plus Q
    ev = n // 6
    u = np.stack([gA[k] for k in ("ux", "uy", "uz")]).reshape(3, ev, 3, 2)      # [d, event, alpha, side]
    assert np.array_equal(u[..., 0], u[..., 1])
    # the reactants of each event: the particles at the alphas' positions
    idx1 = {p: i for i, p in enumerate(zip(sp1["x"], sp1["y"], sp1["z"]))}
    idx2 = {p: i for i, p in enumerate(zip(sp2["x"], sp2["y"], sp2["z"]))}
    pos = np.stack([gA[k] for k in ("x", "y", "z")]).reshape(3, ev, 3, 2)
    for al in range(3):
        assert np.array_equal(pos[:, :, al, :], pos[:, :, 0, :])
    a = np.array([idx1[tuple(pos[:, e, 0, 0])] for e in range(ev)])
    b = np.array([idx2[tuple(pos[:, e, 0, 1])] for e in range(ev)])
    c2, ma = po.C_SQ, po.M_ALPHA
    p_in = np.stack([f["m1"] * sp1[k][a] + f["m2"] * sp2[k][b] for k in ("ux", "uy", "uz")])
    p_out = ma * u[..., 0].sum(axis=2)
    assert np.abs(p_out - p_in).max() <= 1e-13 * np.abs(p_in).max()

    def kinetic(m, ux, uy, uz):
        usq = (ux * ux + uy * uy + uz * uz) / c2
        return m * c2 * usq / (np.sqrt(1.0 + usq) + 1.0)
    k_in = kinetic(f["m1"], sp1["ux"][a], sp1["uy"][a], sp1["uz"][a]) + kinetic(f["m2"], sp2["ux"][b], sp2["uy"][b],
                                                                              sp2["uz"][b])
    k_out = sum(kinetic(ma, u[0, :, al, 0], u[1, :, al, 0], u[2, :, al, 0]) for al in range(3))
    # Q of the reaction with the masses of the kinematics: m_p + m_B11 - 3 m_alpha = E_fusion + E_decay (to the
    # precision of the mass table)
    mass_q = (f["m1"] + f["m2"] - 3.0 * ma) * c2
    assert abs(mass_q - po.Q_TOTAL) <= 2e-3 * po.Q_TOTAL
    assert np.abs(k_out - (k_in + po.Q_TOTAL)).max() <= 1e-8 * po.Q_TOTAL
    assert np.unique(gA["id"]).size == gA["id"].size


def test_host_capacity_overflow_is_refused(host):
    L, t = host
    f, sp1, sp2 = case(E_keV=500.0, mult=1.0)
    with pytest.raises(RuntimeError, match="needs a capacity"):
        pc.run_stage(L, t, "cpu", sp1, sp2, f, 1e-5, 0, cap=6)


def test_fusion_type_and_species_table():
    q, m = species_charge_mass("boron11")
    assert q == 5 * 1.602176634e-19 and m == 11.00930536 * 1.66053906660e-27
    assert nuclear_fusion_type(["hydrogen1", "boron11"], ["helium4"]) == abi.FUSION_PB_3HE4
    assert nuclear_fusion_type(["boron11", "hydrogen1"], ["helium4"]) == abi.FUSION_PB_3HE4
    for bad in (["helium4", "helium4"], ["hydrogen1"], []):
        with pytest.raises(ValueError):
            nuclear_fusion_type(["hydrogen1", "boron11"], bad)


def _pb_sim(Sim, w_scale=1e25, solver=abi.SOLVER_NONE, boron_first=False, **kw):
    f = pc.spec(boron_first)
    sp1 = fc.reactants(51, 6.0, f["m1"], 400.0)
    sp2 = fc.reactants(52, 6.0, f["m2"], 400.0, id_offset=10 ** 6)
    sp1["w"] = sp1["w"] * w_scale
    sp2["w"] = sp2["w"] * w_scale
    sim = Sim(fc.GEOM["n_cell"], fc.GEOM["prob_lo"], fc.GEOM["prob_hi"], nox=1, solver=solver,
              dt=(5e-15 if solver == abi.SOLVER_NONE else None), **kw)
    names = ("b", "p") if boron_first else ("p", "b")
    for name, sp, st in zip(names, (sp1, sp2), ("boron11", "hydrogen1") if boron_first else ("hydrogen1", "boron11")):
        q, m = species_charge_mass(st)
        sim.add_species(name, q, m, sp["x"], sp["y"], sp["z"], sp["w"], sp["ux"], sp["uy"], sp["uz"], species_type=st,
                        ids=sp["id"])
    cap = 12 * (len(sp1["x"]) + len(sp2["x"]))          # two steps' worth of events
    sim.add_empty_species("alpha", cap, species_type="helium4")
    return sim


@pytest.mark.parametrize("boron_first", [False, True])
def test_host_driver_runs_proton_boron(host, boron_first):
    from host_harness import harness
    sim = _pb_sim(harness.host_simulation_class(), boron_first=boron_first)
    sim.add_empty_species("he4b", 10, species_type="helium4")
    for bad in (("alpha", "he4b"), ("p",), ("he4b", "alpha", "alpha")):
        with pytest.raises((RuntimeError, ValueError)):
            sim.add_fusion("p", "b", bad)
    # the engine refuses -1 for a two-product type and two products for proton-boron
    assert sim.L.pic_engine_add_fusion(sim.native, 0, 1, 2, 3, abi.FUSION_PB_3HE4, 1.0, 0.02, 0.002, 1, 0) != 0
    assert sim.L.pic_engine_add_fusion(sim.native, 0, 1, 2, -1, abi.FUSION_DT_NHE4, 1.0, 0.02, 0.002, 1, 0) != 0
    assert sim.collisions == []
    sim.add_fusion("p", "b", ["alpha"], multiplier=1e3, probability_threshold=1e300)
    w0 = [w for _, w in sim.particle_number()]
    sim.Evolve(1)
    nums = sim.particle_number()
    assert nums[2][0] > 0 and nums[2][0] % 6 == 0
    lost = w0[0] - nums[0][1]
    assert lost > 0 and abs(nums[2][1] / 3.0 - lost) <= 1e-12 * lost
    assert abs((w0[1] - nums[1][1]) - lost) <= 1e-12 * lost
    ids = sim.species_numpy(2)["id"]
    assert np.array_equal(np.sort(ids), np.arange(len(ids)))
    assert sim.species_next_id(2) == len(ids)


FLAG_GEOM = dict(n_cell=(12, 12, 12), prob_lo=(0.0, 0.0, 0.0), prob_hi=(12e-6, 12e-6, 12e-6), box_lo=(0, 0, 0),
                 box_hi=(11, 11, 11))


def _flag_sim(Sim, ions=True):
    """electrons (and ions) in fields that are not zero, Yee solver, sorted at every step"""
    import collision_cases as cc
    g = FLAG_GEOM
    sim = Sim(g["n_cell"], g["prob_lo"], g["prob_hi"], nox=2, sort_interval=1)
    rng = np.random.default_rng(3)
    for c in range(6):
        sim.set_field(c, rng.standard_normal(sim.data[c].shape) * (1e9 if c < 3 else 3.0))
    for k, (name, q) in enumerate((("e", -1.602176634e-19), ("i", 1.602176634e-19))[:2 if ions else 1]):
        sp = cc.particle_set(60 + k, g, 5.0, (0.05, 0.05, 0.05), w0=1e6)
        sim.add_species(name, q, 9.1093837015e-31 * (1 if k == 0 else 1836.0), sp["x"], sp["y"], sp["z"], sp["w"],
                        sp["ux"], sp["uy"], sp["uz"], ids=sp["id"])
    return sim


def test_host_do_not_push_keeps_positions_and_momenta(host):
    from host_harness import harness
    sim = _flag_sim(harness.host_simulation_class())
    before = sim.species_numpy(1, sort_by_id=True)
    e_before = sim.species_numpy(0, sort_by_id=True)
    sim.set_species_flags("i", do_not_push=True)
    assert sim.species[1].do_not_push and not sim.species[1].do_not_deposit
    sim.Evolve(2, synchronize_last=False)
    sim.Evolve(3)
    after = sim.species_numpy(1, sort_by_id=True)
    for k in before:
        assert np.array_equal(before[k], after[k]), k
    e_after = sim.species_numpy(0, sort_by_id=True)
    assert not np.array_equal(e_before["ux"], e_after["ux"])          # the other species moved
    # sorted at every step: the bins hold the unpushed species in cell order
    _, rho = sim.rho_numpy()
    assert np.isfinite(rho).all()


def test_host_do_not_deposit_is_as_if_absent(host):
    from host_harness import harness
    Sim = harness.host_simulation_class()
    a = _flag_sim(Sim)
    i0 = a.species_numpy(1, sort_by_id=True)
    a.set_species_flags(1, do_not_deposit=True)
    a.Evolve(3)
    ref = _flag_sim(Sim, ions=False)               # the same run without the ions
    ref.Evolve(3)
    for comp in range(9):
        assert np.array_equal(a.field_numpy(comp)[1], ref.field_numpy(comp)[1]), comp
    assert np.array_equal(a.rho_numpy()[1], ref.rho_numpy()[1])
    assert a.field_numpy(6)[1].any()
    i1 = a.species_numpy(1, sort_by_id=True)
    assert not np.array_equal(i0["ux"], i1["ux"])      # the flagged species was pushed


def test_host_flagged_species_still_fuse(host):
    from host_harness import harness
    sim = _pb_sim(harness.host_simulation_class())
    for name in ("p", "b", "alpha"):
        sim.set_species_flags(name, do_not_push=True, do_not_deposit=True)
    b0 = sim.species_numpy(1, sort_by_id=True)
    sim.add_fusion("p", "b", ["alpha"], multiplier=1e3, probability_threshold=1e300)
    sim.Evolve(2)
    assert sim.particle_number()[2][0] > 0
    b1 = sim.species_numpy(1, sort_by_id=True)
    live = np.isin(b0["id"], b1["id"])
    for k in ("x", "y", "z", "ux", "uy", "uz"):
        assert np.array_equal(b0[k][live], b1[k]), k


def test_host_bad_species_index_is_refused(host):
    from host_harness import harness
    sim = _flag_sim(harness.host_simulation_class())
    for bad in (2, -1):
        with pytest.raises(RuntimeError, match="no species"):
            sim.set_species_flags(bad, do_not_push=True)
    with pytest.raises(ValueError):
        sim.set_species_flags("nope", do_not_push=True)
    assert not any(sp.do_not_push or sp.do_not_deposit for sp in sim.species)
