"""CPU tests of the two-product nuclear fusion: the product's kernel source (csrc/fusion.cu, through the SIMT host build of
tests/host_harness) against the numpy restatement of tests/fusion_oracle.py, the exact invariants of one stage, the C++
driver's fusion loop and its refusals."""
import numpy as np
import pytest

import fusion_cases as fc
import fusion_oracle as fo
from warpx_b200 import abi


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


def case(kind, E_keV=30.0, weights="equal"):
    if kind == "dt":
        f = fc.spec(abi.FUSION_DT_NHE4, mult=1.0e20, thr=0.02, target=0.002)
        sp1 = fc.reactants(1, counts(1), f["m1"], E_keV, weights=weights)
        sp2 = fc.reactants(2, counts(2, 3.0, 150), f["m2"], E_keV, weights=weights, id_offset=10 ** 6)
        return f, sp1, sp2
    f = fc.spec(abi.FUSION_DD_PT if kind == "dd_pt" else abi.FUSION_DD_NHE3, mult=1.0e20)
    return f, fc.reactants(3, counts(3, 5.0, 301), f["m1"], E_keV, weights=weights), None


def oracle(f, sp1, sp2, dt, step):
    return fo.fuse(sp1, sp2, f, fc.GEOM, dt, step)


# dt spans no events, some, and the threshold branch (probability estimates above 0.02 with the multiplier floor)
@pytest.mark.parametrize("dt", [1e-16, 1e-13, 1e-9])
@pytest.mark.parametrize("kind", ["dt", "dd_pt", "dd_nhe3"])
@pytest.mark.parametrize("pending", [True, False])
def test_host_stage_matches_oracle(host, dt, kind, pending):
    L, t = host
    f, sp1, sp2 = case(kind, weights="log" if kind == "dt" else "equal")
    g1, g2, gA, gB, status = fc.run_stage(L, t, "cpu", sp1, sp2, f, dt, 5, pending=pending)
    assert status == 0
    w1, w2, wA, wB = oracle(f, sp1, sp2, dt, 5)
    fc.assert_matches(g1, w1, 1e-14, "reactant")
    if sp2 is not None:
        fc.assert_matches(g2, w2, 1e-14, "reactant")
    fc.assert_matches(gA, wA, 1e-13, "product")
    fc.assert_matches(gB, wB, 1e-13, "product")
    if dt >= 1e-13:
        assert len(wA["x"]) > 0


def test_host_stage_conserves_weight_charge_momentum_energy(host):
    L, t = host
    f, sp1, sp2 = case("dt", E_keV=50.0, weights="log")
    g1, g2, gA, gB, _ = fc.run_stage(L, t, "cpu", sp1, sp2, f, 1e-9, 0)
    # weight: what the reactants lose, each product species gains
    lost = (sp1["w"].sum() - g1["w"].sum())
    assert lost > 0
    assert abs(gA["w"].sum() - lost) <= 1e-12 * lost and abs(gB["w"].sum() - lost) <= 1e-12 * lost
    assert abs((sp2["w"].sum() - g2["w"].sum()) - lost) <= 1e-12 * lost
    # products sit at their reactants' positions: first of each pair at a D, second at a T
    pos1 = set(zip(sp1["x"], sp1["y"], sp1["z"]))
    pos2 = set(zip(sp2["x"], sp2["y"], sp2["z"]))
    for P in (gA, gB):
        assert all(p in pos1 for p in zip(P["x"][0::2], P["y"][0::2], P["z"][0::2]))
        assert all(p in pos2 for p in zip(P["x"][1::2], P["y"][1::2], P["z"][1::2]))
    # per event: both products have momenta and energies of a two-body decay
    mA, mB = f["mA"], f["mB"]
    uA = np.stack([gA[k][0::2] for k in ("ux", "uy", "uz")])
    uB = np.stack([gB[k][0::2] for k in ("ux", "uy", "uz")])
    ps = mA * uA + mB * uB
    c2 = fo.C_SQ
    eA = mA * c2 * np.sqrt(1 + (uA * uA).sum(0) / c2)
    eB = mB * c2 * np.sqrt(1 + (uB * uB).sum(0) / c2)
    assert np.all(np.isfinite(ps)) and np.all(eA > mA * c2) and np.all(eB > mB * c2)
    # the products carry E_fusion plus the pair's kinetic energy (a few hundred keV at most here), the neutron about
    # four fifths of it
    kA, kB = eA - mA * c2, eB - mB * c2
    ef = fo.E_FUSION[fo.DT_NHE4]
    assert np.all(kA + kB > ef) and np.all(kA + kB < ef + 2e6 * fo.Q_E)
    share = kB / (kA + kB)
    assert abs(share.mean() - 0.8) < 0.02 and np.all(np.abs(share - 0.8) < 0.15), share
    assert np.unique(gA["id"]).size == gA["id"].size


def test_host_spent_reactants_are_skipped_by_later_pairs(host):
    """unequal counts in one cell with a probability of 1 (tiny multiplier floor): the lighter-weight partners are used
    up by their first pair and every later pair of their chain is skipped without a draw"""
    L, t = host
    f = fc.spec(abi.FUSION_DT_NHE4, mult=1.0, thr=1.0e300, target=0.002)
    n1 = np.zeros((4, 5, 6), dtype=int)
    n2 = np.zeros((4, 5, 6), dtype=int)
    n1[2, 2, 2], n2[2, 2, 2] = 3, 11
    n1[1, 1, 1], n2[1, 1, 1] = 2500, 40              # the in-place path of cells above 2048 particles
    sp1 = fc.reactants(7, n1, f["m1"], 60.0)
    sp2 = fc.reactants(8, n2, f["m2"], 60.0, id_offset=10 ** 6)
    sp1["w"] *= 1e30                                   # probability ~ 1 for every pair
    sp2["w"] *= 1e30
    g1, g2, gA, gB, status = fc.run_stage(L, t, "cpu", sp1, sp2, f, 1e-6, 3)
    assert status == 0
    w1, w2, wA, wB = oracle(f, sp1, sp2, 1e-6, 3)
    assert (w1["id"] == -1).sum() > 0 or (w2["id"] == -1).sum() > 0
    fc.assert_matches(g1, w1, 1e-14, "reactant")
    fc.assert_matches(g2, w2, 1e-14, "reactant")
    fc.assert_matches(gA, wA, 1e-13, "product")
    # a second call sees only the live particles
    sp1b = {k: v for k, v in g1.items()}
    sp2b = {k: v for k, v in g2.items()}
    h1, h2, hA, _, _ = fc.run_stage(L, t, "cpu", sp1b, sp2b, f, 1e-6, 4)
    v1, v2, vA, _ = oracle(f, sp1b, sp2b, 1e-6, 4)
    fc.assert_matches(h1, v1, 1e-14, "reactant")
    fc.assert_matches(hA, vA, 1e-13, "product")


def test_host_capacity_overflow_is_refused(host):
    L, t = host
    f, sp1, sp2 = case("dt", E_keV=50.0)
    with pytest.raises(RuntimeError, match="needs a capacity"):
        fc.run_stage(L, t, "cpu", sp1, sp2, f, 1e-9, 0, cap=2)


def test_host_driver_runs_fusion_and_removes_spent(host):
    from host_harness import harness
    Sim = harness.host_simulation_class()
    f = fc.spec(abi.FUSION_DT_NHE4)
    sp1 = fc.reactants(21, 6.0, f["m1"], 40.0)
    sp2 = fc.reactants(22, 6.0, f["m2"], 40.0, id_offset=10 ** 6)
    sp1["w"] = sp1["w"] * 1e30                          # probability ~ 1 for every pair
    sp2["w"] = sp2["w"] * 2e30                          # every event uses up its D, never its T
    sim = Sim(fc.GEOM["n_cell"], fc.GEOM["prob_lo"], fc.GEOM["prob_hi"], nox=1, solver=abi.SOLVER_NONE, dt=5e-15)
    for name, sp, st in (("d", sp1, "deuterium"), ("t", sp2, "tritium")):
        q, m = fc.species_charge_mass(st)
        sim.add_species(name, q, m, sp["x"], sp["y"], sp["z"], sp["w"], sp["ux"], sp["uy"], sp["uz"], species_type=st,
                        ids=sp["id"])
    cap = 2 * (len(sp1["x"]) + len(sp2["x"]))
    sim.add_empty_species("he4", cap, species_type="helium4")
    sim.add_empty_species("n", cap, species_type="neutron")
    # refusals leave the engine untouched
    for bad in (dict(products=("d", "n")), dict(products=("he4", "he4")), dict(products=("he4",))):
        with pytest.raises((RuntimeError, ValueError)):
            sim.add_fusion("d", "t", **bad)
    with pytest.raises(ValueError):
        sim.add_fusion("d", "d", ("he4", "n"))
    with pytest.raises(RuntimeError):
        sim.add_fusion("d", "t", ("he4", "n"), ndt=0)
    assert sim.collisions == []
    sim.add_fusion("d", "t", ("he4", "n"), probability_threshold=1e300)
    w0 = [w for _, w in sim.particle_number()]
    sim.Evolve(1)
    nums = sim.particle_number()
    assert nums[2][0] > 0 and nums[2][0] == nums[3][0]
    lost = w0[0] - nums[0][1]
    assert abs(nums[2][1] - lost) <= 1e-12 * lost
    assert abs((w0[1] - nums[1][1]) - lost) <= 1e-12 * lost
    d = sim.species_numpy(0)
    assert np.all(d["id"] != -1) and np.all(d["w"] > 0)       # spent D left the run
    assert nums[0][0] < len(sp1["x"])
    ids = sim.species_numpy(2)["id"]
    assert np.array_equal(np.sort(ids), np.arange(len(ids)))


def _dt_run(Sim, seed=21, w_scale=(1e30, 2e30), cap_factor=2):
    f = fc.spec(abi.FUSION_DT_NHE4)
    sp1 = fc.reactants(seed, 6.0, f["m1"], 40.0)
    sp2 = fc.reactants(seed + 1, 6.0, f["m2"], 40.0, id_offset=10 ** 6)
    sp1["w"] = sp1["w"] * w_scale[0]
    sp2["w"] = sp2["w"] * w_scale[1]
    sim = Sim(fc.GEOM["n_cell"], fc.GEOM["prob_lo"], fc.GEOM["prob_hi"], nox=1, solver=abi.SOLVER_NONE, dt=5e-15)
    for name, sp, st in (("d", sp1, "deuterium"), ("t", sp2, "tritium")):
        q, m = fc.species_charge_mass(st)
        sim.add_species(name, q, m, sp["x"], sp["y"], sp["z"], sp["w"], sp["ux"], sp["uy"], sp["uz"], species_type=st,
                        ids=sp["id"])
    cap = cap_factor * (len(sp1["x"]) + len(sp2["x"]))
    sim.add_empty_species("he4", cap, species_type="helium4")
    sim.add_empty_species("n", cap, species_type="neutron")
    return sim, cap


def test_host_coulomb_after_fusion_on_a_reactant_is_refused(host):
    """a Coulomb entry that would follow a fusion on a shared species would meet the spent reactants of that step"""
    from host_harness import harness
    sim, _ = _dt_run(harness.host_simulation_class())
    sim.add_fusion("d", "t", ("he4", "n"))
    for pair in (("d", "d"), ("t", "d"), ("d", "t"), ("t", "t")):
        with pytest.raises(RuntimeError, match="earlier fusion"):
            sim.add_collision(*pair)
    assert len(sim.collisions) == 1
    sim.add_collision("he4", "he4")                      # products are never spent
    sim2, _ = _dt_run(harness.host_simulation_class())
    sim2.add_collision("d", "t")                         # before the fusion: runs first in every step
    sim2.add_fusion("d", "t", ("he4", "n"))
    sim2.Evolve(1)
    assert sim2.particle_number()[2][0] > 0


def test_host_restart_continues_product_ids(host, tmp_path):
    """a checkpoint carries the product species' id counters and types: the restarted run continues bit for bit"""
    from host_harness import harness
    from warpx_b200 import diagnostics
    Sim = harness.host_simulation_class()
    sim, cap = _dt_run(Sim, seed=31, w_scale=(1e29, 1e29))
    sim.add_fusion("d", "t", ("he4", "n"), probability_threshold=1e300, seed=3)
    sim.Evolve(1)
    n1 = sim.particle_number()[2][0]
    assert n1 > 0 and sim.species_next_id(2) == n1
    root = diagnostics.write_checkpoint(sim, str(tmp_path / "chk"), 1)
    ref = sim
    ref.Evolve(1)
    # the restarted run: same species, types and capacities, the fusion registered again
    r = Sim(fc.GEOM["n_cell"], fc.GEOM["prob_lo"], fc.GEOM["prob_hi"], nox=1, solver=abi.SOLVER_NONE, dt=5e-15)
    diagnostics.read_checkpoint(r, root, capacity={"he4": cap, "n": cap})
    assert [sp.species_type for sp in r.species] == ["hydrogen2", "hydrogen3", "helium4", "neutron"]
    assert r.species_next_id(2) == n1
    r.add_fusion("d", "t", ("he4", "n"), probability_threshold=1e300, seed=3)
    r.Evolve(1)
    for isp in range(4):
        a, b = ref.species_numpy(isp, sort_by_id=True), r.species_numpy(isp, sort_by_id=True)
        for k in a:
            assert np.array_equal(a[k], b[k]), (isp, k)
    # a counter below the particle count is refused
    with pytest.raises(RuntimeError):
        r.set_species_next_id(2, 0)
