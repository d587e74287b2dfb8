"""GPU tests (-m gpu) of the two-product nuclear fusion (csrc/fusion.cu and the C++ driver's fusion stages):

  * the device passes against the numpy restatement (tests/fusion_oracle.py) on seeded multi-cell sets of all three
    reactions -- Poisson counts, cells of 0 to 3 and 300 particles, log-uniform weights, the threshold branch, through a
    pending permutation and on moved particles: identical events and spent reactants, products in the same order with
    positions and ids exact, momenta and weights to 1e-13;
  * a cell of 10 000 D + 10 000 T (the in-place path the decks take) against the restatement;
  * two storage orders of the same particles give the same reactants per id and the same products, bit for bit;
  * a product species without room fails with a clear error;
  * the step driver: a D-T run through Simulation creates what the restatement creates and removes the spent
    reactants."""
import numpy as np
import pytest

import fusion_cases as fc
import fusion_oracle as fo
from warpx_b200 import abi

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(cuda):
    from warpx_b200.lib import lib
    return lib(), cuda, cuda.device("cuda", 0)


def counts(seed, mean=4.0, big=300):
    rng = np.random.default_rng(seed)
    n = rng.poisson(mean, size=(4, 5, 6))
    n[0, 0, 0:4] = (0, 1, 2, 3)
    n[1, 1, 1] = big
    return n


def run(dev, sp1, sp2, f, dt, step, **kw):
    L, t, d = dev
    return fc.run_stage(L, t, d, sp1, sp2, f, dt, step, stream=t.cuda.current_stream().cuda_stream,
                        sync=t.cuda.synchronize, **kw)


def case(kind, weights="log"):
    if kind == "dt":
        f = fc.spec(abi.FUSION_DT_NHE4, mult=1.0e20)
        return f, fc.reactants(1, counts(1), f["m1"], 30.0, weights=weights), \
            fc.reactants(2, counts(2, 3.0, 150), f["m2"], 30.0, weights=weights, id_offset=10 ** 6)
    f = fc.spec(abi.FUSION_DD_PT if kind == "dd_pt" else abi.FUSION_DD_NHE3, mult=1.0e20)
    return f, fc.reactants(3, counts(3, 5.0, 301), f["m1"], 30.0, weights=weights), None


@pytest.mark.parametrize("dt", [1e-13, 1e-9])
@pytest.mark.parametrize("kind", ["dt", "dd_pt", "dd_nhe3"])
@pytest.mark.parametrize("pending", [True, False])
def test_device_stage_matches_oracle(dev, dt, kind, pending):
    f, sp1, sp2 = case(kind)
    g1, g2, gA, gB, status = run(dev, sp1, sp2, f, dt, 7, pending=pending)
    assert status == 0
    w1, w2, wA, wB = fo.fuse(sp1, sp2, f, fc.GEOM, dt, 7)
    assert len(wA["x"]) > 0
    fc.assert_matches(g1, w1, 1e-14, "reactant")
    if sp2 is not None:
        fc.assert_matches(g2, w2, 1e-14, "reactant")
    fc.assert_matches(gA, wA, 1e-13, "product")
    fc.assert_matches(gB, wB, 1e-13, "product")


def test_device_large_cell_matches_oracle(dev):
    f = fc.spec(abi.FUSION_DT_NHE4, mult=1.0e50)           # the multiplier of deck DT test 1: the threshold branch
    n = np.zeros((4, 5, 6), dtype=int)
    n[2, 3, 1] = 10000
    sp1 = fc.reactants(31, n, f["m1"], 0.0, drift_keV=200.0)
    sp2 = fc.reactants(32, n, f["m2"], 20.0, id_offset=10 ** 6)
    g1, g2, gA, gB, status = run(dev, sp1, sp2, f, 1e-12, 0)
    assert status == 0
    w1, w2, wA, wB = fo.fuse(sp1, sp2, f, fc.GEOM, 1e-12, 0)
    assert len(wA["x"]) > 1000
    fc.assert_matches(g1, w1, 1e-14, "reactant")
    fc.assert_matches(g2, w2, 1e-14, "reactant")
    fc.assert_matches(gA, wA, 1e-13, "product")
    fc.assert_matches(gB, wB, 1e-13, "product")


def test_device_storage_order_independence(dev):
    f, sp1, sp2 = case("dt")
    rng = np.random.default_rng(5)
    o1, o2 = rng.permutation(len(sp1["x"])), rng.permutation(len(sp2["x"]))
    a = run(dev, sp1, sp2, f, 1e-9, 2)
    b = run(dev, {k: v[o1] for k, v in sp1.items()}, {k: v[o2] for k, v in sp2.items()}, f, 1e-9, 2)
    for x, y in zip(a[:2], b[:2]):
        x, y = fc.by_id(x), fc.by_id(y)
        live = x["id"] != -1                        # spent reactants share one id: compare them as a set
        assert np.array_equal(live, y["id"] != -1)
        for k in x:
            assert np.array_equal(x[k][live], y[k][live]), k
            assert np.array_equal(np.sort(x[k][~live]), np.sort(y[k][~live])), k
    for x, y in zip(a[2:4], b[2:4]):
        assert len(x["x"]) > 0
        for k in x:
            assert np.array_equal(x[k], y[k]), k


def test_device_capacity_overflow_is_refused(dev):
    f, sp1, sp2 = case("dt")
    L = dev[0]
    L.pic_set_error_mode(abi.PIC_ERR_RETURN)     # a refusal returns an error instead of aborting
    try:
        with pytest.raises(RuntimeError, match="product A needs a capacity of"):
            run(dev, sp1, sp2, f, 1e-9, 0, cap=4)
    finally:
        L.pic_set_error_mode(abi.PIC_ERR_ABORT)


def test_driver_dt_run_matches_oracle(dev):
    from warpx_b200.engine import Simulation
    f = fc.spec(abi.FUSION_DT_NHE4, mult=1.0e25)
    sp1 = fc.reactants(41, 20.0, f["m1"], 40.0)
    sp2 = fc.reactants(42, 20.0, f["m2"], 40.0, id_offset=10 ** 6)
    sim = Simulation(fc.GEOM["n_cell"], fc.GEOM["prob_lo"], fc.GEOM["prob_hi"], nox=1, solver=abi.SOLVER_NONE, dt=5e-15)
    for name, sp, st in (("d", sp1, "deuterium"), ("t", sp2, "tritium")):
        q, m = fc.species_charge_mass(st)
        sim.add_species(name, q, m, sp["x"], sp["y"], sp["z"], sp["w"], sp["ux"], sp["uy"], sp["uz"], species_type=st,
                        ids=sp["id"])
    cap = len(sp1["x"]) + len(sp2["x"])
    sim.add_empty_species("he4", cap, species_type="helium4")
    sim.add_empty_species("n", cap, species_type="neutron")
    sim.add_fusion("d", "t", ("he4", "n"), multiplier=1.0e25, seed=11)
    sim.Evolve(1)
    f["seed"] = 11
    w1, w2, wA, wB = fo.fuse(sp1, sp2, f, fc.GEOM, 5e-15, 0)
    nums = sim.particle_number()
    assert nums[2][0] == len(wA["x"]) > 0 and nums[3][0] == len(wB["x"])
    assert abs(nums[2][1] - wA["w"].sum()) <= 1e-12 * wA["w"].sum()
    assert nums[0][0] == int((w1["id"] != -1).sum()) and nums[1][0] == int((w2["id"] != -1).sum())
    got = fc.by_id(sim.species_numpy(2))
    assert np.array_equal(got["id"], np.arange(len(wA["x"])))
    for k in ("ux", "uy", "uz"):
        scale = np.abs(wA[k]).max()
        assert np.abs(got[k] - wA[k]).max() <= 1e-13 * scale     # gather of zero fields leaves u unchanged
