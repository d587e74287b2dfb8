"""GPU tests (-m gpu) of proton-boron fusion (csrc/fusion.cu, PIC_FUSION_PB_3HE4) and of the do_not_push /
do_not_deposit species flags in the C++ driver:

  * the device passes against the numpy restatement (tests/proton_boron_oracle.py) with the proton or the boron as
    species 1, through a pending permutation and on moved particles, with and without the threshold branch;
  * a cell of 10 000 protons + 10 000 borons (the in-place path) against the restatement;
  * two storage orders of the same particles give the same reactants per id and the same alphas, bit for bit;
  * the step driver: a species that is not pushed keeps x and u bit for bit over several steps in non-zero fields,
    sorted every step; a species that does not deposit leaves J and rho as if it were absent (to the round-off of the
    deposition's atomic sums); flagged species fuse."""
import numpy as np
import pytest

import fusion_cases as fc
import proton_boron_cases as pc
import proton_boron_oracle as po

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
    return pc.run_stage(L, t, d, sp1, sp2, f, dt, step, stream=t.cuda.current_stream().cuda_stream,
                        sync=t.cuda.synchronize, **kw)


def case(boron_first=False, thr=1e300, big=(300, 150), E_keV=300.0):
    f = pc.spec(boron_first, mult=1e5, thr=thr)
    sp1 = fc.reactants(41, counts(41, 4.0, big[0]), f["m1"], E_keV, weights="log")
    sp2 = fc.reactants(42, counts(42, 3.0, big[1]), f["m2"], E_keV, weights="log", id_offset=10 ** 6)
    return f, sp1, sp2


@pytest.mark.parametrize("dt,thr", [(1e-13, 1e300), (1e-9, 0.02)])
@pytest.mark.parametrize("boron_first", [False, True])
@pytest.mark.parametrize("pending", [True, False])
def test_device_stage_matches_oracle(dev, dt, thr, boron_first, pending):
    f, sp1, sp2 = case(boron_first, thr)
    g1, g2, gA, status = run(dev, sp1, sp2, f, dt, 5, pending=pending)
    assert status == 0
    w1, w2, wA = po.fuse(sp1, sp2, f, pc.GEOM, dt, 5)
    assert len(wA["x"]) > 0
    fc.assert_matches(g1, w1, 1e-14, "reactant")
    fc.assert_matches(g2, w2, 1e-14, "reactant")
    fc.assert_matches(gA, wA, 1e-13, "product")


def test_device_large_cell_matches_oracle(dev):
    """10 000 + 10 000 particles in one cell: the in-place canonical-order path"""
    f = pc.spec(mult=1e3)
    n1 = np.zeros((4, 5, 6), dtype=int)
    n1[2, 3, 1] = 10000
    sp1 = fc.reactants(61, n1, f["m1"], 300.0, weights="log")
    sp2 = fc.reactants(62, n1, f["m2"], 300.0, weights="log", id_offset=10 ** 6)
    g1, g2, gA, status = run(dev, sp1, sp2, f, 1e-13, 1)
    assert status == 0
    w1, w2, wA = po.fuse(sp1, sp2, f, pc.GEOM, 1e-13, 1)
    assert len(wA["x"]) > 0
    fc.assert_matches(g1, w1, 1e-14, "reactant")
    fc.assert_matches(g2, w2, 1e-14, "reactant")
    fc.assert_matches(gA, wA, 1e-13, "product")


def test_device_storage_order_independence(dev):
    f, sp1, sp2 = case()
    a1, a2, aA, _ = run(dev, sp1, sp2, f, 1e-13, 3)
    rng = np.random.default_rng(9)
    o1, o2 = rng.permutation(len(sp1["x"])), rng.permutation(len(sp2["x"]))
    b1, b2, bA, _ = run(dev, {k: v[o1] for k, v in sp1.items()}, {k: v[o2] for k, v in sp2.items()}, f, 1e-13, 3)
    assert len(aA["x"]) > 0
    for k in aA:
        assert np.array_equal(aA[k], bA[k]), k
    for a, b in ((a1, b1), (a2, b2)):
        a, b = fc.by_id(a), fc.by_id(b)
        for k in a:
            assert np.array_equal(a[k], b[k]), k


FLAG_GEOM = dict(n_cell=(16, 16, 16), prob_lo=(0.0, 0.0, 0.0), prob_hi=(16e-6, 16e-6, 16e-6), box_lo=(0, 0, 0),
                 box_hi=(15, 15, 15))


def _flag_sim(ions=True):
    import collision_cases as cc
    from warpx_b200.engine import Simulation
    g = FLAG_GEOM
    sim = Simulation(g["n_cell"], g["prob_lo"], g["prob_hi"], nox=2, sort_interval=1)
    rng = np.random.default_rng(3)
    for c in range(6):
        sim.set_field(c, rng.standard_normal(sim.data[c].shape) * (1e9 if c < 3 else 3.0))
    for k, (name, q) in enumerate((("e", -1.602176634e-19), ("i", 1.602176634e-19))[:2 if ions else 1]):
        sp = cc.particle_set(60 + k, g, 8.0, (0.05, 0.05, 0.05), w0=1e6)
        sim.add_species(name, q, 9.1093837015e-31 * (1 if k == 0 else 1836.0), sp["x"], sp["y"], sp["z"], sp["w"],
                        sp["ux"], sp["uy"], sp["uz"], ids=sp["id"])
    return sim


def test_driver_do_not_push_keeps_bits(dev):
    sim = _flag_sim()
    before = sim.species_numpy(1, sort_by_id=True)
    sim.set_species_flags("i", do_not_push=True)
    sim.Evolve(3, synchronize_last=False)
    sim.Evolve(3)
    after = sim.species_numpy(1, sort_by_id=True)
    for k in before:
        assert np.array_equal(before[k], after[k]), k


def test_driver_do_not_deposit_is_as_if_absent(dev):
    a = _flag_sim()
    a.set_species_flags(1, do_not_deposit=True)
    a.Evolve(4)
    ref = _flag_sim(ions=False)
    ref.Evolve(4)
    # the deposition adds with atomics: two runs agree to the round-off of reordered sums, not bit for bit
    for comp in range(9):
        x, y = a.field_numpy(comp)[1], ref.field_numpy(comp)[1]
        assert np.abs(x - y).max() <= 1e-12 * np.abs(y).max(), comp
    x, y = a.rho_numpy()[1], ref.rho_numpy()[1]
    assert np.abs(x - y).max() <= 1e-12 * np.abs(y).max()


def test_driver_flagged_proton_boron_run(dev):
    from warpx_b200 import abi
    from warpx_b200.engine import Simulation, species_charge_mass
    f = pc.spec()
    sp1 = fc.reactants(51, 6.0, f["m1"], 400.0)
    sp2 = fc.reactants(52, 6.0, f["m2"], 400.0, id_offset=10 ** 6)
    sim = Simulation(fc.GEOM["n_cell"], fc.GEOM["prob_lo"], fc.GEOM["prob_hi"], nox=1, solver=abi.SOLVER_NONE, dt=5e-15)
    for name, sp, st in (("p", sp1, "hydrogen1"), ("b", sp2, "boron11")):
        q, m = species_charge_mass(st)
        sim.add_species(name, q, m, sp["x"], sp["y"], sp["z"], sp["w"] * 1e25, sp["ux"], sp["uy"], sp["uz"],
                        species_type=st, ids=sp["id"])
    sim.add_empty_species("alpha", 12 * (len(sp1["x"]) + len(sp2["x"])), species_type="helium4")
    for name in ("p", "b", "alpha"):
        sim.set_species_flags(name, do_not_push=True, do_not_deposit=True)
    sim.add_fusion("p", "b", ["alpha"], multiplier=1e3, probability_threshold=1e300)
    w0 = [w for _, w in sim.particle_number()]
    sim.Evolve(1)
    nums = sim.particle_number()
    lost = w0[0] - nums[0][1]
    assert nums[2][0] > 0 and nums[2][0] % 6 == 0
    assert abs(nums[2][1] / 3.0 - lost) <= 1e-12 * lost
