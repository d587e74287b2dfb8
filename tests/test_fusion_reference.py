"""CPU tests: the fusion restatement (tests/fusion_oracle.py) and the host build of the kernels (csrc/fusion.cu) against
what the reference's own headers compute -- tests/golden/fusion_reference.npz, made by
tests/golden/make_fusion_reference.py from SingleNuclearFusionEvent.H, BoschHaleFusionCrossSection.H,
BinaryCollisionUtils.H, TwoProductFusionUtil.H and ShuffleFisherYates.H, unchanged.  Identical events and spent
reactants; reactant weights, product weights and momenta to 1e-13 of their scale; product positions exact."""
import os

import numpy as np
import pytest

import fusion_cases as fc
import fusion_oracle as fo

Z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fusion_reference.npz"))
NAMES = sorted({k.split("/")[0] for k in Z.files})


def load(name):
    p = name + "/"
    sp1 = {k[len(p) + 4:]: Z[k] for k in Z.files if k.startswith(p + "sp1_")}
    sp2 = {k[len(p) + 4:]: Z[k] for k in Z.files if k.startswith(p + "sp2_")} or None
    s, i = Z[p + "spec"], Z[p + "ints"]
    f = dict(m1=s[0], m2=s[1], mA=s[2], mB=s[3], fusion_multiplier=s[4], fusion_probability_threshold=s[5],
             fusion_probability_target_value=s[6], q1=s[8], q2=s[9], type=int(i[0]), seed=int(i[1]),
             collision_index=int(i[2]), same_species=int(i[3]))
    ref = dict(w1=Z[p + "w1"], spent1=Z[p + "spent1"], prodA=Z[p + "prodA"], prodB=Z[p + "prodB"])
    if sp2 is not None:
        ref.update(w2=Z[p + "w2"], spent2=Z[p + "spent2"])
    return sp1, sp2, f, float(s[7]), int(i[4]), ref


def check(r1, r2, pA, pB, ref):
    """r1 / r2: reactants with w and id in the fixture's storage order; pA / pB: products in creation order"""
    for r, w, spent in ((r1, ref["w1"], ref["spent1"]), (r2, ref.get("w2"), ref.get("spent2"))):
        if r is None:
            continue
        assert np.array_equal(r["id"] == -1, spent)
        scale = np.abs(w).max()
        assert np.abs(r["w"] - w).max() <= 1e-13 * scale
    for got, want in ((pA, ref["prodA"]), (pB, ref["prodB"])):
        assert len(got["x"]) == len(want)
        if len(want) == 0:
            continue
        for k, name in enumerate(("x", "y", "z")):
            assert np.array_equal(got[name], want[:, k]), name
        assert np.abs(got["w"] - want[:, 3]).max() <= 1e-13 * np.abs(want[:, 3]).max()
        um = np.abs(want[:, 4:7]).max()
        for k, name in enumerate(("ux", "uy", "uz")):
            err = np.abs(got[name] - want[:, 4 + k]).max() / um
            assert err <= 1e-13, (name, err)


def test_fixture_covers_the_cases():
    assert len(NAMES) >= 19
    events = {n: len(Z[n + "/prodA"]) // 2 for n in NAMES}
    assert all(events[n] > 40 for n in NAMES if n.endswith(("_kev", "_mev", "_threshold", "_floor")))
    assert all(Z[n + "/spent1"].any() for n in NAMES if n.endswith("_floor") or "spent" in n)


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_headers(name):
    sp1, sp2, f, dt, step, ref = load(name)
    r1, r2, pA, pB = fo.fuse(sp1, sp2, f, fc.GEOM, dt, step)
    check(r1, r2, pA, pB, ref)


@pytest.fixture(scope="module")
def host():
    import torch
    from host_harness import harness
    return harness.host_library(), torch


@pytest.mark.parametrize("name", NAMES)
def test_host_kernels_match_reference_headers(host, name):
    """the kernels read the particles through the pending permutation, so they stay in the fixture's storage order"""
    L, t = host
    sp1, sp2, f, dt, step, ref = load(name)
    g1, g2, gA, gB, status = fc.run_stage(L, t, "cpu", sp1, sp2, f, dt, step, pending=True)
    assert status == 0
    back = []
    for g, sp in ((g1, sp1), (g2, sp2)):
        if sp is None:
            back.append(None)
            continue
        # pending=True leaves the particles in place: the buffer is in the fixture's storage order
        assert np.array_equal(g["x"], sp["x"])
        back.append(g)
    check(back[0], back[1], gA, gB, ref)
