"""CPU tests: the proton-boron restatement (tests/proton_boron_oracle.py) and the host build of the kernels
(csrc/fusion.cu) against what the reference's own headers compute -- tests/golden/proton_boron_reference.npz, made by
tests/golden/make_proton_boron_reference.py from ProtonBoronFusionCrossSection.H, ProtonBoronFusionInitializeMomentum.H,
SingleNuclearFusionEvent.H, TwoProductFusionUtil.H, BinaryCollisionUtils.H and ShuffleFisherYates.H, unchanged.
Identical events and spent reactants; reactant weights, alpha weights and momenta to 1e-13 of their scale; alpha
positions exact."""
import os

import numpy as np
import pytest

import proton_boron_cases as pc
import proton_boron_oracle as po

Z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "proton_boron_reference.npz"))
NAMES = sorted({k.split("/")[0] for k in Z.files} - {"xs"})


def load(name):
    p = name + "/"
    sp1 = {k[len(p) + 4:]: Z[k] for k in Z.files if k.startswith(p + "sp1_")}
    sp2 = {k[len(p) + 4:]: Z[k] for k in Z.files if k.startswith(p + "sp2_")}
    s, i = Z[p + "spec"], Z[p + "ints"]
    f = pc.spec(boron_first=bool(s[7] > s[8]), mult=s[3], thr=s[4], target=s[5], seed=int(i[0]), cidx=int(i[1]))
    assert f["m1"] == s[0] and f["m2"] == s[1] and f["mA"] == s[2]
    ref = dict(w1=Z[p + "w1"], spent1=Z[p + "spent1"], w2=Z[p + "w2"], spent2=Z[p + "spent2"], alphas=Z[p + "alphas"])
    return sp1, sp2, f, float(s[6]), int(i[2]), ref


def check(r1, r2, al, ref):
    for r, w, spent in ((r1, ref["w1"], ref["spent1"]), (r2, ref["w2"], ref["spent2"])):
        assert np.array_equal(r["id"] == -1, spent)
        assert np.abs(r["w"] - w).max() <= 1e-13 * np.abs(w).max()
    want = ref["alphas"]
    assert len(al["x"]) == len(want)
    if len(want) == 0:
        return
    for k, name in enumerate(("x", "y", "z")):
        assert np.array_equal(al[name], want[:, k]), name
    assert np.abs(al["w"] - want[:, 3]).max() <= 1e-13 * np.abs(want[:, 3]).max()
    um = np.abs(want[:, 4:7]).max()
    for k, name in enumerate(("ux", "uy", "uz")):
        err = np.abs(al[name] - want[:, 4 + k]).max() / um
        assert err <= 1e-13, (name, err)


def test_fixture_covers_the_cases():
    assert len(NAMES) >= 17
    events = {n: len(Z[n + "/alphas"]) // 6 for n in NAMES}
    assert all(events[n] > 40 for n in NAMES if not n.endswith(("rest", "midchain")))
    assert events["pb_rest"] == 0
    assert all(Z[n + "/spent1"].any() or Z[n + "/spent2"].any() for n in NAMES if n.endswith(("midchain", "floor")))
    E_keV = Z["xs/E"] / 1.602176634e-16
    for b in (400.0, 668.0, 9760.0):
        assert (E_keV < b).any() and (E_keV == b).any() and (E_keV > b).any()


def test_oracle_cross_section_matches_reference_header():
    got, want = po.cross_section(Z["xs/E"]), Z["xs/sigma"]
    assert want[0] == 0.0 and got[0] == 0.0
    assert np.all(np.abs(got - want) <= 1e-14 * np.abs(want))


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_headers(name):
    sp1, sp2, f, dt, step, ref = load(name)
    r1, r2, al = po.fuse(sp1, sp2, f, pc.GEOM, dt, step)
    check(r1, r2, al, ref)


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
    g1, g2, al, status = pc.run_stage(L, t, "cpu", sp1, sp2, f, dt, step, pending=True)
    assert status == 0
    assert np.array_equal(g1["x"], sp1["x"]) and np.array_equal(g2["x"], sp2["x"])
    check(g1, g2, al, ref)
