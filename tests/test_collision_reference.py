"""CPU tests: the collision stage against what the reference's own headers compute (tests/golden/collision_reference.npz,
written by tests/golden/make_collision_reference.py from ElasticCollisionPerez.H, UpdateMomentumPerezElastic.H,
ComputeTemperature.H and ShuffleFisherYates.H compiled unchanged): the numpy restatement of tests/collision_oracle.py to
1e-14 of the |u| scale of each particle's cell (numpy's and glibc's transcendentals differ by ulps), and the kernel source through the
host build of tests/host_harness to 1e-13; then cells of more than 2048 particles, which take the kernel's
global-memory path, against the restatement."""
import numpy as np
import pytest

import collision_cases as cc
import collision_oracle as co

CASES = cc.reference_cases()


@pytest.fixture(scope="module")
def host():
    import torch
    from host_harness import harness
    return harness.host_library(), torch


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference_headers(name):
    sp1, sp2, coll, geom, dt, step, u1, u2 = CASES[name]
    r1, r2 = co.collide({k: v.copy() for k, v in sp1.items()}, None if sp2 is None else {k: v.copy() for k, v in sp2.items()},
                        coll, geom, dt, step)
    for sp, r, u in ((sp1, r1, u1), (sp2, r2, u2)):
        if sp is None:
            continue
        got = dict(sp)
        got["ux"], got["uy"], got["uz"] = r
        cc.assert_matches_reference(got, sp, u, 1e-14, geom)


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_stage_matches_reference_headers(host, name):
    L, t = host
    sp1, sp2, coll, geom, dt, step, u1, u2 = CASES[name]
    g1, g2, status = cc.run_stage(L, t, "cpu", sp1, sp2, coll, geom, dt, step)
    assert status == 0
    cc.assert_matches_reference(g1, sp1, u1, 1e-13, geom)
    if sp2 is not None:
        cc.assert_matches_reference(g2, sp2, u2, 1e-13, geom)


def test_reference_cases_reach_every_branch():
    """the fixture holds collisions in each s12 regime, a redraw, a pair with p* along z and one with identical momenta"""
    seen = set()
    for name, (sp1, sp2, coll, geom, dt, step, u1, u2) in CASES.items():
        co.LAST_S12[0] = None
        co.collide({k: v.copy() for k, v in sp1.items()}, None if sp2 is None else {k: v.copy() for k, v in sp2.items()},
                   coll, geom, dt, step)
        s = co.LAST_S12[0]
        seen |= {b for b, m in (("small", s <= 0.1), ("fit", (s > 0.1) & (s <= 3)), ("exp", (s > 3) & (s <= 6)),
                                ("iso", s > 6)) if np.any(m)}
    assert seen == {"small", "fit", "exp", "iso"}, seen
    assert {"ee_redraw", "ee_identical_and_axis", "ee_relativistic", "ee_classical", "ee_quantum", "ee_floor"} <= set(CASES)


def huge_cells():
    """cells of 2500 (species 1) and 1500 + 1000 (species 1 + 2) particles beside small ones"""
    n1 = np.full((4, 5, 6), 3)
    n1[1, 1, 1], n1[2, 2, 2] = 2500, 1500
    n2 = np.full((4, 5, 6), 2)
    n2[2, 2, 2] = 1000
    sp1 = cc.particle_set(41, cc.GEOM, n1, (0.01, 0.02, 0.01), weights="log")
    sp2 = cc.particle_set(42, cc.GEOM, n2, (0.004, 0.004, 0.004), weights="log", id_offset=10 ** 6)
    return sp1, sp2


@pytest.mark.parametrize("kind", ["ee", "ei"])
def test_host_cells_beyond_shared_memory_match_oracle(host, kind):
    L, t = host
    sp1, sp2 = huge_cells()
    coll = cc.ee_spec(L=-1.0) if kind == "ee" else cc.ei_spec(L=-1.0)
    if kind == "ee":
        sp2 = None
    g1, g2, status = cc.run_stage(L, t, "cpu", sp1, sp2, coll, cc.GEOM, 3e-15, 6)
    assert status == 0
    r1, r2 = co.collide({k: v.copy() for k, v in sp1.items()}, None if sp2 is None else {k: v.copy() for k, v in sp2.items()},
                        coll, cc.GEOM, 3e-15, 6)
    for got, sp, r in ((g1, sp1, r1), (g2, sp2, r2)):
        if sp is None:
            continue
        cc.assert_matches_reference(got, sp, r, 1e-13)
        assert np.mean(cc.by_id(got)["ux"] != cc.by_id(sp)["ux"]) > 0.5
    # without scratch such cells are reported and left alone
    g1, _, status = cc.run_stage(L, t, "cpu", sp1, sp2, coll, cc.GEOM, 3e-15, 6, scratch=False)
    assert status == 1
    big = co.cells_of(cc.by_id(sp1), cc.GEOM) == 1 + 6 * (1 + 5 * 1)
    assert np.array_equal(cc.by_id(g1)["ux"][big], cc.by_id(sp1)["ux"][big])
