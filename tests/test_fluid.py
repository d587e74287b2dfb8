"""CPU tests (-m "not gpu") of the cold relativistic fluid species: the numpy restatement (tests/fluid_oracle.py)
against WarpX's regression checksums of test_3d_langmuir_fluid and against known answers, and the product's fluid
kernels and C++ step driver, built for the host by tests/host_harness, against that restatement."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import fluid_cases
import fluid_oracle as fo
from warpx_b200 import abi, workloads

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def fluid_golden():
    with open(os.path.join(ROOT, "tests", "golden", "warpx_fluid_checksums.json")) as f:
        return json.load(f)["test_3d_langmuir_fluid"]["lev=0"]


def _close(v, g, rtol=1e-9):
    return abs(v - g) <= rtol * abs(g) + 1e-40


def test_langmuir_fluid_golden_checksums(orc, fluid_golden):
    """Examples/Tests/langmuir_fluids/inputs_test_3d_langmuir_fluid (64^3, two fluids, 40 steps): every checksum of
    WarpX's regression file at its rtol of 1e-9, and the analytic fields of analysis_3d.py within 5 %."""
    wl = workloads.langmuir_fluid_3d()
    run = fo.FluidRun(orc, wl["n_cell"], wl["prob_lo"], wl["prob_hi"])
    for f in wl["fluids"]:
        run.add_fluid(f["q"], f["m"], f["density"], f["momentum"])
    run.evolve(wl["max_step"])
    for c, name in enumerate(abi.COMP_NAMES):
        assert _close(run.checksum_field(c), fluid_golden[name]), name
    assert _close(run.rho_checksum(), fluid_golden["rho"])
    assert fluid_golden["part_per_cell"] == 0.0                      # no particles in the run
    # analysis_3d.py: E, J and rho against the linear Langmuir wave at the cell centres, 5 % of the amplitude
    an = wl["analytic"]
    k, wp, eps = an["k"], an["wp"], an["epsilon"]
    t = wl["max_step"] * run.dt
    n = wl["n_cell"][0]
    xc = wl["prob_lo"][0] + (np.arange(n) + 0.5) * run.dx[0]
    Z, Y, X = np.meshgrid(xc, xc, xc, indexing="ij")
    cc = {True: np.cos, False: np.sin}
    for c in range(3):
        d, a = run.fabs[c].desc, run.fabs[c].a
        got = _cell_centre(d, a)
        f = [cc[c != e](k * v) for e, v in enumerate((X, Y, Z))]
        th = eps * workloads.M_E * workloads.C ** 2 * k / workloads.Q_E * np.sin(wp * t) * f[0] * f[1] * f[2]
        assert np.max(np.abs(got - th)) / np.max(np.abs(th)) < 0.05, c
        dj, aj = run.fabs[6 + c].desc, run.fabs[6 + c].a
        jth = -workloads.EP0 * wp * eps * workloads.M_E * workloads.C ** 2 * k / workloads.Q_E \
            * np.cos(wp * t - wp * run.dt / 2) * f[0] * f[1] * f[2]
        assert np.max(np.abs(_cell_centre(dj, aj) - jth)) / np.max(np.abs(jth)) < 0.05, c
    r = run.rho()
    rth = workloads.EP0 * eps * workloads.M_E * workloads.C ** 2 * 3 * k * k / workloads.Q_E * np.sin(wp * t) \
        * np.cos(k * X) * np.cos(k * Y) * np.cos(k * Z)
    assert np.max(np.abs(_cell_centre(r.desc, r.a) - rth)) / np.max(np.abs(rth)) < 0.05


def _cell_centre(d, a):
    """ablastr::coarsen::sample::Interp to cell centres (the plotfile's values) of a component's valid box."""
    v = a[d.valid_slices()]
    for ax, dd in ((2, 0), (1, 1), (0, 2)):
        if d.stag[dd]:
            v = 0.5 * (np.take(v, range(v.shape[ax] - 1), axis=ax) + np.take(v, range(1, v.shape[ax]), axis=ax))
    return v


def _run(orc, n, density, momentum, steps, fields=None):
    run = fo.FluidRun(orc, (n,) * 3, (-fluid_cases.LX / 2,) * 3, (fluid_cases.LX / 2,) * 3)
    run.add_fluid(-workloads.Q_E, workloads.M_E, density, momentum)
    before = [a.copy() for a in run.fluids[0]["state"]]
    run.evolve(steps)
    return run, before


def test_uniform_fluid_at_rest_is_unchanged(orc):
    run, before = _run(orc, 12, lambda x, y, z: np.full(np.shape(x), 1e24), lambda x, y, z: (0.0, 0.0, 0.0), 5)
    V = run.fluids[0]["desc"].valid_slices()
    for c in range(4):
        assert np.array_equal(run.fluids[0]["state"][c][V], before[c][V])
    for c in range(9):
        assert not np.any(run.fabs[c].a)


def _unique_sum(state, desc):
    return float(np.sum(state[0][fo._owned(desc)]))


@pytest.mark.parametrize("kind", ["langmuir", "drift"])
def test_fluid_charge_is_conserved_by_the_flux_form(orc, kind):
    """Periodic faces: sum N over the unique nodes changes only by round-off (the update is a flux difference).  Not
    where the positivity limiter acts on the box's outer layer: there the reference limits a guard node's edge by its
    own density alone (MusclHancockUtils.H:279-293), so the two sides of a box face see different edge states."""
    density, momentum, _ = fluid_cases._inputs(kind, (16,) * 3)
    run = fo.FluidRun(orc, (16,) * 3, (-fluid_cases.LX / 2,) * 3, (fluid_cases.LX / 2,) * 3)
    run.add_fluid(-workloads.Q_E, workloads.M_E, density, momentum)
    fl = run.fluids[0]
    s0 = _unique_sum(fl["state"], fl["desc"])
    run.evolve(6)
    assert abs(_unique_sum(fl["state"], fl["desc"]) - s0) <= 1e-12 * s0


def test_vacuum_edge_keeps_density_non_negative_and_exercises_both_paths(orc):
    density, momentum, _ = fluid_cases._inputs("vacuum", (16,) * 3, u=0.3)
    run = fo.FluidRun(orc, (16,) * 3, (-fluid_cases.LX / 2,) * 3, (fluid_cases.LX / 2,) * 3)
    run.add_fluid(-workloads.Q_E, workloads.M_E, density, momentum)
    run.evolve(6)
    fl = run.fluids[0]
    assert np.min(fl["state"][0][fl["desc"].valid_slices()]) >= 0.0
    assert run.counters["zero_edges"] > 0 and run.counters["limited"] > 0, run.counters


# ---- the product's kernels and step driver, built for the host ---------------------------------------------------
@pytest.fixture(scope="module")
def host():
    import torch
    from host_harness import harness
    return harness.host_library(), torch


@pytest.mark.parametrize("kind,box_lo,box_hi", [("langmuir", (0, 0, 0), (11, 11, 11)),
                                                ("vacuum", (0, 0, 0), (11, 11, 11)),
                                                ("drift", (0, 0, 0), (11, 11, 11)),
                                                ("vacuum", (8, 4, 12), (15, 11, 19))])
def test_host_fluid_stages_match_oracle_bit_for_bit(host, kind, box_lo, box_hi):
    L, torch = host
    err, counters = fluid_cases.check_stages(L, torch, torch.device("cpu"), kind, (24, 24, 24), box_lo, box_hi, 0.0)
    if kind == "vacuum":
        assert counters["zero_edges"] > 0


def test_host_fluid_advection_matches_the_reference_headers(host):
    """The reference's MusclHancockUtils.H / UpdateMomentumHigueraCary.H compiled verbatim (stored outputs): the host
    build of the kernels and the numpy restatement give their bits, zero-edge and limiter paths included."""
    L, torch = host
    fluid_cases.check_reference_fixture(L, torch, torch.device("cpu"))


def test_host_fluid_loop_matches_oracle(orc):
    """The C++ driver with two fluids runs the same stages at the same place of the step as the oracle loop.  The
    fluid stages agree bit for bit; the field solver's kernels and the oracle's round a few sums in another order, so
    fields and fluids are compared to 1e-12 of their scale."""
    from fluid_cases import rel_linf
    sim, run = _host_pair(orc, 4)
    for c in range(9):
        d, a = sim.field_numpy(c)
        V = d.valid_slices()
        assert rel_linf(a[V], run.fabs[c].a[V]) <= 1e-12, c
    for i in range(2):
        d, st = sim.fluid_numpy(i)
        V = d.valid_slices()
        for c, name in enumerate(("N", "NUx", "NUy", "NUz")):
            assert rel_linf(st[name][V], run.fluids[i]["state"][c][V]) <= 1e-12, (i, name)
    _, rho = sim.rho_numpy()
    r = run.rho()
    assert rel_linf(rho[r.desc.valid_slices()], r.a[r.desc.valid_slices()]) <= 1e-12


def _host_pair(orc, steps):
    from host_harness import harness
    Sim = harness.host_simulation_class()
    wl = workloads.langmuir_fluid_3d(n=12)
    sim = Sim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=1)
    run = fo.FluidRun(orc, wl["n_cell"], wl["prob_lo"], wl["prob_hi"])
    for f in wl["fluids"]:
        sim.add_fluid_species(f["name"], f["q"], f["m"], f["density"], f["momentum"])
        run.add_fluid(f["q"], f["m"], f["density"], f["momentum"])
    sim.Evolve(steps)
    run.evolve(steps)
    return sim, run


def _fabs(desc, fill, n=4):
    arrs = [np.full(desc.shape, fill) for _ in range(n)]
    F = (abi.pic_fab * n)()
    for c in range(n):
        F[c] = desc
        F[c].p = arrs[c].ctypes.data
    return F, arrs


def test_host_fluid_refusals_leave_the_run_untouched():
    from host_harness import harness
    from warpx_b200 import diagnostics
    Sim = harness.host_simulation_class()
    wl = workloads.langmuir_fluid_3d(n=8)
    f = wl["fluids"][0]
    args = (f["name"], f["q"], f["m"], f["density"], f["momentum"])
    dom = (wl["n_cell"], wl["prob_lo"], wl["prob_hi"])
    bnd = abi.make_boundaries(("periodic", "periodic", "pec"), ("periodic", "periodic", "pec"))
    refused = [(Sim(*dom, nox=1, boundaries=bnd), "periodic"),
               (Sim(*dom, nox=1, boundaries=bnd, moving_window=(2, 1.0)), "periodic|moving"),
               (Sim(*dom, nox=1, gamma_boost=2.0), "boost")]
    withp = Sim(*dom, nox=1)
    p = workloads.langmuir_3d(n=8)["species"][0]
    withp.add_species(p["name"], p["q"], p["m"], p["x"], p["y"], p["z"], p["w"], p["ux"], p["uy"], p["uz"])
    refused.append((withp, "particle species"))
    for sim, msg in refused:
        with pytest.raises(NotImplementedError, match=msg):
            sim.add_fluid_species(*args)
        assert sim.fluids == []
    sim = Sim(*dom, nox=1)
    sim.add_fluid_species(*args)
    with pytest.raises(NotImplementedError, match="fluid"):
        sim.add_species(p["name"], p["q"], p["m"], p["x"], p["y"], p["z"], p["w"], p["ux"], p["uy"], p["uz"])
    assert sim.species == []
    with pytest.raises(NotImplementedError, match="fluid"):
        diagnostics.write_checkpoint(sim, "/nonexistent/chk")
    # the library refuses bad arguments before it changes anything
    L = harness.host_library()
    good = abi.make_fab(None, (0, 0, 0), (7, 7, 7), (2, 2, 2), (1, 1, 1))
    U, _ = _fabs(good, 1.0)
    thin = abi.make_fab(None, (0, 0, 0), (7, 7, 7), (1, 1, 1), (1, 1, 1))
    Ut, _ = _fabs(thin, 1.0)
    Uo, out = _fabs(good, 7.0)
    assert L.pic_fluid_advect(Ut, Uo, abi.dbl3((1.0, 1.0, 1.0)), 1e-15, None, None) != 0     # 1 guard node < 2
    assert L.pic_fluid_advect(U, U, abi.dbl3((1.0, 1.0, 1.0)), 1e-15, None, None) != 0       # in place
    assert all(np.all(o == 7.0) for o in out)
    # E / B without the guard the interpolation reads; J on another box
    E, eb = _fabs(abi.make_fab(None, (0, 0, 0), (7, 7, 7), (0, 0, 0), (0, 1, 1)), 3.0, 3)
    for c in range(3):
        E[c].stag[0], E[c].stag[1], E[c].stag[2] = abi.YEE_STAG[c]
    B, _ = _fabs(abi.make_fab(None, (0, 0, 0), (7, 7, 7), (0, 0, 0), (1, 0, 0)), 3.0, 3)
    for c in range(3):
        B[c].stag[0], B[c].stag[1], B[c].stag[2] = abi.YEE_STAG[3 + c]
    Ug, ug = _fabs(good, 1.0)
    assert L.pic_fluid_gather_push(Ug, E, B, -1.0, 1.0, 1e-15, None) != 0
    assert all(np.all(a == 1.0) for a in ug)
    J = (abi.pic_fab * 3)()
    jarrs = []
    for c in range(3):
        J[c] = abi.make_fab(None, (1, 0, 0), (8, 7, 7), (2, 2, 2), abi.YEE_STAG[6 + c])
        jarrs.append(np.full(J[c].shape, 5.0))
        J[c].p = jarrs[c].ctypes.data
    assert L.pic_fluid_deposit_current(Ug, J, -1.0, None) != 0
    assert all(np.all(a == 5.0) for a in jarrs)
    rd = abi.make_fab(None, (0, 0, 0), (8, 7, 7), (2, 2, 2), (1, 1, 1))
    rho = np.full(rd.shape, 5.0)
    rd.p = rho.ctypes.data
    assert L.pic_fluid_deposit_charge(C.byref(Ug[0]), C.byref(rd), -1.0, None) != 0
    assert np.all(rho == 5.0)
    # the C++ driver: a state not on its box, and fluids after particle species
    native = Sim(*dom, nox=1)
    assert L.pic_engine_add_fluid_species(native.native, -1.0, 1.0, Ut, Uo) != 0
    assert L.pic_engine_fluid_state(native.native, 0) == -1
