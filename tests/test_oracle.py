"""CPU tests (-m "not gpu"): the oracle against the reference's golden vectors and against what the
reference's own leaf headers compute (digests in tests/golden/reference_leaves.json); host logic of the
decomposition."""
import ctypes as C
import math

import numpy as np
import pytest

from warpx_b200 import abi, workloads


def _close(v, g, rtol=1e-9):
    return abs(v - g) <= rtol * abs(g) + 1e-40


def test_langmuir_golden_checksums(orc, golden):
    """Config 1 == Examples/Tests/langmuir/inputs_test_3d_langmuir_multi; WarpX's own regression
    checksums at its own tolerance (Regression/Checksum/checksum.py:219: rtol 1e-9)."""
    wl = workloads.langmuir_3d()
    sim = orc.OracleSim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=1)
    assert sim.guards() == {"ng_EB": [2, 2, 2], "ng_J": [2, 2, 2], "ng_FG": [1, 1, 1], "ng_FS": [1, 1, 1]}
    assert sim.dt == pytest.approx(1.203645750966544e-15, rel=1e-14)
    for s in wl["species"]:
        sim.add_species(s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    sim.evolve(40)
    g = golden["test_3d_langmuir_multi"]
    for c, name in enumerate(abi.COMP_NAMES):
        assert _close(sim.checksum_field(c), g["lev=0"][name]), name
    for isp, sname in enumerate(("electrons", "positrons")):
        P = sim.particles(isp)
        vals = {"particle_position_x": P["x"], "particle_position_y": P["y"], "particle_position_z": P["z"],
                "particle_momentum_x": P["ux"] * workloads.M_E, "particle_momentum_z": P["uz"] * workloads.M_E,
                "particle_weight": P["w"]}
        for key, gv in g[sname].items():
            assert _close(float(np.sum(np.abs(vals[key]))), gv), (sname, key)
    # the diagnostics of that file that lie outside the path: rho (charge deposition + SumBoundary) and
    # part_per_cell (the particle count)
    assert _close(sim.rho_checksum(), g["lev=0"]["rho"])
    assert float(sum(len(sim.particles(i)["x"]) for i in range(2))) == g["lev=0"]["part_per_cell"]
    # analytic Langmuir field, 5 % (Examples/Tests/langmuir/analysis_3d.py:77-91,124-164)
    an = wl["analytic"]
    t = 40 * sim.dt
    d, ex = sim.fab(0)
    n = wl["n_cell"][0]
    dx = (wl["prob_hi"][0] - wl["prob_lo"][0]) / n
    exv = ex[d.valid_slices()]
    x = wl["prob_lo"][0] + (np.arange(n) + 0.5) * dx           # Ex: cell-centred in x
    yz = wl["prob_lo"][1] + np.arange(n + 1) * dx              # nodal in y, z
    Z, Y, X = np.meshgrid(yz, yz, x, indexing="ij")
    k, wp, eps = an["k"], an["wp"], an["epsilon"]
    e_th = eps * (workloads.M_E * workloads.C ** 2 * k / workloads.Q_E) * np.sin(k * X) * np.cos(k * Y) \
        * np.cos(k * Z) * np.sin(wp * t)
    assert np.max(np.abs(exv - e_th)) / np.max(np.abs(e_th)) < 0.05


@pytest.mark.parametrize("pusher,name", [(abi.PUSHER_HC, "higuera_cary"), (abi.PUSHER_VAY, "vay"),
                                         (abi.PUSHER_BORIS, "boris")])
def test_particle_pusher_known_answer(orc, golden, pusher, name):
    """Examples/Tests/particle_pusher: force-free E x B drift at gamma = 20, 10 000 steps.
    |x| < 1e-3 for Vay / Higuera-Cary, documented error magnitudes (analysis.py:17-21), and the
    stored checksums for the Higuera-Cary run."""
    L = orc.lib()
    half = 2.077023075927835e+07
    dx = 2 * half / 8
    dt = 1.0 / (math.sqrt(3.0 / dx ** 2) * workloads.C)
    q = m = 1.0
    u = (C.c_double * 3)(0.0, 19.974984355438178 * workloads.C, 0.0)
    x = (C.c_double * 3)(0.0, 0.0, 0.0)
    EB = (C.c_double * 6)(-2.994174829214179e+08, 0.0, 0.0, 0.0, 0.0, 1.0)
    P = orc.HostParticles(x=[0.0], y=[0.0], z=[0.0], w=[0.0], ux=[0.0], uy=[0.0], uz=[0.0])
    geom = abi.make_geom((8, 8, 8), (-half,) * 3, (half,) * 3)
    L.orc_push_momentum(pusher, u, EB, q, m, -0.5 * dt)        # first step: u^0 -> u^{-1/2}
    for n in range(10000):
        L.orc_push_momentum(pusher, u, EB, q, m, dt)
        L.orc_update_position(x, u, dt)
        if n == 9999:
            L.orc_push_momentum(pusher, u, EB, q, m, 0.5 * dt)  # Synchronize()
        P.x[0], P.y[0], P.z[0] = x[0], x[1], x[2]
        L.orc_wrap_periodic(C.byref(P.soa), C.byref(geom))
        x[0], x[1], x[2] = P.x[0], P.y[0], P.z[0]
    expected = golden["_provenance"]["pusher_expected_error"][name]
    assert abs(x[0]) == pytest.approx(expected, rel=2e-4)
    if pusher != abi.PUSHER_BORIS:
        assert abs(x[0]) < 1e-3
    if pusher == abi.PUSHER_HC:
        g = golden["test_3d_particle_pusher"]["positron"]
        assert _close(abs(x[0]), g["particle_position_x"], 1e-9)
        assert _close(abs(x[1]), g["particle_position_y"], 1e-9)
        assert _close(abs(u[0] * m), g["particle_momentum_x"], 1e-9)
        assert _close(abs(u[1] * m), g["particle_momentum_y"], 1e-9)


def _assert_matches_reference(got, want):
    """got: {name: array}; want: {name: SHA-256} recorded with the reference's headers (helpers.digest)."""
    from helpers import digest
    assert sorted(got) == sorted(want)
    for k in sorted(got):
        assert digest(got[k]) == want[k], k


def test_restated_leaves_match_reference_headers_bitwise(orc, reference_leaves):
    """The hand-restated leaf arithmetic vs the reference's own headers compiled verbatim (digests of what
    oracle/_ref computed on the same seeded inputs, tests/golden/reference_leaves.json): identical bits on shape
    factors, pushers, stencil coefficients and dt."""
    from helpers import leaf_outputs
    A = orc.lib("restated")
    assert A.orc_leaf_name() == b"restated"
    _assert_matches_reference(leaf_outputs(orc, A), reference_leaves["leaves"])


def test_restated_stages_match_reference_headers_bitwise(orc, reference_leaves):
    """Whole stages (FDTD Yee/CKC, gather+push, deposition) with restated leaves vs the reference's digests."""
    from helpers import stage_outputs
    _assert_matches_reference(stage_outputs(orc, orc.lib("restated")), reference_leaves["stages"])


def test_decomposition_independence_of_oracle(orc):
    """One box vs a 2x2x1 brick grid (the multi-GPU oracle): same physics after 6 steps."""
    wl = workloads.uniform_plasma_3d(n_cell=(16, 16, 16), ppc=(1, 1, 2), u_th=0.05, lx=8e-6, perturbation=0.02)
    sp = wl["species"][0]
    out = []
    for nb in ((1, 1, 1), (2, 2, 1)):
        sim = orc.OracleSim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=3, nb=nb)
        sim.add_species(sp["q"], sp["m"], sp["x"], sp["y"], sp["z"], sp["w"], sp["ux"], sp["uy"], sp["uz"])
        sim.evolve(6)
        P = sim.particles(0)
        order = np.lexsort((P["z"], P["y"], P["x"]))
        out.append((sim.field_energy(), [sim.checksum_field(c) for c in range(9)], {k: v[order] for k, v in P.items()}))
    (e1, c1, p1), (e2, c2, p2) = out
    assert e1[0] == pytest.approx(e2[0], rel=1e-11) and e1[1] == pytest.approx(e2[1], rel=1e-9)
    for a, b in zip(c1, c2):
        assert a == pytest.approx(b, rel=1e-10)
    for k in p1:
        scale = np.max(np.abs(p1[k]))
        assert np.max(np.abs(p1[k] - p2[k])) <= 1e-11 * scale


def test_bilinear_filter_stencil_and_properties(orc):
    """BilinearFilter.cpp:26-62 known answers ((1,2,1)/4 per pass, first element halved), and
    Filter.cpp:92-133 applied to a delta / a constant / zero padding at the array edge."""
    import ctypes as C
    L = orc.lib()
    expect = {0: [0.5], 1: [0.25, 0.25], 2: [3 / 16, 4 / 16, 1 / 16], 3: [10 / 64, 15 / 64, 6 / 64, 1 / 64]}
    for n, ref in expect.items():
        out = (C.c_double * (n + 1))()
        L.orc_filter_stencil(n, out)
        assert list(out) == ref                           # dyadic rationals: exact
    lo, hi, ng, stag = (0, 0, 0), (7, 7, 7), (3, 3, 3), (0, 1, 1)
    src, dst = orc.HostFab(lo, hi, ng, stag), orc.HostFab(lo, hi, ng, stag)
    # delta in the middle -> outer product of the 1D kernels
    c = (7, 6, 5)
    src.a[c] = 1.0
    npass = (2, 1, 0)
    L.orc_apply_filter(C.byref(src.desc), C.byref(dst.desc), abi.int3(npass))
    k2, k1, k0 = np.array([1, 4, 6, 4, 1]) / 16, np.array([1, 2, 1]) / 4, np.array([1.0])
    want = np.zeros_like(src.a)
    want[c[0]:c[0] + 1, c[1] - 1:c[1] + 2, c[2] - 2:c[2] + 3] = k0[:, None, None] * k1[None, :, None] * k2[None, None, :]
    assert np.array_equal(dst.a, want)                    # a.shape is [k, j, i]: npass[0] acts on the last axis
    assert dst.a.sum() == 1.0
    # constant: preserved where the stencil stays inside the array, reduced at the zero-padded rim
    src.a[...] = 2.0
    L.orc_apply_filter(C.byref(src.desc), C.byref(dst.desc), abi.int3((1, 1, 1)))
    assert np.all(dst.a[1:-1, 1:-1, 1:-1] == 2.0)
    assert dst.a[0, 0, 0] == 2.0 * 0.75 ** 3 and dst.a[0, 5, 5] == 2.0 * 0.75


def test_filtered_loop_is_decomposition_independent(orc):
    """use_filter=1 (the WarpX default): J guards grow by npass (GuardCellManager.cpp:169-172), the
    filter runs per box before SumBoundaryJ; 1 box vs 2x1x2 boxes agree, and the filter matters."""
    wl = workloads.uniform_plasma_3d(n_cell=(16, 16, 16), ppc=(1, 1, 2), u_th=0.05, lx=8e-6, perturbation=0.02)
    sp = wl["species"][0]
    out = {}
    for key, nb, filt, npass in (("a", (1, 1, 1), True, (1, 1, 1)), ("b", (2, 1, 2), True, (1, 1, 1)),
                                 ("c", (1, 1, 1), False, (1, 1, 1)), ("d", (1, 1, 1), True, (2, 1, 3)),
                                 ("e", (1, 2, 2), True, (2, 1, 3))):
        sim = orc.OracleSim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=3, nb=nb, use_filter=filt, filter_npass=npass)
        g = sim.guards()
        base = 4                                             # order 3 + ceil(c dt/2 / dx)
        assert g["ng_J"] == ([base + n for n in npass] if filt else [base] * 3)
        sim.add_species(sp["q"], sp["m"], sp["x"], sp["y"], sp["z"], sp["w"], sp["ux"], sp["uy"], sp["uz"])
        sim.evolve(5)
        out[key] = [sim.checksum_field(c) for c in range(9)]
    for x, y in (("a", "b"), ("d", "e")):
        for u, v in zip(out[x], out[y]):
            assert u == pytest.approx(v, rel=1e-10)
    assert abs(out["a"][6] - out["c"][6]) > 1e-4 * abs(out["c"][6])     # jx checksum changes with the filter


def test_counter_based_momenta_are_decomposition_independent():
    full = workloads.uniform_plasma_3d(n_cell=(8, 8, 8), ppc=(2, 2, 2), lx=4e-6)["species"][0]
    part = workloads.uniform_plasma_3d(n_cell=(8, 8, 8), ppc=(2, 2, 2), lx=4e-6, box_lo=(4, 0, 4),
                                       box_hi=(7, 7, 7))["species"][0]
    key = lambda s: np.round(np.stack([s["x"], s["y"], s["z"]], 1) * 1e12).astype(np.int64)
    kf = {tuple(k): i for i, k in enumerate(key(full))}
    idx = np.array([kf[tuple(k)] for k in key(part)])
    for c in ("ux", "uy", "uz"):
        assert np.array_equal(full[c][idx], part[c])
    u = full["ux"] / workloads.C
    assert abs(np.std(u) - 0.01) < 0.001 and abs(np.mean(u)) < 0.001


# ---------------------------------------------------------------------------------------------
# Laser-wakefield additions (SURVEY.md 8f rank 3): PEC, moving window, antenna, continuous injection
# ---------------------------------------------------------------------------------------------
def make_lwfa_oracle(orc, wl, kind="restated"):
    sim = orc.OracleSim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=wl["nox"], cfl=wl["cfl"],
                        use_filter=wl["use_filter"], kind=kind, solver=wl["solver"], pusher=wl["pusher"])
    sim.set_boundaries(abi.make_boundaries(wl["field_lo"], wl["field_hi"]))
    sim.set_moving_window(wl["moving_window_dir"], wl["moving_window_v"])
    if wl.get("gamma_boost", 1.0) > 1.0:
        sim.set_boost(wl["gamma_boost"])
    if wl.get("use_fdtd_nci_corr"):
        dz = (wl["prob_hi"][2] - wl["prob_lo"][2]) / wl["n_cell"][2]
        sim.set_nci_corrector(*oracle_nci_stencils(orc, workloads.C * sim.L.orc_sim_dt(sim.h) / dz))
    for s in wl["species"]:
        sim.add_plasma(s["q"], s["m"], abi.make_injector(s["ppc"], s["bound_lo"], s["bound_hi"], s["density"],
                                                         s["do_continuous_injection"]))
    for la in wl["lasers"]:
        sim.add_laser(abi.make_laser(la["position"], la["direction"], la["polarization"], la["wavelength"],
                                     la["e_max"], la["waist"], la["duration"], la["t_peak"], la["focal_distance"]))
    return sim


def test_laser_acceleration_golden_checksums(orc, golden):
    """Examples/Physics_applications/laser_acceleration/inputs_test_3d_laser_acceleration: WarpX's own
    regression checksums (100 steps, 32x32x256, order 3, filter, PEC z, moving window, Gaussian antenna,
    continuous injection; no RNG) at WarpX's tolerance.  This is the reference-golden pin of the
    order-3 gather / Esirkepov deposition, the bilinear filter and every config-4 enabler built so far.
    Every key of the file is compared, the `rho` diagnostic included (charge deposition of the electrons
    and of the antenna, PEC image charge, filter, SumBoundary)."""
    wl = workloads.laser_acceleration_3d()
    sim = make_lwfa_oracle(orc, wl, kind="reference" if orc.have_ref() else "restated")
    assert sim.guards() == {"ng_EB": [4, 4, 4], "ng_J": [5, 5, 5], "ng_FG": [2, 2, 2], "ng_FS": [1, 1, 1]}
    info = sim.laser_info(0)
    assert info["S_X"] == 1.875e-6 and info["S_Y"] == 1.875e-6
    assert sim.L.orc_sim_laser_np(sim.h, 0) == 2 * 32 * 32
    assert sim.L.orc_sim_np(sim.h, 0) == 22 * 22 * 45
    sim.evolve(wl["max_step"])
    g = golden["test_3d_laser_acceleration"]
    for c, name in enumerate(abi.COMP_NAMES):
        assert _close(sim.checksum_field(c), g["lev=0"][name]), name
    P = sim.particles(0)
    vals = {"particle_position_x": P["x"], "particle_position_y": P["y"], "particle_position_z": P["z"],
            "particle_momentum_x": P["ux"] * workloads.M_E, "particle_momentum_y": P["uy"] * workloads.M_E,
            "particle_momentum_z": P["uz"] * workloads.M_E, "particle_weight": P["w"]}
    for key, arr in vals.items():
        assert _close(float(np.sum(np.abs(arr))), g["electrons"][key]), key
    assert _close(sim.rho_checksum(), g["lev=0"]["rho"])
    assert g["electrons"]["particle_initialenergy"] == 0.0          # ux^2 + uy^2 + uz^2 at injection: at rest
    lo, hi = wl["region_of_interest"]
    z0 = sim.z_at_injection(0)
    assert float(np.sum((z0 > lo) & (z0 < hi))) == g["electrons"]["particle_regionofinterest"]
    # the window moved 98 cells and injected 98 layers of 22 x 22 electrons
    plo, phi = sim.prob_domain()
    dz = (wl["prob_hi"][2] - wl["prob_lo"][2]) / wl["n_cell"][2]
    assert round((plo[2] - wl["prob_lo"][2]) / dz) == 98 and len(P["x"]) == 22 * 22 * (45 + 98)


def test_pec_known_answers(orc):
    """PEC::ApplyPECtoEfield / ApplyPECtoBfield semantics on a z-PEC box (WarpX_PEC.cpp:120-318):
    tangential E (normal B) vanish on the wall and are odd across it; normal E (tangential B) are even."""
    L = orc.lib()
    n, ng = (4, 4, 8), (2, 2, 2)
    geom = abi.make_geom(n, (0, 0, 0), (1, 1, 1), periodic=(1, 1, 0))
    bnd = abi.make_boundaries(("periodic", "periodic", "pec"), ("periodic", "periodic", "pec"))
    rng = np.random.default_rng(5)
    for is_E in (1, 0):
        F = [orc.HostFab((0, 0, 0), (n[0] - 1, n[1] - 1, n[2] - 1), ng, abi.YEE_STAG[c + (0 if is_E else 3)])
             for c in range(3)]
        for f in F:
            f.a[...] = rng.standard_normal(f.a.shape)
        before = [f.a.copy() for f in F]
        L.orc_apply_pec_field(orc.fab_array(F), is_E, C.byref(geom), C.byref(bnd), abi.int3(ng))
        for c, f in enumerate(F):
            a, b0 = f.a, before[c]
            nodal_z = f.desc.stag[2]
            flips = (c != 2) if is_E else (c == 2)
            sgn = -1.0 if flips else 1.0
            klo, khi = ng[2], a.shape[0] - 1 - ng[2]           # first / last valid k (array index)
            if nodal_z:
                if flips:
                    assert np.all(a[klo] == 0.0) and np.all(a[khi] == 0.0)
                else:
                    assert np.array_equal(a[klo], b0[klo])
                for gk in (1, 2):
                    assert np.array_equal(a[klo - gk], sgn * a[klo + gk])
                    assert np.array_equal(a[khi + gk], sgn * a[khi - gk])
            else:
                for gk in (1, 2):
                    assert np.array_equal(a[klo - gk], sgn * a[klo + gk - 1])
                    assert np.array_equal(a[khi + gk], sgn * a[khi - gk + 1])
            # interior untouched
            assert np.array_equal(a[klo + 1:khi], b0[klo + 1:khi])


def test_pec_current_known_answers(orc):
    """PEC::ApplyReflectiveBoundarytoJfield (WarpX_PEC.cpp:702-880) with absorbing particles: the image
    of what was deposited beyond the wall is subtracted from tangential J / added to normal J, wall
    values of the nodal (tangential) components vanish, guards hold the image current."""
    L = orc.lib()
    n, ng = (4, 4, 8), (3, 3, 3)
    geom = abi.make_geom(n, (0, 0, 0), (1, 1, 1), periodic=(1, 1, 0))
    bnd = abi.make_boundaries(("periodic", "periodic", "pec"), ("periodic", "periodic", "pec"))
    rng = np.random.default_rng(6)
    J = [orc.HostFab((0, 0, 0), (n[0] - 1, n[1] - 1, n[2] - 1), ng, abi.YEE_STAG[6 + c]) for c in range(3)]
    for f in J:
        f.a[...] = rng.standard_normal(f.a.shape)
    before = [f.a.copy() for f in J]
    L.orc_apply_pec_current(orc.fab_array(J), C.byref(geom), C.byref(bnd))
    vx = slice(ng[0], -ng[0]); vy = slice(ng[1], -ng[1])      # the reference loops over valid points only
    for c, f in enumerate(J):
        a, b0 = f.a[:, vy, vx], before[c][:, vy, vx]
        klo, khi = ng[2], f.a.shape[0] - 1 - ng[2]
        if f.desc.stag[2]:          # jx, jy: nodal in z, tangential
            assert np.all(a[klo] == 0.0) and np.all(a[khi] == 0.0)
            for gk in (1, 2, 3):
                assert np.allclose(a[klo + gk], b0[klo + gk] - b0[klo - gk], rtol=0, atol=1e-15)
                assert np.array_equal(a[klo - gk], -a[klo + gk])
                assert np.allclose(a[khi - gk], b0[khi - gk] - b0[khi + gk], rtol=0, atol=1e-15)
                assert np.array_equal(a[khi + gk], -a[khi - gk])
        else:                        # jz: cell-centred in z, normal
            for gk in (1, 2, 3):
                assert np.allclose(a[klo + gk - 1], b0[klo + gk - 1] + b0[klo - gk], rtol=0, atol=1e-15)
                assert np.array_equal(a[klo - gk], a[klo + gk - 1])
                assert np.allclose(a[khi - gk + 1], b0[khi - gk + 1] + b0[khi + gk], rtol=0, atol=1e-15)
                assert np.array_equal(a[khi + gk], a[khi - gk + 1])


def test_shift_fab_known_answers(orc):
    """WarpX::shiftMF (Utils/WarpXMovingWindow.cpp:478-604): data move down by num_shift cells, zeros
    enter at the top, the last num_shift allocated planes keep their old values."""
    L = orc.lib()
    n, ng = (4, 4, 8), (2, 2, 3)
    geom = abi.make_geom(n, (0, 0, 0), (1, 1, 1), periodic=(1, 1, 0))
    rng = np.random.default_rng(7)
    for c in (0, 2):     # Ex nodal in z, Ez cell-centred in z
        f = orc.HostFab((0, 0, 0), (n[0] - 1, n[1] - 1, n[2] - 1), ng, abi.YEE_STAG[c])
        f.a[...] = rng.standard_normal(f.a.shape)
        b0 = f.a.copy()
        L.orc_shift_fab(C.byref(f.desc), C.byref(geom), 1, 2, 0.0)
        vx = slice(ng[0], -ng[0]); vy = slice(ng[1], -ng[1])
        khi = f.a.shape[0] - 1 - ng[2]                            # last valid plane
        nk = f.a.shape[0]
        # valid x,y: planes shifted by one; zeros from beyond the old domain face
        assert np.array_equal(f.a[0:khi, vy, vx], b0[1:khi + 1, vy, vx])
        assert np.all(f.a[khi:nk - 1] == 0.0)
        assert np.array_equal(f.a[nk - 1], b0[nk - 1])
        # the first x/y guard layer was refreshed periodically before the shift (ng_mw = 1)
        # (rows below the periodic duplicate j = N: the oracle fills from the owner of a location)
        klo, vyo = ng[2], slice(ng[1], ng[1] + n[1])
        assert np.array_equal(f.a[klo - 1:khi, vyo, ng[0] - 1], b0[klo:khi + 1, vyo, ng[0] - 1 + n[0]])


def test_boosted_antenna_emits_the_lorentz_transformed_wave(orc):
    """Known answer for the boosted-frame antenna (LaserParticleContainer.cpp:183-197,573-579,775,908-915):
    a plane-wave-like antenna (huge waist) in vacuum, frame boosted by gamma = 5 along the propagation
    direction.  The forward wave must have the Doppler-shifted wavelength lambda gamma (1 + beta) and the
    amplitude e_max / (gamma (1 + beta)); the antenna itself drifts with -beta c."""
    gb = 5.0
    beta = abi.beta_of_gamma(gb)
    doppler = gb * (1 + beta)
    lam, e0 = 0.8e-6, 1.e12
    dz, nz, nx = lam * doppler / 20, 1024, 4
    zlo = -160.e-6
    sim = orc.OracleSim((nx, nx, nz), (-nx * dz / 2, -nx * dz / 2, zlo), (nx * dz / 2, nx * dz / 2, zlo + nz * dz), nox=1, cfl=1.0)
    sim.set_boundaries(abi.make_boundaries(("periodic", "periodic", "pec"), ("periodic", "periodic", "pec")))
    sim.set_boost(gb)
    sim.add_laser(abi.make_laser((0, 0, -1.e-7), (0, 0, 1), (1, 0, 0), lam, e0, 1.0, 10.e-15, 30.e-15, 0.0))
    nsteps = 600
    sim.evolve(nsteps)
    d, ex = sim.fab(0)
    line = ex[d.ng[2]:-d.ng[2], d.ng[1], d.ng[0]]
    k0 = int((0 - zlo) / dz) + 5                       # ahead of where the antenna started: the forward wave
    k = k0 + int(np.argmax(np.abs(line[k0:])))
    assert abs(abs(line[k]) * doppler / e0 - 1.0) < 0.02
    seg = line[k - 60:k + 60]
    zc = np.where(np.diff(np.sign(seg)) != 0)[0]
    assert abs(2 * np.mean(np.diff(zc)) * dz / (lam * doppler) - 1.0) < 0.02
    # emitted at lab time t_peak from the drifting antenna, then propagated at c
    t = sim.time()
    t_emit = gb * (30.e-15 - beta * (-1.e-7) / workloads.C)
    z_expect = -1.e-7 / gb - beta * workloads.C * t_emit + workloads.C * (t - t_emit)
    assert abs((zlo + k * dz) - z_expect) < 0.5 * lam * doppler
    P = sim.laser_particles(0)
    assert np.allclose(P["z"], -1.e-7 / gb - beta * workloads.C * t, rtol=1e-10)


def test_boosted_continuous_injection_continues_the_lattice(orc):
    """Known answer for AddPlasma + MoveWindow in a boosted frame (PhysicalParticleContainer.cpp:138-148,
    1017-1022,1209-1247; WarpXMovingWindow.cpp:108-133,156): the plasma, at rest in the lab, streams with
    -beta c; the injection front follows it, so the planes injected step after step continue ONE regular
    lattice; density x gamma; the lab-frame edge z_lab = 0 sits at z = -beta c t."""
    wl = workloads.laser_acceleration_boosted_3d(n_cell=(8, 8, 64), density=1.e20)   # tenuous: fields stay ~0
    wl["lasers"] = []
    for sp in wl["species"]:                           # semi-infinite plasma: z_lab >= 0
        sp["bound_hi"] = sp["bound_hi"][:2] + (float("inf"),)
    sim = make_lwfa_oracle(orc, wl)
    gb, beta = wl["gamma_boost"], abi.beta_of_gamma(wl["gamma_boost"])
    dx = [(wl["prob_hi"][d] - wl["prob_lo"][d]) / wl["n_cell"][d] for d in range(3)]
    assert sim.L.orc_sim_np(sim.h, 0) == 0            # the domain starts behind the plasma edge
    nsteps = 30
    sim.evolve(nsteps)
    t = sim.time()
    plo, phi = sim.prob_domain()
    assert round((phi[2] - wl["prob_hi"][2]) / dx[2]) == nsteps       # the window moves with c: one cell per step (CKC, cfl 1)
    for isp in (0, 1):
        P = sim.particles(isp)
        planes = np.unique(np.round(P["z"] / dx[2], 6))
        assert len(P["z"]) == len(planes) * 8 * 8 - 0 * isp and len(planes) >= 2 * nsteps - 2
        assert np.allclose(np.diff(planes), 1.0, atol=1e-5)           # one lattice across all injection seams
        assert np.allclose(P["uz"], -gb * beta * workloads.C, rtol=1e-9) and np.max(np.abs(P["ux"])) < 1e-6
        assert np.allclose(P["w"], gb * 1.e20 * dx[0] * dx[1] * dx[2], rtol=1e-13)
        z_lab = gb * (P["z"] + beta * workloads.C * t)
        assert z_lab.min() >= -1e-9 * dx[2] * gb and P["z"].min() < -beta * workloads.C * t + dx[2]
        assert P["z"].max() > phi[2] - 2 * dx[2]           # floor() of the uncovered length + the cell centre
    assert np.array_equal(sim.particles(0)["z"], sim.particles(1)["z"])
    # the deck's plasma ends at z_lab = 3 mm: a slab of 3 mm / gamma in the boosted frame
    wl = workloads.laser_acceleration_boosted_3d(n_cell=(8, 8, 64), density=1.e20)
    wl["lasers"] = []
    sim = make_lwfa_oracle(orc, wl)
    sim.evolve(nsteps)
    z_lab = gb * (sim.particles(0)["z"] + beta * workloads.C * sim.time())
    assert z_lab.min() >= -1e-9 * dx[2] * gb and 0.003 - gb * dx[2] < z_lab.max() < 0.003


def test_boosted_deck_runs_and_stays_quiet_ahead_of_the_laser(orc):
    """The boosted laser-acceleration deck (workloads.laser_acceleration_boosted_3d): 40 steps of CKC + Vay +
    order 3 + filter + NCI corrector + moving window + boosted antenna + two continuously injected species.  Sanity: finite,
    the laser field is there with the boosted amplitude scale, the neutral plasma carries the current
    of the wake only (|jz| of the two streaming species cancels to << n q beta c)."""
    wl = workloads.laser_acceleration_boosted_3d(use_fdtd_nci_corr=True)
    sim = make_lwfa_oracle(orc, wl)
    assert sim.guards() == {"ng_EB": [4, 4, 8], "ng_J": [5, 5, 5], "ng_FG": [2, 2, 6], "ng_FS": [1, 1, 1]}
    sim.evolve(40)
    gb, beta = wl["gamma_boost"], abi.beta_of_gamma(wl["gamma_boost"])
    d, ey = sim.fab(1)
    assert np.all(np.isfinite(ey))
    emax = np.max(np.abs(ey))
    assert 0.05 < emax * gb * (1 + beta) / 2.e12 < 1.5
    d, jz = sim.fab(8)
    stream = wl["species"][0]["density"] * gb * workloads.Q_E * beta * workloads.C
    assert np.max(np.abs(jz)) < 0.2 * stream
    assert sim.L.orc_sim_np(sim.h, 0) == sim.L.orc_sim_np(sim.h, 1) > 0


def _nci_lines():
    import json
    import os
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nci_godfrey_lines.json")) as f:
        return json.load(f)


def oracle_nci_stencils(orc, cdtodz, galerkin=True):
    lines = _nci_lines()
    tab_length = lines["_provenance"]["tab_length"]
    L = orc.lib()
    index = L.orc_nci_table_index(cdtodz, tab_length)
    out = []
    for which in ("Ex_Ey_Bz", "Bx_By_Ez"):
        t = lines[("galerkin_" if galerkin else "momentum_") + which]
        st = (C.c_double * 5)()
        L.orc_nci_godfrey_stencil(abi.dbl4(t[str(index)]), abi.dbl4(t[str(index + 1)]), index, tab_length, cdtodz, st)
        out.append(list(st))
    return out


def test_nci_godfrey_stencil_known_answers(orc):
    """NCIGodfreyFilter::ComputeStencils (Filter/NCIGodfreyFilter.cpp:49-139) on lines of the reference's
    tables: table index clamping, linear interpolation in c dt / dz, the 5-point combination.  Whatever the
    four coefficients, the combination has unit DC gain (s0 + 2 (s1 + s2 + s3 + s4) = 1 with the halved s0
    counted twice) -- the corrector must not change a uniform field."""
    L = orc.lib()
    assert L.orc_nci_table_index(0.0, 101) == 0 and L.orc_nci_table_index(1.0, 101) == 99      # clamped to tab_length - 2
    assert L.orc_nci_table_index(0.5, 101) == 50 and L.orc_nci_table_index(0.9 / math.sqrt(3), 101) == 52
    assert L.orc_nci_table_index(1.7, 101) == 99 and L.orc_nci_table_index(-0.1, 101) == 0
    lines = _nci_lines()
    for cdtodz in (0.0, 0.5, 0.9 / math.sqrt(3), 0.98, 1.0):
        for galerkin in (True, False):
            for st in oracle_nci_stencils(orc, cdtodz, galerkin):
                assert abs(2 * st[0] + 2 * sum(st[1:]) - 1.0) < 1e-14
    # at c dt / dz = 0 the weight of the upper line is 0: the first line of the table alone
    st = oracle_nci_stencils(orc, 0.0)[0]
    p = lines["galerkin_Ex_Ey_Bz"]["0"]
    assert st[4] == p[3] / 256 and st[3] == -(4 * p[2] + 8 * p[3]) / 256
    assert st[0] == (256 + 128 * p[0] + 96 * p[1] + 80 * p[2] + 70 * p[3]) / 256 / 2
    # c dt / dz = 1 extrapolates beyond the last pair of lines (index 99, weight 1 - 99/101), as the reference does
    st = oracle_nci_stencils(orc, 1.0)[1]
    lo, hi = lines["galerkin_Bx_By_Ez"]["99"], lines["galerkin_Bx_By_Ez"]["100"]
    w = 1.0 - 99.0 / 101.0
    assert st[4] == ((1.0 - w) * lo[3] + w * hi[3]) / 256


def test_nci_filter_known_answers(orc):
    """Filter::DoFilter with the NCI stencils over the grown tile box: a uniform field is unchanged where the
    stencil stays inside the array, a z-independent field is filtered to itself, the filter acts along z only,
    and points outside the grown tile box are not written."""
    L = orc.lib()
    n, ng, nox = (6, 5, 12), (4, 4, 8), 3
    rng = np.random.default_rng(11)
    stz = oracle_nci_stencils(orc, 0.98)[0]
    for c in (0, 2, 4):
        src = orc.HostFab((0, 0, 0), (n[0] - 1, n[1] - 1, n[2] - 1), ng, abi.YEE_STAG[c])
        dst = orc.HostFab((0, 0, 0), (n[0] - 1, n[1] - 1, n[2] - 1), ng, abi.YEE_STAG[c])
        plane = rng.standard_normal(src.a.shape[1:])
        src.a[:] = plane[None, :, :]                     # no z dependence
        dst.a[:] = np.nan
        tlo = [-nox] * 3
        thi = [n[d] - 1 + nox + abi.YEE_STAG[c][d] for d in range(3)]
        L.orc_apply_nci_filter(C.byref(src.desc), C.byref(dst.desc), (C.c_double * 5)(*stz), abi.int3(tlo), abi.int3(thi))
        o = [ng[d] - nox for d in range(3)]
        inner = dst.a[o[2]:dst.a.shape[0] - o[2], o[1]:dst.a.shape[1] - o[1], o[0]:dst.a.shape[2] - o[0]]
        assert np.all(np.isfinite(inner))
        want = np.broadcast_to(plane[None, o[1]:plane.shape[0] - o[1], o[0]:plane.shape[1] - o[0]], inner.shape)
        assert np.max(np.abs(inner - want)) <= 4e-15 * np.max(np.abs(plane))     # nox + 4 = 7 <= 8 guard cells: no zero padding reached
        mask = np.ones(dst.a.shape, dtype=bool)
        mask[o[2]:dst.a.shape[0] - o[2], o[1]:dst.a.shape[1] - o[1], o[0]:dst.a.shape[2] - o[0]] = False
        assert np.all(np.isnan(dst.a[mask]))
        # a single plane z = k0 spreads to k0 +- 4 with the stencil weights (2 x the halved centre)
        src.a[:] = 0.0
        k0 = ng[2] + 5
        src.a[k0, :, :] = 1.0
        L.orc_apply_nci_filter(C.byref(src.desc), C.byref(dst.desc), (C.c_double * 5)(*stz), abi.int3(tlo), abi.int3(thi))
        col = dst.a[:, ng[1] + 1, ng[0] + 1]
        for dk in range(-4, 5):
            w = 2 * stz[0] if dk == 0 else stz[abs(dk)]
            assert col[k0 + dk] == pytest.approx(w, rel=1e-15)
        assert col[k0 + 5] == 0.0 and col[k0 - 5] == 0.0


def nci_streaming_plasma(n=(16, 16, 32), length=20.e-6, density=1.e27, uz=-30.0, seed=1.e-5):
    """A cold neutral plasma streaming along z through a periodic box (the 3D analogue of Examples/Tests/
    nci_fdtd_stability/inputs_base_2d): the numerical Cherenkov instability grows from the tiny thermal seed
    unless the gather is corrected.  CKC at c dt = dz, Vay, order 3, Galerkin gather, bilinear filter."""
    lo = (-length / 2 * n[0] / n[2], -length / 2 * n[1] / n[2], -length / 2)
    hi = tuple(-v for v in lo)
    x, y, z = workloads.lattice_positions(n, lo, hi, (1, 1, 1))
    w = np.full_like(x, density * (length / n[2]) ** 3)
    u = workloads.philox_normal(7, 0, len(x)) * seed * workloads.C
    zero = np.zeros_like(x)
    species = [dict(name="electrons", q=-workloads.Q_E, m=workloads.M_E, x=x, y=y, z=z, w=w,
                    ux=u[:, 0].copy(), uy=u[:, 1].copy(), uz=u[:, 2] + uz * workloads.C),
               dict(name="ions", q=workloads.Q_E, m=1.67262192369e-27, x=x.copy(), y=y.copy(), z=z.copy(), w=w.copy(),
                    ux=zero.copy(), uy=zero.copy(), uz=np.full_like(x, uz * workloads.C))]
    return dict(n_cell=n, prob_lo=lo, prob_hi=hi, nox=3, cfl=1.0, use_filter=True, solver=abi.SOLVER_CKC,
                pusher=abi.PUSHER_VAY, species=species)


def test_nci_corrector_damps_the_instability_of_a_streaming_plasma(orc):
    """What the corrector is for, as a known answer (the reference's own acceptance test is of this kind:
    Examples/Tests/nci_fdtd_stability/analysis_ncicorr.py compares the field energy with a threshold 100x below
    the uncorrected run): without it the field energy of the streaming plasma grows by ten orders of magnitude in
    200 steps; with the two stencils on the right components it stays within a factor 1000 of the seed level."""
    wl = nci_streaming_plasma()
    energy = {}
    for nci in (False, True):
        sim = orc.OracleSim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=wl["nox"], cfl=wl["cfl"],
                            use_filter=wl["use_filter"], solver=wl["solver"], pusher=wl["pusher"])
        if nci:
            dz = (wl["prob_hi"][2] - wl["prob_lo"][2]) / wl["n_cell"][2]
            cdtodz = workloads.C * sim.L.orc_sim_dt(sim.h) / dz
            assert cdtodz == pytest.approx(1.0, rel=1e-12)
            sim.set_nci_corrector(*oracle_nci_stencils(orc, cdtodz))
            assert sim.guards()["ng_EB"] == [4, 4, 8] and sim.guards()["ng_FG"] == [2, 2, 6]
        for s in wl["species"]:
            sim.add_species(s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
        sim.evolve(50, synchronize_last=False)
        first = sum(sim.field_energy())
        sim.evolve(150, synchronize_last=False)
        energy[nci] = (first, sum(sim.field_energy()))
    assert energy[False][1] > 1e8 * energy[False][0]            # the instability is there ...
    assert energy[True][1] < 1e3 * energy[True][0]              # ... and the corrected gather holds it down
    assert energy[True][1] < 1e-6 * energy[False][1]


def test_particle_energy_known_answer_and_conservation(orc):
    """ParticleEnergy (ReducedDiags/ParticleEnergy.cpp:86-170): (gamma - 1) m c^2 per particle, and
    field + kinetic energy of the Langmuir deck conserved to the level the scheme allows."""
    L = orc.lib()
    g = np.array([1.0, 1.5, 20.0])
    u = np.sqrt(g * g - 1.0) * workloads.C
    P = orc.HostParticles(x=[0, 0, 0], y=[0, 0, 0], z=[0, 0, 0], w=[2.0, 3.0, 0.5], ux=[u[0], 0, 0], uy=[0, u[1], 0],
                          uz=[0, 0, u[2]])
    out = (C.c_double * 2)()
    L.orc_particle_energy(C.byref(P.soa), workloads.M_E, out)
    assert out[1] == 5.5
    assert out[0] == pytest.approx(float(np.sum(P.w * (g - 1.0)) * workloads.M_E * workloads.C ** 2), rel=1e-14)
    wl = workloads.langmuir_3d(n=16)
    sim = orc.OracleSim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=1)
    for s in wl["species"]:
        sim.add_species(s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    k0 = sum(sim.particle_energy(i)[0] for i in range(2))
    assert sim.particle_energy(0)[1] == pytest.approx(float(np.sum(wl["species"][0]["w"])), rel=1e-14)
    sim.evolve(20)
    k1 = sum(sim.particle_energy(i)[0] for i in range(2))
    e1 = sum(sim.field_energy())
    assert k1 < k0 and e1 > 0                      # the wave draws its energy from the particles ...
    assert abs((k1 + e1) - k0) <= 0.05 * k0        # ... and the total is conserved to a few per cent at 16^3


def test_order4_oracle_identity_and_leaf_agreement(orc, reference_leaves):
    """algo.particle_shape = 4 (Source/WarpX.cpp:1307-1316): the Esirkepov identity sum J dV = sum q w v
    holds for the order-4 stencil, a 6-step loop runs with the guard cells guardCellManager gives
    (ng_EB 4, ng_J 5), and the restated leaves agree with the reference's headers bit for bit (digests)."""
    wl = workloads.uniform_plasma_3d(n=12, ppc=(2, 1, 2), u_th=0.3, lx=3e-6, perturbation=0.02)
    s = wl["species"][0]
    from helpers import order4_loop_fields
    fields = order4_loop_fields(orc, "restated")
    assert all(np.isfinite(f).all() for f in fields.values()) and np.max(np.abs(fields["Ex"])) > 0
    _assert_matches_reference(fields, reference_leaves["order4_loop"])
    # stage-level identity
    L = orc.lib()
    n = wl["n_cell"]
    dx = [(wl["prob_hi"][d] - wl["prob_lo"][d]) / n[d] for d in range(3)]
    dinv = [1.0 / v for v in dx]
    dt = 0.9 / (math.sqrt(sum(1.0 / v ** 2 for v in dx)) * workloads.C)
    ng = (5, 5, 5)
    J = [orc.HostFab((0, 0, 0), tuple(v - 1 for v in n), ng, abi.YEE_STAG[c]) for c in (6, 7, 8)]
    P = orc.HostParticles(**{k: s[k] for k in orc.HostParticles.NAMES})
    lo = [-ng[d] for d in range(3)]
    xyzmin = [wl["prob_lo"][d] + dx[d] * lo[d] for d in range(3)]
    assert L.orc_deposit_esirkepov(C.byref(P.soa), 0, P.np, orc.fab_array(J), abi.dbl3(dinv), abi.dbl3(xyzmin),
                                   abi.int3(lo), s["q"], dt, -0.5 * dt, 4) == 0
    gam = np.sqrt(1.0 + (P.ux ** 2 + P.uy ** 2 + P.uz ** 2) / workloads.C ** 2)
    dV = dx[0] * dx[1] * dx[2]
    for c, u in enumerate((P.ux, P.uy, P.uz)):
        rhs = float(np.sum(s["q"] * P.w * u / gam))
        assert float(J[c].a.sum()) * dV == pytest.approx(rhs, rel=1e-10, abs=1e-12 * float(np.sum(np.abs(s["q"] * P.w * u / gam))))


def make_pec_field_oracle(orc, wl):
    sim = orc.OracleSim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=wl["nox"], cfl=wl["cfl"],
                        use_filter=wl["use_filter"])
    sim.set_boundaries(abi.make_boundaries(wl["field_lo"], wl["field_hi"]))
    dx = [(wl["prob_hi"][d] - wl["prob_lo"][d]) / wl["n_cell"][d] for d in range(3)]
    for c, fn in wl["init_fields"].items():       # AddExternalFields at start-up: valid points and guards
        d, a = sim.fab(c)
        a[...] = fn(*workloads.staggered_coordinates(d, wl["prob_lo"], dx))
    return sim


def test_pec_field_golden_checksums(orc, golden):
    """Examples/Tests/pec/inputs_test_3d_pec_field (test_3d_pec_field.json): a wave packet bouncing
    between two PEC walls for 125 steps -- the reference-golden pin of ApplyPECtoEfield / ApplyPECtoBfield
    (in the laser-acceleration deck the fields at the walls are ~0)."""
    wl = workloads.pec_field_3d()
    sim = make_pec_field_oracle(orc, wl)
    sim.evolve(wl["max_step"])
    g = golden["test_3d_pec_field"]["lev=0"]
    assert _close(sim.checksum_field(1), g["Ey"]) and _close(sim.checksum_field(3), g["Bx"])


# keys of test_3d_pec_particle.json that are round-off noise (|value| < 1e-12 of the family's scale:
# By against Bz, the z coordinates / momenta of particles that never leave z = 0)
PEC_PARTICLE_NOISE = {"By", "particle_position_z", "particle_momentum_z"}


def check_pec_particle(golden, field_checksum, particles, mass, rtol=1e-9, with_jx=False):
    """All keys of test_3d_pec_particle.json at WarpX's rtol except the noise keys; jx only for a run decomposed
    like the reference's regression run (see the test).  Returns jx / golden jx."""
    g = golden["test_3d_pec_particle"]
    for c, name in enumerate(abi.COMP_NAMES):
        if name in PEC_PARTICLE_NOISE or (name == "jx" and not with_jx):
            continue
        assert abs(field_checksum(c) - g["lev=0"][name]) <= rtol * abs(g["lev=0"][name]) + 1e-40, name
    for isp, sname in enumerate(("electron", "proton")):
        P = particles(isp)
        vals = {"particle_position_x": P["x"], "particle_position_y": P["y"], "particle_momentum_x": P["ux"] * mass,
                "particle_momentum_y": P["uy"] * mass, "particle_weight": P["w"]}
        for key, arr in vals.items():
            assert _close(float(np.sum(np.abs(arr))), g[sname][key], rtol), (sname, key)
    return field_checksum(6) / g["lev=0"]["jx"]


def test_pec_particle_golden_checksums(orc, golden):
    """Examples/Tests/pec/inputs_test_3d_pec_particle (test_3d_pec_particle.json): two heavy particles
    2 nm from a PEC wall in x, Vay pusher, order 3, bilinear filter: pins the PEC treatment of E, B and
    of the current next to a wall with particles (jy: 5e-15), and the Vay pusher inside a full loop.

    jx, the component normal to the wall, is 1e-11 of jy here and is not physics: it comes from the one particle
    whose displacement per step (1.6e-14 cells) is below the spacing of doubles at its grid coordinate
    (xp - xmin) / dx, so Esirkepov's x_old = x_new - dt v / dx moves by exactly one unit in the last place.
    That unit depends on the box decomposition: the reference's regression run uses 2 MPI ranks
    (Examples/Tests/pec/CMakeLists.txt), AMReX chops the 128-cell domain into two 64-cell boxes along x, the
    coordinate of the particle in its box is 69 instead of 133 and the unit -- hence jx -- is exactly half.
    With the same two boxes the oracle reproduces EVERY key of the file, jx to 1e-15 and even the round-off
    key By to 1e-5; with one box everything but jx agrees and jx is twice the stored value."""
    wl = workloads.pec_particle_3d()
    ratio = {}
    for nb in ((2, 1, 1), (1, 1, 1)):
        sim = orc.OracleSim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=wl["nox"], cfl=wl["cfl"],
                            use_filter=wl["use_filter"], pusher=abi.PUSHER_VAY, nb=nb)
        sim.set_boundaries(abi.make_boundaries(wl["field_lo"], wl["field_hi"]))
        for s in wl["species"]:
            sim.add_species(s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
        sim.evolve(wl["max_step"])
        ratio[nb] = check_pec_particle(golden, sim.checksum_field, sim.particles, wl["mass"], with_jx=(nb[0] == 2))
        if nb[0] == 2:
            by = golden["test_3d_pec_particle"]["lev=0"]["By"]
            assert abs(sim.checksum_field(4) - by) <= 1e-3 * by
    assert ratio[(2, 1, 1)] == pytest.approx(1.0, rel=1e-12)
    assert ratio[(1, 1, 1)] == pytest.approx(2.0, rel=1e-12)


def test_laser_injection_golden_checksums(orc, golden):
    """Examples/Tests/laser_injection/inputs_test_3d_laser_injection (test_3d_laser_injection.json): the
    Gaussian antenna radiating into vacuum, order 1, no filter, moving window, 20 steps.  jy at 1e-12; the
    radiated Ey / Bx sit 8.2e-10 below the stored values (inside WarpX's 1e-9, same on every build and
    thread count here -- the stored file was produced on another platform)."""
    wl = workloads.laser_injection_3d()
    sim = make_lwfa_oracle(orc, wl)
    sim.evolve(wl["max_step"])
    g = golden["test_3d_laser_injection"]["lev=0"]
    for c, name in enumerate(abi.COMP_NAMES):
        if name in g:
            assert _close(sim.checksum_field(c), g[name]), name


def check_particle_boundaries(golden, particles):
    g = golden["test_3d_particle_boundaries"]
    for isp, sname in enumerate(("reflecting_particles", "absorbing_particles", "periodic_particles")):
        P = particles(isp)
        vals = {"particle_position_x": P["x"], "particle_position_y": P["y"], "particle_position_z": P["z"],
                "particle_momentum_x": P["ux"] * workloads.M_E, "particle_momentum_y": P["uy"] * workloads.M_E,
                "particle_momentum_z": P["uz"] * workloads.M_E, "particle_weight": P["w"]}
        for key, arr in vals.items():
            assert _close(float(np.sum(np.abs(arr))), g[sname][key]), (sname, key)


def test_particle_boundaries_golden_checksums(orc, golden):
    """Examples/Tests/boundaries/inputs_test_3d_particle_boundaries (test_3d_particle_boundaries.json):
    reflecting x, absorbing y, periodic z for neutral particles -- the golden pin of
    ApplyBoundaryConditions + Redistribute (two of the three absorbing particles disappear)."""
    wl = workloads.particle_boundaries_3d()
    sim = orc.OracleSim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=wl["nox"], cfl=wl["cfl"], use_filter=wl["use_filter"])
    sim.set_boundaries(abi.make_boundaries(wl["field_lo"], wl["field_hi"], wl["particle_lo"], wl["particle_hi"]))
    for s in wl["species"]:
        sim.add_species(s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    sim.evolve(wl["max_step"])
    check_particle_boundaries(golden, sim.particles)
    assert sim.checksum_field(0) == 0.0 and len(sim.particles(1)["x"]) == 1


# ---------------------------------------------------------------------------------------------
# Gauss's law through the whole step (tests/helpers.py: gauss_residual).  G = div E - rho/ep0 must stay what it was at
# the start on every node.  G cannot see the gather, the push or EvolveB (continuity holds whatever velocity a particle
# gets, div curl B = 0 for any B); div B = 0 is checked beside it.
# ---------------------------------------------------------------------------------------------
GAUSS_ORACLE_TOL = 1e-12


def _oracle_gauss(orc, osim, wl, nox, use_filter=False):
    """(G, rho) of the oracle run's current state; rho from orc_deposit_charge + orc_sum_boundary."""
    from helpers import gauss_residual, oracle_rho
    s = wl["species"][0]
    E = []
    for c in range(3):
        d, a = osim.fab(c)
        E.append(a[d.valid_slices()])
    rho = oracle_rho(orc, wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox, osim.particles(0), s["q"], use_filter)
    dx = [(wl["prob_hi"][d] - wl["prob_lo"][d]) / wl["n_cell"][d] for d in range(3)]
    return gauss_residual(E, rho, dx, wl["n_cell"]), rho


@pytest.mark.parametrize("nox,solver,pusher,use_filter,u_th", [
    (1, abi.SOLVER_YEE, abi.PUSHER_BORIS, False, 0.01), (2, abi.SOLVER_YEE, abi.PUSHER_BORIS, False, 0.01),
    (3, abi.SOLVER_YEE, abi.PUSHER_BORIS, False, 0.01), (4, abi.SOLVER_YEE, abi.PUSHER_BORIS, False, 0.01),
    (3, abi.SOLVER_CKC, abi.PUSHER_VAY, False, 0.01), (3, abi.SOLVER_YEE, abi.PUSHER_BORIS, True, 0.01),
    (1, abi.SOLVER_YEE, abi.PUSHER_BORIS, False, 0.3), (3, abi.SOLVER_CKC, abi.PUSHER_VAY, True, 0.3)])
def test_oracle_keeps_gauss_law(orc, nox, solver, pusher, use_filter, u_th):
    """32^3 x 8 ppc, 60 steps: max|G^n - G^0| / max|rho^0/ep0| <= 1e-12 at every checkpoint, and div B = 0 (Yee)."""
    from helpers import div_b_ratio, gauss_drift
    wl = workloads.uniform_plasma_3d(n=32, ppc=(2, 2, 2), u_th=u_th, lx=5e-6)
    s = wl["species"][0]
    osim = orc.OracleSim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=nox, solver=solver, pusher=pusher,
                         use_filter=use_filter)
    osim.add_species(s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    G0, rho0 = _oracle_gauss(orc, osim, wl, nox, use_filter)
    dx = [(wl["prob_hi"][d] - wl["prob_lo"][d]) / wl["n_cell"][d] for d in range(3)]
    done, moved = 0, 0.0
    for step in (1, 4, 5, 20, 60):
        osim.evolve(step - done, synchronize_last=False)
        done = step
        G, rho = _oracle_gauss(orc, osim, wl, nox, use_filter)
        r = gauss_drift(G, G0, rho0)
        assert r <= GAUSS_ORACLE_TOL, (step, r)
        if solver == abi.SOLVER_YEE:      # CKC's EvolveB smooths transversely: its B is not free of the Yee divergence
            B = []
            for c in range(3, 6):
                d, a = osim.fab(c)
                B.append(a[d.valid_slices()])
            assert div_b_ratio(B, dx, wl["n_cell"]) <= 1e-9, step
        moved = max(moved, float(np.max(np.abs(rho - rho0)) / np.max(np.abs(rho0))))
    assert moved > 1e-3           # the charge did move: the check is not comparing a frozen plasma with itself


def _periodic_distance(shape, pos_cells):
    """Distance in cells (max norm, periodic) of every node of a [k, j, i] array from the point pos_cells (x, y, z)."""
    dist = np.zeros(shape)
    for ax in range(3):
        n = shape[2 - ax]
        d = np.abs(np.arange(n) - pos_cells[ax]) % n
        d = np.minimum(d, n - d)
        sh = [1, 1, 1]
        sh[2 - ax] = n
        dist = np.maximum(dist, d.reshape(sh))
    return dist


@pytest.mark.parametrize("edit", ["move", "weight"])
def test_oracle_gauss_check_sees_one_edited_particle(orc, edit):
    """Negative control: between steps 5 and 6 one particle moves by 0.37 dx (or its weight grows by half) without a
    current.  Three steps later G differs from G^0 by more than 1e-4 of max|rho^0/ep0| next to that particle, and by
    no more than the usual round-off everywhere else."""
    from helpers import gauss_drift
    nox = 3
    wl = workloads.uniform_plasma_3d(n=16, ppc=(2, 2, 2), u_th=0.01, lx=2.5e-6)
    s = wl["species"][0]
    kw = dict(nox=nox)
    osim = orc.OracleSim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], **kw)
    osim.add_species(s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    G0, rho0 = _oracle_gauss(orc, osim, wl, nox)
    osim.evolve(5, synchronize_last=False)
    assert gauss_drift(_oracle_gauss(orc, osim, wl, nox)[0], G0, rho0) <= GAUSS_ORACLE_TOL
    # continue in a new oracle run from the same fields and particles, with one particle edited
    P = osim.particles(0)
    ip = 1234
    dx = (wl["prob_hi"][0] - wl["prob_lo"][0]) / wl["n_cell"][0]
    if edit == "move":
        P["x"][ip] += 0.37 * dx
    else:
        P["w"][ip] *= 1.5
    nsim = orc.OracleSim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], **kw)
    nsim.add_species(s["q"], s["m"], *[P[k] for k in ("x", "y", "z", "w", "ux", "uy", "uz")])
    for c in range(9):
        nsim.fab(c)[1][...] = osim.fab(c)[1]
    nsim.evolve(3, synchronize_last=False)
    G, _ = _oracle_gauss(orc, nsim, wl, nox)
    scale = float(np.max(np.abs(rho0))) / workloads.EP0
    err = np.abs(G - G0) / scale
    Q = nsim.particles(0)
    at = [(Q[k][ip] - wl["prob_lo"][d]) / dx for d, k in enumerate("xyz")]
    near = _periodic_distance(G.shape, at) <= nox
    assert err[near].max() > 1e-4
    assert err[~near].max() <= GAUSS_ORACLE_TOL
