"""CPU tests (-m "not gpu") of the thin kernels in warpx_b200/csrc/lwfa.cu (PEC walls, moving-window
shift, laser antenna, plasma injection, particle boundaries): the kernel BODIES and the host-side
argument builders, run over the same thread ids by tests/host_harness (no GPU in the authoring
container), against the oracle.  The same comparisons run on the device in test_gpu_lwfa.py."""
import ctypes as C
import math

import numpy as np
import pytest

from warpx_b200 import abi, workloads


@pytest.fixture(scope="module")
def hh():
    from host_harness import harness
    return harness.lib()


def _check(L, rc):
    assert rc == 0, L.pic_last_error().decode()


def _sync_periodic_duplicates(f, periodic):
    """Make the upper nodal layer of every periodic direction equal to the lower one (what
    FillBoundaryAndSync / SumBoundary maintain in a run), guards included."""
    a = f.a
    for d in range(3):
        if periodic[d] and f.desc.stag[d]:
            ax = 2 - d
            ng = f.desc.ng[d]
            n = a.shape[ax] - 2 * ng - 1
            sl_hi = [slice(None)] * 3
            sl_lo = [slice(None)] * 3
            sl_hi[ax], sl_lo[ax] = ng + n, ng
            a[tuple(sl_hi)] = a[tuple(sl_lo)]


BND = {
    "pec_z": dict(field_lo=("periodic", "periodic", "pec"), field_hi=("periodic", "periodic", "pec"), periodic=(1, 1, 0)),
    "pec_xz": dict(field_lo=("pec", "periodic", "pec"), field_hi=("pec", "periodic", "pec"), periodic=(0, 1, 0)),
    "pec_zlo_only": dict(field_lo=("periodic", "periodic", "pec"), field_hi=("periodic", "periodic", "pec"),
                         periodic=(1, 1, 0)),
}


@pytest.mark.parametrize("case", ["pec_z", "pec_xz"])
@pytest.mark.parametrize("is_E", [1, 0])
def test_pec_field_body_matches_oracle(orc, hh, case, is_E):
    n, ng, ngfg = (6, 5, 9), (4, 4, 4), (2, 2, 2)
    cfg = BND[case]
    geom = abi.make_geom(n, (0, 0, 0), (1, 1, 1), periodic=cfg["periodic"])
    bnd = abi.make_boundaries(cfg["field_lo"], cfg["field_hi"])
    rng = np.random.default_rng(11)
    box_hi = tuple(v - 1 for v in n)
    F = [orc.HostFab((0, 0, 0), box_hi, ng, abi.YEE_STAG[c + (0 if is_E else 3)]) for c in range(3)]
    for f in F:
        f.a[...] = rng.standard_normal(f.a.shape)
    G = [orc.HostFab((0, 0, 0), box_hi, ng, abi.YEE_STAG[c + (0 if is_E else 3)], data=f.a.copy()) for c, f in enumerate(F)]
    orc.lib().orc_apply_pec_field(orc.fab_array(F), is_E, C.byref(geom), C.byref(bnd), abi.int3(ngfg))
    _check(hh, hh.pic_apply_pec_field(orc.fab_array(G), is_E, C.byref(geom), C.byref(bnd), abi.int3(ngfg), None))
    for f, gq in zip(F, G):
        assert np.array_equal(f.a, gq.a)


@pytest.mark.parametrize("case,pbc", [("pec_z", None), ("pec_xz", None),
                                      ("pec_z", (("periodic", "periodic", "reflecting"), ("periodic", "periodic", "absorbing")))])
def test_pec_current_body_matches_oracle(orc, hh, case, pbc):
    n, ng = (6, 5, 9), (5, 5, 5)
    cfg = BND[case]
    geom = abi.make_geom(n, (0, 0, 0), (1, 1, 1), periodic=cfg["periodic"])
    bnd = abi.make_boundaries(cfg["field_lo"], cfg["field_hi"], *(pbc or (None, None)))
    rng = np.random.default_rng(12)
    box_hi = tuple(v - 1 for v in n)
    J = [orc.HostFab((0, 0, 0), box_hi, ng, abi.YEE_STAG[6 + c]) for c in range(3)]
    for f in J:
        f.a[...] = rng.standard_normal(f.a.shape)
    K = [orc.HostFab((0, 0, 0), box_hi, ng, abi.YEE_STAG[6 + c], data=f.a.copy()) for c, f in enumerate(J)]
    orc.lib().orc_apply_pec_current(orc.fab_array(J), C.byref(geom), C.byref(bnd))
    _check(hh, hh.pic_apply_pec_current(orc.fab_array(K), C.byref(geom), C.byref(bnd), None))
    for f, gq in zip(J, K):
        assert np.array_equal(f.a, gq.a)


@pytest.mark.parametrize("shift", [1, 2, -1])
@pytest.mark.parametrize("comp", [0, 2, 4, 6, 8])
def test_shift_body_matches_oracle(orc, hh, shift, comp):
    n, ng = (6, 5, 9), (4, 4, 5) if comp >= 6 else (4, 4, 4)
    periodic = (1, 1, 0)
    geom = abi.make_geom(n, (0, 0, 0), (1, 1, 1), periodic=periodic)
    rng = np.random.default_rng(13)
    box_hi = tuple(v - 1 for v in n)
    f = orc.HostFab((0, 0, 0), box_hi, ng, abi.YEE_STAG[comp])
    f.a[...] = rng.standard_normal(f.a.shape)
    _sync_periodic_duplicates(f, periodic)
    h = orc.HostFab((0, 0, 0), box_hi, ng, abi.YEE_STAG[comp], data=f.a.copy())
    tmp = np.empty(h.a.size)
    orc.lib().orc_shift_fab(C.byref(f.desc), C.byref(geom), shift, 2, 0.25)
    _check(hh, hh.pic_shift_fab(C.byref(h.desc), tmp.ctypes.data, C.byref(geom), shift, 2, 0.25, None))
    assert np.array_equal(f.a, h.a)


def _laser():
    la = workloads.laser_acceleration_3d()["lasers"][0]
    return abi.make_laser(la["position"], la["direction"], la["polarization"], la["wavelength"], la["e_max"],
                          la["waist"], la["duration"], la["t_peak"], la["focal_distance"])


@pytest.mark.parametrize("tilted", [False, True])
def test_laser_antenna_setup_and_push_match_oracle(orc, hh, tilted):
    wl = workloads.laser_acceleration_3d()
    dx = [(wl["prob_hi"][d] - wl["prob_lo"][d]) / wl["n_cell"][d] for d in range(3)]
    las = _laser()
    if tilted:      # propagation along x, polarisation in the y-z plane
        for d, v in enumerate((1.0, 0.0, 0.0)):
            las.nvec[d] = v
        for d, v in enumerate((0.0, 1.0, 1.0)):
            las.p_X[d] = v
        for d, v in enumerate((-10.e-6, 1.e-6, -20.e-6)):
            las.position[d] = v
    dxa = abi.dbl3(dx)
    info = (C.c_double * 4)()
    _check(hh, hh.pic_laser_antenna_info(C.byref(las), dxa, info))
    n = hh.pic_laser_antenna_particles(C.byref(las), dxa, abi.dbl3(wl["prob_lo"]), abi.dbl3(wl["prob_hi"]),
                                       None, None, None, None, 0)
    assert n > 0
    A = [np.empty(n) for _ in range(4)]
    assert hh.pic_laser_antenna_particles(C.byref(las), dxa, abi.dbl3(wl["prob_lo"]), abi.dbl3(wl["prob_hi"]),
                                          *[a.ctypes.data for a in A], n) == n
    B = [np.empty(n) for _ in range(4)]
    dp = lambda a: a.ctypes.data_as(abi.c_double_p)   # noqa: E731
    assert orc.lib().orc_antenna_particles(C.byref(las), dxa, abi.dbl3(wl["prob_lo"]), abi.dbl3(wl["prob_hi"]),
                                           *[dp(b) for b in B], n) == n
    for a, b in zip(A, B):
        assert np.array_equal(a, b)
    if not tilted:
        assert n == 2 * 32 * 32 and info[0] == 1.875e-6 and info[3] == pytest.approx(9.960961289400001e-09, rel=1e-15)
    z = np.zeros(n)
    dt = 8.687655225973464e-16
    for t in (0.0, 17 * dt, 30.e-15, 61 * dt):
        P = orc.HostParticles(x=A[0], y=A[1], z=A[2], w=A[3], ux=z, uy=z, uz=z)
        Q = P.copy()
        orc.lib().orc_antenna_push(C.byref(las), dxa, C.byref(P.soa), t, dt)
        _check(hh, hh.pic_laser_antenna_push(C.byref(las), dxa, C.byref(Q.soa), t, dt, None))
        umax = max(np.max(np.abs(P.ux)), np.max(np.abs(P.uy)), np.max(np.abs(P.uz)))
        assert umax > 0
        for k in ("ux", "uy", "uz"):
            assert np.max(np.abs(getattr(P, k) - getattr(Q, k))) <= 1e-13 * umax
        for k in ("x", "y", "z"):
            assert np.max(np.abs(getattr(P, k) - getattr(Q, k))) <= 1e-15 * dx[0]


def test_boosted_laser_antenna_matches_oracle(orc, hh):
    """warpx.gamma_boost = 10 along the propagation direction: the antenna plane moves to Z0 / gamma
    (LaserParticleContainer.cpp:183-197), the profile is evaluated at the lab time of the plane (:573-579),
    the mobility is divided by gamma (:775) and the antenna drifts with -beta c nvec (:908-915)."""
    wl = workloads.laser_acceleration_3d()
    dx = [(wl["prob_hi"][d] - wl["prob_lo"][d]) / wl["n_cell"][d] for d in range(3)]
    las = _laser()
    gamma = 10.0
    las.gamma_boost, las.beta_boost = gamma, abi.beta_of_gamma(gamma)
    lab = _laser()
    dxa = abi.dbl3(dx)
    info, info_lab = (C.c_double * 4)(), (C.c_double * 4)()
    _check(hh, hh.pic_laser_antenna_info(C.byref(las), dxa, info))
    _check(hh, hh.pic_laser_antenna_info(C.byref(lab), dxa, info_lab))
    assert info[2] == info_lab[2] / gamma and info[3] == info_lab[3]       # mobility / gamma, same weight
    lo, hi = abi.dbl3(wl["prob_lo"]), abi.dbl3(wl["prob_hi"])
    n = hh.pic_laser_antenna_particles(C.byref(las), dxa, lo, hi, None, None, None, None, 0)
    A = [np.empty(n) for _ in range(4)]
    assert hh.pic_laser_antenna_particles(C.byref(las), dxa, lo, hi, *[a.ctypes.data for a in A], n) == n
    B = [np.empty(n) for _ in range(4)]
    dp = lambda a: a.ctypes.data_as(abi.c_double_p)   # noqa: E731
    assert orc.lib().orc_antenna_particles(C.byref(las), dxa, lo, hi, *[dp(b) for b in B], n) == n
    for a, b in zip(A, B):
        assert np.array_equal(a, b)
    z0_lab = las.position[2]
    assert n == 2 * 32 * 32 and np.all(A[2] == z0_lab + (z0_lab / gamma - z0_lab))
    z = np.zeros(n)
    dt = 8.687655225973464e-16
    for t in (0.0, 170 * dt, 300.e-15, 610 * dt):
        P = orc.HostParticles(x=A[0], y=A[1], z=A[2], w=A[3], ux=z, uy=z, uz=z)
        Q = P.copy()
        orc.lib().orc_antenna_push(C.byref(las), dxa, C.byref(P.soa), t, dt)
        _check(hh, hh.pic_laser_antenna_push(C.byref(las), dxa, C.byref(Q.soa), t, dt, None))
        umax = max(np.max(np.abs(P.ux)), np.max(np.abs(P.uy)))
        assert umax > 0
        for k in ("ux", "uy", "uz"):
            assert np.max(np.abs(getattr(P, k) - getattr(Q, k))) <= 1e-13 * max(umax, np.max(np.abs(P.uz)))
        for k in ("x", "y", "z"):
            assert np.max(np.abs(getattr(P, k) - getattr(Q, k))) <= 1e-15 * dx[0]
        # the drift: z advances by -beta c dt whatever the amplitude, uz = gamma_particle * (-beta c)
        assert np.allclose(P.z - A[2], -las.beta_boost * workloads.C * dt, rtol=1e-12, atol=0)
        # the lab-frame amplitude at the same lab time gives gamma times the transverse velocity
        R = orc.HostParticles(x=A[0], y=A[1], z=A[2], w=A[3], ux=z, uy=z, uz=z)
        t_lab = t / gamma + las.beta_boost * z0_lab / workloads.C
        lab_here = _laser()
        lab_here.position[2] = A[2][0]
        orc.lib().orc_antenna_push(C.byref(lab_here), dxa, C.byref(R.soa), t_lab, dt)
        # (polarisation along y: v_lab = gamma_boost v', u_lab = v_lab / sqrt(1 - v_lab^2/c^2),
        #  u' = gamma_boost v' / sqrt(1 - v'^2/c^2))
        assert np.max(np.abs(R.uy)) > 0
        v_lab = R.uy / np.sqrt(1.0 + (R.uy / workloads.C) ** 2)
        expect = v_lab / np.sqrt(1.0 - (v_lab / gamma / workloads.C) ** 2)
        assert np.allclose(P.uy, expect, rtol=1e-9, atol=1e-9 * np.max(np.abs(R.uy)))


@pytest.mark.parametrize("t", [0.0, 3.3e-14, 2.0e-13])
@pytest.mark.parametrize("ppc", [(1, 1, 1), (2, 1, 2)])
def test_boosted_add_plasma_matches_oracle(orc, hh, ppc, t):
    """AddPlasma in a frame boosted along z (PhysicalParticleContainer.cpp:1017-1022,1209-1247): the
    plasma bounds are lab-frame values tested at z_lab = gamma (z + beta c t); density x gamma;
    uz = -gamma beta c.  The lab-frame plasma edge z_lab = 0 cuts through the slab."""
    gamma = 10.0
    beta = abi.beta_of_gamma(gamma)
    n_cell, prob_lo, prob_hi = (6, 4, 24), (-30.e-6, -20.e-6, -200.e-6), (30.e-6, 20.e-6, 40.e-6)
    geom = abi.make_geom(n_cell, prob_lo, prob_hi, periodic=(1, 1, 0))
    inj = abi.make_injector(ppc, (-20.e-6, -20.e-6, 0.0), (20.e-6, 11.e-6, 3.e-3), 2.e23, True, gamma_boost=gamma)
    assert inj.beta_boost == beta
    cap = n_cell[0] * n_cell[1] * n_cell[2] * ppc[0] * ppc[1] * ppc[2]
    s, arrs, ids = _host_soa(cap)
    n = hh.pic_add_plasma(C.byref(inj), C.byref(geom), None, None, None, abi.dbl3(prob_lo), abi.dbl3(prob_hi), C.byref(s), cap, 7, t, None)
    assert n > 0, hh.pic_last_error().decode()
    B = [np.empty(cap) for _ in range(5)]
    dp = lambda a: a.ctypes.data_as(abi.c_double_p)   # noqa: E731
    m = orc.lib().orc_add_plasma(C.byref(inj), C.byref(geom), abi.dbl3(prob_lo), abi.dbl3(prob_hi), *[dp(b) for b in B[:4]], cap, t, dp(B[4]))
    assert m == n
    for k, b in zip(("x", "y", "z", "w", "uz"), B):
        assert np.array_equal(arrs[k][:n], b[:n]), k
    assert np.all(arrs["ux"][:n] == 0.0) and np.all(arrs["uy"][:n] == 0.0)
    assert np.all(arrs["uz"][:n] == gamma * (0.0 - beta * 1.0) * workloads.C)
    dv = np.prod([(prob_hi[d] - prob_lo[d]) / n_cell[d] for d in range(3)]) / np.prod(ppc)
    assert np.allclose(arrs["w"][:n], gamma * 2.e23 * dv, rtol=1e-14)
    # every particle lies behind the lab-frame plasma edge, and the edge moves with -beta c
    z_lab = gamma * (arrs["z"][:n] + beta * workloads.C * t)
    assert z_lab.min() >= 0.0 and z_lab.max() < 3.e-3
    dz = (prob_hi[2] - prob_lo[2]) / n_cell[2]
    assert arrs["z"][:n].min() < -beta * workloads.C * t + dz
    # the lab-frame injector over the same box creates more particles (no edge inside the box at t = 0 ... )
    lab = abi.make_injector(ppc, (-20.e-6, -20.e-6, -1.0), (20.e-6, 11.e-6, 1.0), 2.e23, True)
    s2, arrs2, _ = _host_soa(cap)
    n_lab = hh.pic_add_plasma(C.byref(lab), C.byref(geom), None, None, None, abi.dbl3(prob_lo), abi.dbl3(prob_hi), C.byref(s2), cap, 0, t, None)
    assert n_lab > n and np.all(arrs2["uz"][:n_lab] == 0.0)


@pytest.mark.parametrize("galerkin", [True, False])
@pytest.mark.parametrize("cdtodz", [0.0, 0.5, 0.9 / math.sqrt(3), 0.98, 1.0])
def test_nci_godfrey_stencils_match_oracle(orc, hh, cdtodz, galerkin):
    """pic_nci_godfrey_table_index / pic_nci_godfrey_stencil and the Python helper on top of them against the
    oracle's restatement of NCIGodfreyFilter::ComputeStencils, bit for bit."""
    from test_oracle import oracle_nci_stencils, _nci_lines
    from warpx_b200.engine import nci_godfrey_stencils
    want = oracle_nci_stencils(orc, cdtodz, galerkin)
    got = nci_godfrey_stencils(hh, _nci_lines(), cdtodz, galerkin)
    assert hh.pic_nci_godfrey_table_index(cdtodz, 101) == orc.lib().orc_nci_table_index(cdtodz, 101)
    assert got[0] == want[0] and got[1] == want[1]


@pytest.mark.parametrize("comp", range(6))
def test_nci_filter_matches_oracle(orc, hh, comp):
    """pic_apply_nci_filter (applyNCIFilter -> Filter::DoFilter, slen = {1,1,5}) on random data, every staggering,
    a tile box in the middle of the array and one whose grown box reaches the zero padding: bit for bit."""
    from test_oracle import oracle_nci_stencils
    n, ng, nox = (7, 5, 11), (4, 4, 8), 3
    rng = np.random.default_rng(100 + comp)
    stz = (C.c_double * 5)(*oracle_nci_stencils(orc, 0.98)[0 if comp in (0, 1, 5) else 1])
    src = orc.HostFab((0, 0, 0), (n[0] - 1, n[1] - 1, n[2] - 1), ng, abi.YEE_STAG[comp])
    src.a[:] = rng.standard_normal(src.a.shape)
    for tile_lo, tile_hi, grow in (((0, 0, 0), (n[0] - 1, n[1] - 1, n[2] - 1), nox), ((2, 1, 3), (4, 3, 7), nox),
                                   ((0, 0, 0), (n[0] - 1, n[1] - 1, n[2] - 1), 4)):
        a = orc.HostFab((0, 0, 0), (n[0] - 1, n[1] - 1, n[2] - 1), ng, abi.YEE_STAG[comp])
        b = orc.HostFab((0, 0, 0), (n[0] - 1, n[1] - 1, n[2] - 1), ng, abi.YEE_STAG[comp])
        a.a[:] = -7.0
        b.a[:] = -7.0
        tlo = [tile_lo[d] - grow for d in range(3)]
        thi = [tile_hi[d] + grow + abi.YEE_STAG[comp][d] for d in range(3)]
        orc.lib().orc_apply_nci_filter(C.byref(src.desc), C.byref(a.desc), stz, abi.int3(tlo), abi.int3(thi))
        _check(hh, hh.pic_apply_nci_filter(C.byref(src.desc), C.byref(b.desc), stz, abi.int3(tile_lo), abi.int3(tile_hi), grow, None))
        assert np.array_equal(a.a, b.a)
        assert np.any(a.a != -7.0) and (grow == 4 or np.any(a.a == -7.0))
    # the grown box must fit the destination
    assert hh.pic_apply_nci_filter(C.byref(src.desc), C.byref(b.desc), stz, abi.int3((0, 0, 0)), abi.int3((n[0] - 1, n[1] - 1, n[2] - 1)), 9, None) != 0
    assert b"leaves the destination" in hh.pic_last_error()


def test_host_guard_cells_with_nci_match_oracle(orc):
    """engine.guard_cells with the NCI corrector: 4 more cells along z for E, B and the field gather
    (GuardCellManager.cpp:87-90,319-330), with and without the moving window, orders 1-3."""
    from warpx_b200 import engine
    from test_oracle import oracle_nci_stencils
    for nox in (1, 2, 3):
        for mw in (False, True):
            sim = orc.OracleSim((8, 8, 16), (0, 0, 0), (8e-6, 8e-6, 16e-6), nox=nox, cfl=1.0, use_filter=1, solver=abi.SOLVER_CKC)
            if mw:
                sim.set_boundaries(abi.make_boundaries(("periodic", "periodic", "pec"), ("periodic", "periodic", "pec")))
                sim.set_moving_window(2, 1.0)
            sim.set_nci_corrector(*oracle_nci_stencils(orc, 1.0))
            g = engine.guard_cells(nox, sim.L.orc_sim_dt(sim.h), [1e-6] * 3, True, (1, 1, 1), mw, True)
            og = sim.guards()
            assert g["ng_EB"] == og["ng_EB"] and g["ng_J"] == og["ng_J"] and g["ng_FG"] == og["ng_FG"], (nox, mw)
            assert g["ng_EB"][2] == nox + 4 + (nox + 4) % 2 and g["ng_FG"][2] == min((nox + 1) // 2 + 4, g["ng_EB"][2])


def _host_soa(n):
    arrs = {k: np.full(n, np.nan) for k in ("x", "y", "z", "w", "ux", "uy", "uz")}
    ids = np.zeros(n, dtype=np.uint64)
    s = abi.pic_soa()
    for k, a in arrs.items():
        setattr(s, k, a.ctypes.data)
    s.idcpu = ids.ctypes.data
    s.np = 0
    return s, arrs, ids


@pytest.mark.parametrize("ppc", [(1, 1, 1), (2, 2, 2), (1, 2, 3), (3, 1, 2)])
@pytest.mark.parametrize("slab", ["domain", "top_slab", "two_cells", "cut"])
def test_add_plasma_matches_oracle(orc, hh, ppc, slab):
    """PhysicalParticleContainer::AddPlasma on the regular lattice: positions, weights, creation order
    and count, for the start-up call (whole domain) and for continuous-injection slabs, with plasma
    bounds that cut through cells."""
    n_cell, prob_lo, prob_hi = (8, 6, 16), (-30.e-6, -20.e-6, -56.e-6 + 3.1e-7), (30.e-6, 25.e-6, 12.e-6 + 3.1e-7)
    geom = abi.make_geom(n_cell, prob_lo, prob_hi, periodic=(1, 1, 0))
    dz = (prob_hi[2] - prob_lo[2]) / n_cell[2]
    inf = math.inf
    blo, bhi = (-20.e-6, -20.e-6, 0.0), (20.e-6, 11.e-6, inf)
    if slab == "cut":
        blo, bhi = (-7.3e-6, -3.1e-6, -31.7e-6), (9.9e-6, 8.4e-6, -2.2e-6)
    inj = abi.make_injector(ppc, blo, bhi, 2.e23, True)
    plo, phi = list(prob_lo), list(prob_hi)
    if slab == "top_slab":
        plo[2] = prob_hi[2] - dz
    elif slab == "two_cells":
        plo[2], phi[2] = prob_hi[2] - 2 * dz - 1e-22, prob_hi[2] - 1e-22
    cap = n_cell[0] * n_cell[1] * n_cell[2] * ppc[0] * ppc[1] * ppc[2]
    s, arrs, ids = _host_soa(cap + 5)
    s.np = 5                                  # appended after the particles already present
    n = hh.pic_add_plasma(C.byref(inj), C.byref(geom), None, None, None, abi.dbl3(plo), abi.dbl3(phi), C.byref(s), cap + 5, 1000, 0.0, None)
    assert n >= 0, hh.pic_last_error().decode()
    B = [np.empty(cap) for _ in range(4)]
    dp = lambda a: a.ctypes.data_as(abi.c_double_p)   # noqa: E731
    m = orc.lib().orc_add_plasma(C.byref(inj), C.byref(geom), abi.dbl3(plo), abi.dbl3(phi), *[dp(b) for b in B], cap, 0.0, None)
    assert m == n and n > 0
    for k, b in zip(("x", "y", "z", "w"), B):
        assert np.array_equal(arrs[k][5:5 + n], b[:n]), k
        assert np.all(np.isnan(arrs[k][:5])) and np.all(np.isnan(arrs[k][5 + n:]))
    for k in ("ux", "uy", "uz"):
        assert np.all(arrs[k][5:5 + n] == 0.0)
    assert np.array_equal(ids[5:5 + n], 1000 + np.arange(n, dtype=np.uint64))


def test_add_plasma_capacity_and_empty(hh):
    geom = abi.make_geom((4, 4, 4), (0, 0, 0), (1, 1, 1), periodic=(1, 1, 0))
    inj = abi.make_injector((1, 1, 1), (0, 0, 0), (1, 1, 1), 1.0, True)
    s, arrs, ids = _host_soa(10)
    assert hh.pic_add_plasma(C.byref(inj), C.byref(geom), None, None, None, abi.dbl3((0, 0, 0)), abi.dbl3((1, 1, 1)), C.byref(s), 10, 0, 0.0, None) == -1
    assert b"capacity" in hh.pic_last_error()
    # a slab that lies outside the plasma bounds adds nothing
    inj2 = abi.make_injector((1, 1, 1), (0, 0, 2.0), (1, 1, 3.0), 1.0, True)
    assert hh.pic_add_plasma(C.byref(inj2), C.byref(geom), None, None, None, abi.dbl3((0, 0, 0)), abi.dbl3((1, 1, 1)), C.byref(s), 10, 0, 0.0, None) == 0


@pytest.mark.parametrize("pbc_z", [("absorbing", "absorbing"), ("reflecting", "absorbing")])
def test_particle_boundaries_match_oracle(orc, hh, pbc_z):
    """ApplyBoundaryConditions + removal: the surviving particles (matched by id) and their reflected
    positions / momenta equal the oracle's; the survivors are compacted into [0, np - n_lost)."""
    rng = np.random.default_rng(21)
    n = 5000
    geom = abi.make_geom((8, 8, 8), (-1.0, -1.0, -2.0), (1.0, 1.0, 2.0), periodic=(1, 1, 0))
    bnd = abi.make_boundaries(("periodic", "periodic", "pec"), ("periodic", "periodic", "pec"),
                              ("periodic", "periodic", pbc_z[0]), ("periodic", "periodic", pbc_z[1]))
    arr = {k: rng.uniform(-1.2, 1.2, n) for k in ("x", "y")}
    arr["z"] = rng.uniform(-2.3, 2.3, n)
    arr["z"][-40:] = 2.2           # a lost tail
    arr["z"][-80:-60] = 0.0        # survivors inside the tail
    for k in ("w", "ux", "uy", "uz"):
        arr[k] = rng.standard_normal(n)
    P = orc.HostParticles(**arr)
    keep = C.create_string_buffer(n)
    orc.lib().orc_apply_particle_boundaries(C.byref(P.soa), C.byref(geom), C.byref(bnd), keep)
    keep = np.frombuffer(keep.raw, dtype=np.int8)[:n].astype(bool)
    Q = orc.HostParticles(**arr)
    ids = np.arange(n, dtype=np.uint64)
    Q.soa.idcpu = ids.ctypes.data
    cap = 4096
    work = np.zeros(hh.pic_particles_boundary_workspace_ints(cap), dtype=np.int32)
    _check(hh, hh.pic_particles_boundary_mark(C.byref(Q.soa), C.byref(geom), C.byref(bnd), work.ctypes.data, cap, None))
    n_lost = int(work[0])
    assert n_lost == int(np.sum(~keep)) and 0 < n_lost < cap
    _check(hh, hh.pic_particles_boundary_compact(C.byref(Q.soa), work.ctypes.data, cap, n_lost, None))
    m = n - n_lost
    got = ids[:m]
    assert np.array_equal(np.sort(got), np.flatnonzero(keep).astype(np.uint64))
    order = np.argsort(got)
    for k in ("x", "y", "z", "w", "ux", "uy", "uz"):
        assert np.array_equal(getattr(Q, k)[:m][order], getattr(P, k)[keep]), k
    # list overflow is reported, not silently truncated
    work[:] = 0
    R = orc.HostParticles(**arr)              # (kept alive: its arrays back the descriptor)
    _check(hh, hh.pic_particles_boundary_mark(C.byref(R.soa), C.byref(geom), C.byref(bnd), work.ctypes.data, 8, None))
    assert int(work[0]) == n_lost
    assert hh.pic_particles_boundary_compact(C.byref(Q.soa), work.ctypes.data, 8, n_lost, None) != 0


def test_host_guard_cells_with_moving_window_match_oracle(orc):
    """engine.guard_cells (the Python mirror of guardCellManager::Init) against the oracle's, for the
    laser-acceleration deck: the moving window raises ng_EB / ng_J to at least 2."""
    from test_oracle import make_lwfa_oracle
    from warpx_b200 import engine
    wl = workloads.laser_acceleration_3d()
    osim = make_lwfa_oracle(orc, wl)
    dx = [(wl["prob_hi"][d] - wl["prob_lo"][d]) / wl["n_cell"][d] for d in range(3)]
    g = engine.guard_cells(wl["nox"], osim.dt, dx, True, (1, 1, 1), do_moving_window=True)
    og = osim.guards()
    assert (g["ng_EB"], g["ng_J"], g["ng_FG"], g["ng_FS"]) == (og["ng_EB"], og["ng_J"], og["ng_FG"], og["ng_FS"])
    assert engine.max_dt(abi.SOLVER_YEE, dx) == osim.dt
    g1 = engine.guard_cells(1, osim.dt, dx, False, (1, 1, 1), do_moving_window=True)
    assert g1["ng_EB"] == [2, 2, 2] and g1["ng_J"] == [3, 3, 3]


@pytest.mark.parametrize("order", [1, 2, 3, 4])
def test_device_shape_factors_match_reference_leaves(orc, hh, order, reference_leaves):
    """The shape-factor templates the kernels use (pic_common.cuh, __host__ __device__) against the
    reference's ShapeFactors.H compiled verbatim (digests of what oracle/_ref computed on the same positions),
    including the order-4 spline and the shifted (old-position) factors of the Esirkepov scheme."""
    from helpers import digest, shape_factor_outputs
    got = shape_factor_outputs(order, hh.pic_host_shape, hh.pic_host_shifted_shape)
    for row in got["shape"]:
        assert abs(sum(row[1:]) - 1.0) < 1e-14, row
    want = reference_leaves["shape_factors"][str(order)]
    for k in ("shape", "shifted_shape"):
        assert digest(got[k]) == want[k], k


# ---------------------------------------------------------------------------------------------
# Slab decomposition along a non-periodic z (what the C++ driver does over several ranks), emulated on
# the host: split the single-box arrays into two slabs, give each slab the neighbour planes a halo
# exchange would deliver, run the kernels per slab, compare with the single-box oracle.
# ---------------------------------------------------------------------------------------------
def _slab_of(orc, full, comp, ng, klo, khi):
    """HostFab of the cells [klo, khi] along z cut out of the single-box HostFab `full` (guards included:
    they hold the neighbour's valid data or, beyond the domain faces, the box's own guards)."""
    n = full.desc
    blo = (n.lo[0] + ng[0], n.lo[1] + ng[1], klo)
    bhi = (n.hi[0] - ng[0] - n.stag[0], n.hi[1] - ng[1] - n.stag[1], khi)
    f = orc.HostFab(blo, bhi, ng, abi.YEE_STAG[comp])
    k0 = f.desc.lo[2] - n.lo[2]
    f.a[...] = full.a[k0:k0 + f.a.shape[0]]
    return f


@pytest.mark.parametrize("comp", [0, 2, 5, 6])
@pytest.mark.parametrize("shift", [1, 2])
def test_shift_on_slabs_equals_single_box(orc, hh, comp, shift):
    n, ng = (6, 5, 24), (4, 4, 5) if comp >= 6 else (4, 4, 4)
    geom = abi.make_geom(n, (0, 0, 0), (1, 1, 1), periodic=(1, 1, 0))
    rng = np.random.default_rng(71)
    full = orc.HostFab((0, 0, 0), tuple(v - 1 for v in n), ng, abi.YEE_STAG[comp])
    full.a[...] = rng.standard_normal(full.a.shape)
    _sync_periodic_duplicates(full, (1, 1, 0))
    slabs = [_slab_of(orc, full, comp, ng, 0, 11), _slab_of(orc, full, comp, ng, 12, 23)]
    orc.lib().orc_shift_fab(C.byref(full.desc), C.byref(geom), shift, 2, 0.0)
    for f in slabs:
        tmp = np.empty(f.a.size)
        _check(hh, hh.pic_shift_fab(C.byref(f.desc), tmp.ctypes.data, C.byref(geom), shift, 2, 0.0, None))
        k0 = f.desc.lo[2] - full.desc.lo[2]
        vz = slice(ng[2], f.a.shape[0] - ng[2])               # the slab's valid planes (shared node included)
        # x / y: the valid points and the first guard layer (what FillBoundary(1) of the temporary refreshes);
        # rows at the periodic duplicate j = N: the oracle fills guards from the owner j = 0
        sl = (vz, slice(ng[1] - 1, ng[1] + n[1]), slice(ng[0] - 1, -ng[0] + 1))
        ref = full.a[k0:k0 + f.a.shape[0]]
        assert np.array_equal(f.a[sl], ref[sl]), (comp, shift)


@pytest.mark.parametrize("is_E", [1, 0])
def test_pec_on_slabs_equals_single_box(orc, hh, is_E):
    n, ng, ngfg = (6, 5, 24), (4, 4, 4), (2, 2, 2)
    geom = abi.make_geom(n, (0, 0, 0), (1, 1, 1), periodic=(1, 1, 0))
    bnd = abi.make_boundaries(("periodic", "periodic", "pec"), ("periodic", "periodic", "pec"))
    rng = np.random.default_rng(72)
    comps = [c + (0 if is_E else 3) for c in range(3)]
    full = [orc.HostFab((0, 0, 0), tuple(v - 1 for v in n), ng, abi.YEE_STAG[c]) for c in comps]
    for f in full:
        f.a[...] = rng.standard_normal(f.a.shape)
    slabs = [[_slab_of(orc, f, c, ng, klo, khi) for f, c in zip(full, comps)] for klo, khi in ((0, 11), (12, 23))]
    orc.lib().orc_apply_pec_field(orc.fab_array(full), is_E, C.byref(geom), C.byref(bnd), abi.int3(ngfg))
    for S in slabs:
        _check(hh, hh.pic_apply_pec_field(orc.fab_array(S), is_E, C.byref(geom), C.byref(bnd), abi.int3(ngfg), None))
        for f, ref in zip(S, full):
            k0 = f.desc.lo[2] - ref.desc.lo[2]
            assert np.array_equal(f.a, ref.a[k0:k0 + f.a.shape[0]])


@pytest.mark.parametrize("ppc", [(1, 1, 1), (2, 1, 2)])
def test_add_plasma_on_slabs_equals_single_box(orc, hh, ppc):
    """Initial plasma created slab by slab (tile = the rank's box, ids offset by the lower slabs' counts)
    is the single-box creation, particle for particle; a continuous-injection slab at the top of the
    domain is created by the top slab only, and the count-only call agrees with it."""
    n_cell, prob_lo, prob_hi = (8, 6, 16), (-30.e-6, -20.e-6, -56.e-6), (30.e-6, 25.e-6, 12.e-6)
    geom = abi.make_geom(n_cell, prob_lo, prob_hi, periodic=(1, 1, 0))
    dz = (prob_hi[2] - prob_lo[2]) / n_cell[2]
    inj = abi.make_injector(ppc, (-20.e-6, -20.e-6, -30.e-6), (20.e-6, 11.e-6, math.inf), 2.e23, True)
    cap = n_cell[0] * n_cell[1] * n_cell[2] * ppc[0] * ppc[1] * ppc[2]
    for plo, phi in ((list(prob_lo), list(prob_hi)), ([prob_lo[0], prob_lo[1], prob_hi[2] - dz], list(prob_hi))):
        s1, a1, id1 = _host_soa(cap)
        n1 = hh.pic_add_plasma(C.byref(inj), C.byref(geom), None, None, None, abi.dbl3(plo), abi.dbl3(phi), C.byref(s1), cap, 0, 0.0, None)
        assert n1 > 0
        assert hh.pic_add_plasma(C.byref(inj), C.byref(geom), None, None, None, abi.dbl3(plo), abi.dbl3(phi), None, 0, 0, 0.0, None) == n1
        got = {k: [] for k in ("x", "y", "z", "w")}
        ids, first = [], 0
        for klo, khi in ((0, 7), (8, 15)):
            blo, bhi = abi.int3((0, 0, klo)), abi.int3((n_cell[0] - 1, n_cell[1] - 1, khi))
            s2, a2, id2 = _host_soa(cap)
            m = hh.pic_add_plasma(C.byref(inj), C.byref(geom), None, blo, bhi, abi.dbl3(plo), abi.dbl3(phi), C.byref(s2), cap, first, 0.0, None)
            assert m >= 0
            assert hh.pic_add_plasma(C.byref(inj), C.byref(geom), None, blo, bhi, abi.dbl3(plo), abi.dbl3(phi), None, 0, 0, 0.0, None) == m
            for k in got:
                got[k].append(a2[k][:m])
            ids.append(id2[:m])
            first += m
        assert first == n1
        for k in got:
            cat = np.concatenate(got[k])
            if k == "z" and plo[2] == prob_lo[2]:
                # whole-domain creation: a slab's lattice starts from ITS overlap corner (find_overlap,
                # AddPlasmaUtilities.cpp:22-23), so z agrees with the single-box value to rounding only --
                # the reference's positions depend on the box decomposition in exactly the same way
                assert np.max(np.abs(cat - a1[k][:n1])) <= 4 * np.finfo(float).eps * abs(prob_lo[2])
            else:
                assert np.array_equal(cat, a1[k][:n1]), k
        assert np.array_equal(np.concatenate(ids), id1[:n1])


@pytest.mark.parametrize("nox", [1, 2, 3, 4])
def test_charge_deposition_and_pec_rho_match_oracle(orc, hh, nox):
    """doChargeDepositionShapeN on a nodal rho and ApplyReflectiveBoundarytoRhofield (the `rho`
    diagnostic): body + argument builder against the oracle, bit for bit on the host."""
    rng = np.random.default_rng(80 + nox)
    n, ng = (10, 8, 12), (5, 5, 5)
    prob_lo, prob_hi = (-1.0, -2.0, 0.5), (1.5, 2.0, 3.5)
    dx = [(prob_hi[d] - prob_lo[d]) / n[d] for d in range(3)]
    dinv = [1.0 / v for v in dx]
    npart = 3000
    arr = {k: rng.uniform(prob_lo[d], prob_hi[d], npart) for d, k in enumerate(("x", "y", "z"))}
    arr["w"] = rng.uniform(0.5, 2.0, npart)
    for k in ("ux", "uy", "uz"):
        arr[k] = np.zeros(npart)
    P = orc.HostParticles(**arr)
    lo = [-ng[d] for d in range(3)]
    xyzmin = [prob_lo[d] + dx[d] * lo[d] for d in range(3)]
    geom = abi.make_geom(n, prob_lo, prob_hi, periodic=(1, 1, 0))
    bnd = abi.make_boundaries(("periodic", "periodic", "pec"), ("periodic", "periodic", "pec"))
    A = orc.HostFab((0, 0, 0), tuple(v - 1 for v in n), ng, (1, 1, 1))
    B = orc.HostFab((0, 0, 0), tuple(v - 1 for v in n), ng, (1, 1, 1))
    assert orc.lib().orc_deposit_charge(C.byref(P.soa), C.byref(A.desc), abi.dbl3(dinv), abi.dbl3(xyzmin), abi.int3(lo),
                                        -1.6e-19, nox) == 0
    _check(hh, hh.pic_deposit_charge(C.byref(P.soa), 0, npart, C.byref(B.desc), abi.dbl3(dinv), abi.dbl3(xyzmin),
                                     abi.int3(lo), -1.6e-19, nox, None))
    assert np.array_equal(A.a, B.a) and np.abs(A.a).max() > 0
    # total charge: sum rho dV = q sum w
    assert A.a.sum() * dx[0] * dx[1] * dx[2] == pytest.approx(-1.6e-19 * arr["w"].sum(), rel=1e-12)
    orc.lib().orc_apply_pec_rho(C.byref(A.desc), C.byref(geom), C.byref(bnd))
    _check(hh, hh.pic_apply_pec_rho(C.byref(B.desc), C.byref(geom), C.byref(bnd), None))
    assert np.array_equal(A.a, B.a)
    kz, vy, vx = ng[2], slice(ng[1], -ng[1]), slice(ng[0], -ng[0])
    assert np.all(A.a[kz, vy, vx] == 0.0) and np.all(A.a[-kz - 1, vy, vx] == 0.0)   # the wall planes (valid x, y)
