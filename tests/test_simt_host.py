"""CPU tests (-m "not gpu"): the warp-level deposition kernels of warpx_b200/csrc/deposit_runs.cu run
UNMODIFIED under the SIMT emulator of tests/host_harness/simt_host.h (every CUDA thread a cooperative
fiber, warp collectives as lock-step exchanges) against the oracle.  Covers the default register-run
kernel and the three experimental variants of pic_set_deposit_mode (two lines per lane, per-slot
reductions), cell-sorted, jittered (stale order: lone-particle and flush paths) and shuffled particles,
and the general kernel for the particles that changed cell.  The emulator checks indexing, lane roles and
arithmetic -- not memory-model races or speed."""
import ctypes as C

import numpy as np
import pytest

import particle_sets as ps
from helpers import lower_corner, rel_linf
from particle_sets import host_bins
from warpx_b200 import abi, workloads


@pytest.fixture(scope="module")
def simt():
    from host_harness import harness
    return harness.simt()


CASES = [(3, 0.02, "sorted"), (3, 0.5, "sorted"), (3, 0.02, "jitter"), (3, 0.3, "shuffled"), (1, 0.02, "jitter"),
         (2, 0.3, "sorted")]


@pytest.mark.parametrize("variant", [0, 1, 2, 3, 4, 6])
@pytest.mark.parametrize("nox,u_th,order", CASES)
def test_deposit_runs_kernels_under_simt_emulation(orc, simt, variant, nox, u_th, order):
    if variant and (nox, order) not in ((3, "sorted"), (3, "jitter"), (1, "jitter"), (2, "sorted")):
        pytest.skip("the experimental variants are covered on a subset")
    if variant >= 4 and nox != 3:
        pytest.skip("four lines per lane: order 3 only")
    n, lx = (8, 6, 6), (4e-6, 3e-6, 3e-6)
    wl = workloads.uniform_plasma_3d(n_cell=n, ppc=(2, 2, 2), u_th=u_th, lx=lx, seed=3)
    s = wl["species"][0]
    prob_lo = wl["prob_lo"]
    dx = [(wl["prob_hi"][d] - prob_lo[d]) / n[d] for d in range(3)]
    dinv = [1.0 / v for v in dx]
    dt = 0.95 / (np.sqrt(sum(1.0 / v ** 2 for v in dx)) * workloads.C)
    rng = np.random.default_rng(5)
    idx = np.arange(len(s["x"]))
    if order == "shuffled":
        rng.shuffle(idx)
    if order == "jitter":      # moved inside +-0.6 cell after the (cell-sorted) lattice order was fixed
        for d, k in enumerate("xyz"):
            s[k] = s[k] + rng.uniform(-0.6, 0.6, len(idx)) * dx[d]
    P = orc.HostParticles(**{k: s[k][idx] for k in orc.HostParticles.NAMES})
    ngJ = (nox + 2,) * 3
    xyzmin, lo = lower_corner(prob_lo, dx, (0, 0, 0), ngJ)
    box_hi = tuple(v - 1 for v in n)
    J = [orc.HostFab((0, 0, 0), box_hi, ngJ, abi.YEE_STAG[c]) for c in (6, 7, 8)]
    K = [orc.HostFab((0, 0, 0), box_hi, ngJ, abi.YEE_STAG[c]) for c in (6, 7, 8)]
    assert orc.lib().orc_deposit_esirkepov(C.byref(P.soa), 0, P.np, orc.fab_array(J), abi.dbl3(dinv), abi.dbl3(xyzmin),
                                           abi.int3(lo), s["q"], dt, -0.5 * dt, nox) == 0
    assert simt.simt_deposit_runs(C.byref(P.soa), 0, P.np, orc.fab_array(K), abi.dbl3(dinv), abi.dbl3(xyzmin),
                                  abi.int3(lo), s["q"], dt, -0.5 * dt, nox, variant) == 0
    for c in range(3):
        assert rel_linf(K[c].a, J[c].a) <= 1e-13, "j" + "xyz"[c]


# ---------------------------------------------------------------------------------------------------------
# the supercell gather + push kernels of warpx_b200/csrc/gather_push_tile.cu under the same emulator
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
@pytest.mark.parametrize("nox,galerkin,tile,kind", [(3, 1, (8, 8, 8), "sorted"), (3, 1, (8, 8, 8), "moved"),
                                                    (3, 1, (4, 4, 4), "moved"), (1, 1, (8, 8, 8), "moved"),
                                                    (2, 1, (4, 4, 4), "sorted"), (3, 0, (4, 4, 4), "sorted"),
                                                    (3, 1, (8, 8, 8), "odd")])
def test_gather_push_tile_kernels_under_simt_emulation(orc, simt, mode, nox, galerkin, tile, kind):
    """gather_push_tile_kernel (mode 0) and gather_push_pair_kernel (modes 1, 2: two particles of a cell per lane)
    against the oracle's gather + push: cell-sorted particles, particles that moved up to 0.9 cell since the sort
    (stray lists, lone survivors of a pair), cells with odd counts, the fixed 8x8x8 and the run-time supercell.
    Orders / gathers whose stencils do not coincide inside a cell fall back to the default kernel in modes 1, 2."""
    if mode in (2, 3) and kind not in ("sorted", "odd"):
        pytest.skip("the wide / 192-thread instances differ only in their launch shape")
    n = (16, 8, 8) if tile == (8, 8, 8) else (8, 8, 4)
    lx = tuple(0.5e-6 * v for v in n)
    wl = workloads.uniform_plasma_3d(n_cell=n, ppc=(2, 1, 2) if kind != "odd" else (1, 1, 1), u_th=0.1, lx=lx, seed=11)
    sp = wl["species"][0]
    prob_lo = wl["prob_lo"]
    dx = [(wl["prob_hi"][d] - prob_lo[d]) / n[d] for d in range(3)]
    dinv = [1.0 / v for v in dx]
    rng = np.random.default_rng(17)
    arr = {k: sp[k].copy() for k in orc.HostParticles.NAMES}
    if kind == "odd":            # 1, 2 or 3 particles per cell
        extra = rng.integers(0, 3, len(arr["x"]))
        for k in arr:
            arr[k] = np.repeat(arr[k], 1 + extra)
        for d, k in enumerate("xyz"):
            arr[k] = arr[k] + rng.uniform(-0.49, 0.49, len(arr[k])) * dx[d]
    order, cell_start = host_bins(arr["x"], arr["y"], arr["z"], prob_lo, dx, n, tile)
    arr = {k: np.ascontiguousarray(v[order]) for k, v in arr.items()}
    if kind == "moved":          # after the sort: bins are stale but must stay correct
        for d, k in enumerate("xyz"):
            arr[k] = arr[k] + rng.uniform(-0.9, 0.9, len(arr[k])) * dx[d]
    P = orc.HostParticles(**arr)
    Q = P.copy()
    ngEB = (4, 4, 4)
    box_hi = tuple(v - 1 for v in n)
    xyzmin, lo = lower_corner(prob_lo, dx, (0, 0, 0), ngEB)
    from helpers import random_fields
    F = random_fields(orc, (0, 0, 0), box_hi, ngEB, 5, comps=range(6), scale=[1e10] * 3 + [30.0] * 3)
    bins = abi.pic_bins()
    bins.cell_start = cell_start.ctypes.data
    for d in range(3):
        bins.box_lo[d], bins.box_hi[d], bins.tile[d] = 0, box_hi[d], tile[d]
    bins.np_binned = P.np
    dt = 0.9 * dx[0] / workloads.C
    for push_position in (1, 0):
        assert simt.simt_gather_push(C.byref(Q.soa), orc.fab_array(F[0:3]), orc.fab_array(F[3:6]), abi.dbl3(dinv),
                                     abi.dbl3(xyzmin), abi.int3(lo), sp["q"], sp["m"], dt, nox, galerkin,
                                     abi.PUSHER_BORIS, push_position, C.byref(bins), mode) == 0
        orc.lib().orc_gather_push(C.byref(P.soa), 0, P.np, orc.fab_array(F[0:3]), orc.fab_array(F[3:6]), abi.dbl3(dinv),
                                  abi.dbl3(xyzmin), abi.int3(lo), sp["q"], sp["m"], dt, nox, galerkin, abi.PUSHER_BORIS,
                                  push_position)
    for k in ("x", "y", "z"):
        assert np.max(np.abs(getattr(Q, k) - getattr(P, k))) <= 1e-13 * lx[0], k
    for k in ("ux", "uy", "uz"):
        assert rel_linf(getattr(Q, k), getattr(P, k)) <= 1e-13, k


@pytest.mark.parametrize("nox", [1, 2, 3, 4])
def test_order_agnostic_kernels_under_simt_emulation(orc, nox):
    """deposit_global<N> and gather_push_global<N, G> (one thread per particle; the path of particle shape order 4
    and of callers without cell bins) against the oracle, unsorted thermal particles, all three pushers -- through
    the C ABI of the host library (pic_deposit_esirkepov / pic_gather_push with bins = NULL)."""
    from host_harness import harness
    hl = harness.host_library()
    n, lx = (8, 6, 6), (4e-6, 3e-6, 3e-6)
    wl = workloads.uniform_plasma_3d(n_cell=n, ppc=(2, 1, 2), u_th=0.4, lx=lx, seed=9)
    s = wl["species"][0]
    prob_lo = wl["prob_lo"]
    dx = [(wl["prob_hi"][d] - prob_lo[d]) / n[d] for d in range(3)]
    dinv = [1.0 / v for v in dx]
    dt = 0.95 / (np.sqrt(sum(1.0 / v ** 2 for v in dx)) * workloads.C)
    box_hi = tuple(v - 1 for v in n)
    # current deposition
    P = orc.HostParticles(**{k: s[k] for k in orc.HostParticles.NAMES})
    ngJ = (nox + 2,) * 3
    xyzmin, lo = lower_corner(prob_lo, dx, (0, 0, 0), ngJ)
    J = [orc.HostFab((0, 0, 0), box_hi, ngJ, abi.YEE_STAG[c]) for c in (6, 7, 8)]
    K = [orc.HostFab((0, 0, 0), box_hi, ngJ, abi.YEE_STAG[c]) for c in (6, 7, 8)]
    assert orc.lib().orc_deposit_esirkepov(C.byref(P.soa), 0, P.np, orc.fab_array(J), abi.dbl3(dinv), abi.dbl3(xyzmin),
                                           abi.int3(lo), s["q"], dt, -0.5 * dt, nox) == 0
    assert hl.pic_deposit_esirkepov(C.byref(P.soa), 0, P.np, orc.fab_array(K), abi.dbl3(dinv), abi.dbl3(xyzmin), abi.int3(lo),
                                    s["q"], dt, -0.5 * dt, nox, None, None) == 0, hl.pic_last_error()
    for c in range(3):
        assert rel_linf(K[c].a, J[c].a) <= 1e-13, "j" + "xyz"[c]
    # gather + push
    from helpers import random_fields
    ngEB = (4, 4, 4)
    xyzmin, lo = lower_corner(prob_lo, dx, (0, 0, 0), ngEB)
    F = random_fields(orc, (0, 0, 0), box_hi, ngEB, 5, comps=range(6), scale=[1e10] * 3 + [30.0] * 3)
    for galerkin in (1, 0):
        for pusher in (abi.PUSHER_BORIS, abi.PUSHER_VAY, abi.PUSHER_HC):
            A = orc.HostParticles(**{k: s[k] for k in orc.HostParticles.NAMES})
            B = A.copy()
            for push_position in (1, 0):
                orc.lib().orc_gather_push(C.byref(A.soa), 0, A.np, orc.fab_array(F[0:3]), orc.fab_array(F[3:6]),
                                          abi.dbl3(dinv), abi.dbl3(xyzmin), abi.int3(lo), s["q"], s["m"], dt, nox, galerkin,
                                          pusher, push_position)
                assert hl.pic_gather_push(C.byref(B.soa), 0, B.np, orc.fab_array(F[0:3]), orc.fab_array(F[3:6]),
                                          abi.dbl3(dinv), abi.dbl3(xyzmin), abi.int3(lo), s["q"], s["m"], dt, nox,
                                          galerkin, pusher, push_position, None, None, None) == 0, hl.pic_last_error()
            for k in ("x", "y", "z"):
                assert np.max(np.abs(getattr(A, k) - getattr(B, k))) <= 1e-13 * lx[0], (galerkin, pusher, k)
            for k in ("ux", "uy", "uz"):
                assert rel_linf(getattr(B, k), getattr(A, k)) <= 1e-13, (galerkin, pusher, k)


def test_weightless_particles_outside_the_fab_deposit_nothing(orc):
    """The antenna of a multi-rank run is replicated on every rank with zero weights outside the owning brick
    (engine.cu, lasers): such particles lie far outside the rank's J fabs and must not be turned into addresses.
    (Found on 4 GPUs: the zero adds of the three non-owning slabs went out of bounds.)"""
    from host_harness import harness
    hl = harness.host_library()
    n, lx, nox = (8, 6, 6), (4e-6, 3e-6, 3e-6), 3
    wl = workloads.uniform_plasma_3d(n_cell=n, ppc=(1, 1, 1), u_th=0.1, lx=lx, seed=4)
    s = wl["species"][0]
    dx = [(wl["prob_hi"][d] - wl["prob_lo"][d]) / n[d] for d in range(3)]
    dinv = [1.0 / v for v in dx]
    dt = 0.95 / (np.sqrt(sum(1.0 / v ** 2 for v in dx)) * workloads.C)
    box_hi = tuple(v - 1 for v in n)
    ngJ = (nox + 2,) * 3
    xyzmin, lo = lower_corner(wl["prob_lo"], dx, (0, 0, 0), ngJ)
    real = {k: s[k] for k in orc.HostParticles.NAMES}
    ghost = {k: np.concatenate([s[k], s[k][:16]]) for k in orc.HostParticles.NAMES}
    ghost["z"][-16:] += 3.0e6 * dx[2]                 # three million cells above the box
    ghost["w"][-16:] = 0.0
    P, G = orc.HostParticles(**real), orc.HostParticles(**ghost)
    J = [orc.HostFab((0, 0, 0), box_hi, ngJ, abi.YEE_STAG[c]) for c in (6, 7, 8)]
    K = [orc.HostFab((0, 0, 0), box_hi, ngJ, abi.YEE_STAG[c]) for c in (6, 7, 8)]
    assert orc.lib().orc_deposit_esirkepov(C.byref(P.soa), 0, P.np, orc.fab_array(J), abi.dbl3(dinv), abi.dbl3(xyzmin),
                                           abi.int3(lo), s["q"], dt, -0.5 * dt, nox) == 0
    assert hl.pic_deposit_esirkepov(C.byref(G.soa), 0, G.np, orc.fab_array(K), abi.dbl3(dinv), abi.dbl3(xyzmin), abi.int3(lo),
                                    s["q"], dt, -0.5 * dt, nox, None, None) == 0, hl.pic_last_error()
    for c in range(3):
        assert rel_linf(K[c].a, J[c].a) <= 1e-13, "j" + "xyz"[c]


# ---------------------------------------------------------------------------------------------------------
# the lane-per-cell deposition kernel of warpx_b200/csrc/deposit_cells.cu (PIC_DEPOSIT_CELLS) under the emulator
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nox,n,ppc,u_th,kind", [
    (3, (16, 8, 8), (2, 2, 2), 0.02, "sorted"),       # the benchmark's situation: every particle quiet in its bin
    (3, (16, 8, 8), (2, 1, 2), 0.3, "sorted"),        # relativistic: many particles change cell during the step
    (3, (16, 8, 8), (2, 2, 1), 0.05, "moved"),        # bins stale by up to 0.9 cell: listed particles
    (3, (12, 8, 10), (1, 1, 1), 0.1, "odd"),          # box not a multiple of the supercell, 1..3 particles per cell
    (1, (16, 8, 8), (2, 1, 2), 0.05, "moved"),
    (1, (12, 8, 10), (1, 1, 1), 0.3, "odd"),
    (3, (8, 8, 8), (2, 2, 2), 0.02, "tail"),          # particles appended behind the binned range
])
@pytest.mark.parametrize("mode", [abi.PIC_DEPOSIT_CELLS, abi.PIC_DEPOSIT_CELLS2, abi.PIC_DEPOSIT_CELLS3])
def test_deposit_cells_kernel_under_simt_emulation(orc, nox, n, ppc, u_th, kind, mode):
    from host_harness import harness
    hl = harness.host_library()
    lx = tuple(0.5e-6 * v for v in n)
    wl = workloads.uniform_plasma_3d(n_cell=n, ppc=ppc, u_th=u_th, lx=lx, seed=21)
    sp = wl["species"][0]
    prob_lo = wl["prob_lo"]
    dx = [(wl["prob_hi"][d] - prob_lo[d]) / n[d] for d in range(3)]
    dinv = [1.0 / v for v in dx]
    dt = 0.95 / (np.sqrt(sum(1.0 / v ** 2 for v in dx)) * workloads.C)
    rng = np.random.default_rng(23)
    arr = {k: sp[k].copy() for k in orc.HostParticles.NAMES}
    if kind == "odd":
        extra = rng.integers(0, 3, len(arr["x"]))
        for k in arr:
            arr[k] = np.repeat(arr[k], 1 + extra)
        for d, k in enumerate("xyz"):
            arr[k] = arr[k] + rng.uniform(-0.49, 0.49, len(arr[k])) * dx[d]
    order, cell_start = host_bins(arr["x"], arr["y"], arr["z"], prob_lo, dx, n, (8, 8, 8))
    arr = {k: np.ascontiguousarray(v[order]) for k, v in arr.items()}
    np_binned = len(arr["x"])
    if kind == "moved":
        for d, k in enumerate("xyz"):
            arr[k] = arr[k] + rng.uniform(-0.9, 0.9, len(arr[k])) * dx[d]
    if kind == "tail":           # 100 unsorted particles behind the bins (injected after the sort)
        for k in arr:
            arr[k] = np.concatenate([arr[k], arr[k][rng.integers(0, np_binned, 100)]])
        for d, k in enumerate("xyz"):
            arr[k][np_binned:] += rng.uniform(-0.4, 0.4, 100) * dx[d]
    P = orc.HostParticles(**arr)
    ngJ = (nox + 2,) * 3
    box_hi = tuple(v - 1 for v in n)
    xyzmin, lo = lower_corner(prob_lo, dx, (0, 0, 0), ngJ)
    J = [orc.HostFab((0, 0, 0), box_hi, ngJ, abi.YEE_STAG[c]) for c in (6, 7, 8)]
    K = [orc.HostFab((0, 0, 0), box_hi, ngJ, abi.YEE_STAG[c]) for c in (6, 7, 8)]
    bins = abi.pic_bins()
    bins.cell_start = cell_start.ctypes.data
    for d in range(3):
        bins.box_lo[d], bins.box_hi[d], bins.tile[d] = 0, box_hi[d], 8
    bins.np_binned = np_binned
    assert orc.lib().orc_deposit_esirkepov(C.byref(P.soa), 0, P.np, orc.fab_array(J), abi.dbl3(dinv), abi.dbl3(xyzmin),
                                           abi.int3(lo), sp["q"], dt, -0.5 * dt, nox) == 0
    hl.pic_set_deposit_mode(mode)
    try:
        assert hl.pic_deposit_esirkepov(C.byref(P.soa), 0, P.np, orc.fab_array(K), abi.dbl3(dinv), abi.dbl3(xyzmin),
                                        abi.int3(lo), sp["q"], dt, -0.5 * dt, nox, C.byref(bins), None) == 0, hl.pic_last_error()
    finally:
        hl.pic_set_deposit_mode(0)
    for c in range(3):
        assert rel_linf(K[c].a, J[c].a) <= 1e-13, "j" + "xyz"[c]


# ---------------------------------------------------------------------------------------------------------
# the FDTD kernels on the host: plain loads (fdtd.cu) and the bulk-asynchronous staging of fdtd_bulk.cu (the emulator
# performs the bulk copies synchronously: ring indexing, row / plane clamps, alignment widening, tail element)
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [3, 1, 0])
@pytest.mark.parametrize("algo", [abi.SOLVER_YEE, abi.SOLVER_CKC])
@pytest.mark.parametrize("n,ng", [((16, 12, 10), (2, 2, 2)), ((70, 9, 37), (1, 2, 1)), ((7, 6, 5), (4, 4, 4))])
def test_fdtd_kernels_under_simt_emulation(orc, mode, algo, n, ng):
    from host_harness import harness
    from helpers import random_fields
    hl = harness.host_library()
    L = orc.lib()
    box_lo, box_hi = (0, 0, 0), tuple(v - 1 for v in n)
    dx = [1e-6, 1.5e-6, 0.8e-6]
    st = abi.pic_stencil()
    L.orc_stencil_coefs(algo, (C.c_double * 3)(*dx), C.byref(st))
    scale = [1e9] * 3 + [3.0] * 3 + [1e12] * 3
    F = random_fields(orc, box_lo, box_hi, ng, 11, comps=range(9), scale=scale)
    G = random_fields(orc, box_lo, box_hi, ng, 11, comps=range(9), scale=scale)
    dt = 1.1e-15
    hl.pic_set_fdtd_mode(mode)
    before = hl.pic_fdtd_bulk_launches()
    try:
        E, B, J = orc.fab_array(G[0:3]), orc.fab_array(G[3:6]), orc.fab_array(G[6:9])
        assert hl.pic_evolve_b(B, E, C.byref(st), 0.5 * dt, None) == 0, hl.pic_last_error()
        assert hl.pic_evolve_e(E, B, J, C.byref(st), dt, None) == 0, hl.pic_last_error()
        assert hl.pic_evolve_b(B, E, C.byref(st), 0.5 * dt, None) == 0, hl.pic_last_error()
    finally:
        hl.pic_set_fdtd_mode(1)
    # EvolveE is staged for both solvers, EvolveB for Yee (numpy arrays are 16-byte aligned)
    want = (2 if (mode & 1) and algo == abi.SOLVER_YEE else 0) + (1 if mode & 2 else 0)
    assert hl.pic_fdtd_bulk_launches() - before == want
    Eo, Bo, Jo = orc.fab_array(F[0:3]), orc.fab_array(F[3:6]), orc.fab_array(F[6:9])
    L.orc_evolve_b(Bo, Eo, C.byref(st), 0.5 * dt)
    L.orc_evolve_e(Eo, Bo, Jo, C.byref(st), dt)
    L.orc_evolve_b(Bo, Eo, C.byref(st), 0.5 * dt)
    for c in range(6):
        assert rel_linf(G[c].a, F[c].a) <= 1e-13, abi.COMP_NAMES[c]


# ---------------------------------------------------------------------------------------------------------
# bilinear filter: the streaming (marching) kernel of npass = (1,1,1) and the direct kernel, under the emulator
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("npass", [(1, 1, 1), (2, 1, 3)])
def test_bilinear_filter_kernels_under_simt_emulation(orc, npass):
    """pic_apply_filter / pic_apply_filter_multi of the host library against the oracle's Filter::DoFilter: three
    components of different staggering in one launch, a box that is ragged against the 32 x 8 CTA and longer than one
    chunk of planes, zero padding at the array edge, a destination larger than the source; the single-component call
    gives the same bits as the multi call."""
    from host_harness import harness
    from helpers import random_fields
    hl = harness.host_library()
    n = (37, 11, 35)
    box_lo, box_hi = (0, 0, 0), tuple(v - 1 for v in n)
    ng = (3, 2, 2)
    src = random_fields(orc, box_lo, box_hi, ng, 31, comps=[6, 7, 8])
    want = [orc.HostFab(box_lo, box_hi, ng, abi.YEE_STAG[c]) for c in (6, 7, 8)]
    for a, b in zip(src, want):
        orc.lib().orc_apply_filter(C.byref(a.desc), C.byref(b.desc), abi.int3(npass))
    got = [orc.HostFab(box_lo, box_hi, ng, abi.YEE_STAG[c]) for c in (6, 7, 8)]
    for g in got:
        g.a[...] = 7.0                                        # every point of dst must be overwritten
    assert hl.pic_apply_filter_multi(orc.fab_array(src), orc.fab_array(got), 3, abi.int3(npass), None) == 0, hl.pic_last_error()
    for c in range(3):
        assert rel_linf(got[c].a, want[c].a) <= 1e-14, c
    one = orc.HostFab(box_lo, box_hi, ng, abi.YEE_STAG[7])
    assert hl.pic_apply_filter(C.byref(src[1].desc), C.byref(one.desc), abi.int3(npass), None) == 0, hl.pic_last_error()
    assert np.array_equal(one.a, got[1].a)
    # a destination with more guard cells than the source: zero padding outside the source's allocation
    big = orc.HostFab(box_lo, box_hi, (4, 4, 3), abi.YEE_STAG[6])
    wbig = orc.HostFab(box_lo, box_hi, (4, 4, 3), abi.YEE_STAG[6])
    orc.lib().orc_apply_filter(C.byref(src[0].desc), C.byref(wbig.desc), abi.int3(npass))
    assert hl.pic_apply_filter(C.byref(src[0].desc), C.byref(big.desc), abi.int3(npass), None) == 0, hl.pic_last_error()
    assert rel_linf(big.a, wbig.a) <= 1e-14


# ---------------------------------------------------------------------------------------------------------
# the particle sets of tests/particle_sets.py (steady state, Poisson counts, a full sub-particle queue) through the
# host library's C ABI: the cell-sorted deposition modes and the supercell gather, against the oracle
# ---------------------------------------------------------------------------------------------------------
EMULATED_SETS = ("steady", "poisson", "crowded_movers")


@pytest.mark.parametrize("mode", [abi.PIC_DEPOSIT_RUNS, abi.PIC_DEPOSIT_RUNS_SLAB, abi.PIC_DEPOSIT_CELLS,
                                  abi.PIC_DEPOSIT_CELLS3])
@pytest.mark.parametrize("nox", [1, 3])
@pytest.mark.parametrize("name", EMULATED_SETS)
def test_deposition_modes_on_particle_sets_under_simt_emulation(orc, name, nox, mode):
    from host_harness import harness
    hl = harness.host_library()
    s = ps.get(name)
    ng = (nox + 2,) * 3
    xyzmin, lo = s.corner(ng)
    P = orc.HostParticles(**s.arrays())
    J = [orc.HostFab(s.box_lo, s.box_hi, ng, abi.YEE_STAG[c]) for c in (6, 7, 8)]
    K = [orc.HostFab(s.box_lo, s.box_hi, ng, abi.YEE_STAG[c]) for c in (6, 7, 8)]
    args = (abi.dbl3(s.dinv), abi.dbl3(xyzmin), abi.int3(lo), s.q, s.dt, -0.5 * s.dt, nox)
    assert orc.lib().orc_deposit_esirkepov(C.byref(P.soa), 0, P.np, orc.fab_array(J), *args) == 0
    cs = s.cell_start.astype(np.int32)
    bins = abi.pic_bins()
    bins.cell_start = cs.ctypes.data
    for d in range(3):
        bins.box_lo[d], bins.box_hi[d], bins.tile[d] = s.box_lo[d], s.box_hi[d], ps.TILE
    bins.np_binned = s.np
    hl.pic_set_deposit_mode(mode)
    try:
        assert hl.pic_deposit_esirkepov(C.byref(P.soa), 0, P.np, orc.fab_array(K), *args, C.byref(bins), None) == 0, \
            hl.pic_last_error()
    finally:
        hl.pic_set_deposit_mode(0)
    for c in range(3):
        assert rel_linf(K[c].a, J[c].a) <= 1e-13, "j" + "xyz"[c]


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("name", EMULATED_SETS + ("scrambled_rows",))
def test_gather_push_tile_kernels_on_particle_sets_under_simt_emulation(orc, simt, name, mode):
    s = ps.get(name)
    nox, galerkin = 3, 1
    ngEB = (4, 4, 4)
    xyzmin, lo = s.corner(ngEB)
    from helpers import random_fields
    F = random_fields(orc, s.box_lo, s.box_hi, ngEB, 5, comps=range(6), scale=[1e10] * 3 + [30.0] * 3)
    P = orc.HostParticles(**s.arrays())
    Q = P.copy()
    cs = s.cell_start.astype(np.int32)
    bins = abi.pic_bins()
    bins.cell_start = cs.ctypes.data
    for d in range(3):
        bins.box_lo[d], bins.box_hi[d], bins.tile[d] = s.box_lo[d], s.box_hi[d], ps.TILE
    bins.np_binned = s.np
    for push_position in (1, 0):
        assert simt.simt_gather_push(C.byref(Q.soa), orc.fab_array(F[0:3]), orc.fab_array(F[3:6]), abi.dbl3(s.dinv),
                                     abi.dbl3(xyzmin), abi.int3(lo), s.q, s.m, s.dt, nox, galerkin,
                                     abi.PUSHER_BORIS, push_position, C.byref(bins), mode) == 0
        orc.lib().orc_gather_push(C.byref(P.soa), 0, P.np, orc.fab_array(F[0:3]), orc.fab_array(F[3:6]), abi.dbl3(s.dinv),
                                  abi.dbl3(xyzmin), abi.int3(lo), s.q, s.m, s.dt, nox, galerkin, abi.PUSHER_BORIS,
                                  push_position)
    lx = s.n[0] * s.dx[0]
    for k in ("x", "y", "z"):
        assert np.max(np.abs(getattr(Q, k) - getattr(P, k))) <= 1e-13 * lx, k
    for k in ("ux", "uy", "uz"):
        assert rel_linf(getattr(Q, k), getattr(P, k)) <= 1e-13, k
