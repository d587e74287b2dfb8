"""GPU parity tests (-m gpu) of the deposition and gather kernels on the particle sets of tests/particle_sets.py: the
steady state the benchmark runs in (movers, lone strays, register-window jumps, stray lists) and adversarial sets
(Poisson counts and long runs, particles on faces, a full sub-particle queue, overflowing gather lists, nearly empty
boxes, a brick at a nonzero box_lo), every deposition mode and every gather mode, against the CPU oracle.

Deposition: J starts from a random background B of about the size of the deposited current, so a retire or flush that
stores instead of adding is caught.  Bars: |J_gpu - J_oracle| <= 1e-12 max|J_oracle - B| (the CUDA code contracts into
FMAs and reorders sums; the oracle is built with -ffp-contract=off), and J_gpu == B bit for bit on every node that no
particle's stencil reaches.  Gather + push: as test_gpu_parity.py, positions 1e-13 of the box, momenta rel-Linf 1e-13.
Steady-state loop: as test_order3_loop_matches_oracle."""
import ctypes as C

import numpy as np
import pytest

import particle_sets as ps
from helpers import random_fields, rel_linf
from test_gpu_parity import Dev, _match_particles, _run_both  # noqa: F401
from warpx_b200 import abi, workloads

pytestmark = pytest.mark.gpu


@pytest.fixture()
def dev(cuda):
    return Dev(cuda)


CASES = ps.SETS + ("poisson+offset", "crowded_movers+offset", "steady+offset")
GLOBAL = "global"         # bins = NULL: the order-agnostic kernel
DEPOSIT_MODES = (GLOBAL, abi.PIC_DEPOSIT_RUNS, abi.PIC_DEPOSIT_TILE, abi.PIC_DEPOSIT_RUNS2, abi.PIC_DEPOSIT_RUNS_SLOTRED,
                 abi.PIC_DEPOSIT_RUNS2_SLOTRED, abi.PIC_DEPOSIT_RUNS4, abi.PIC_DEPOSIT_RUNS4_SLOTRED, abi.PIC_DEPOSIT_CELLS,
                 abi.PIC_DEPOSIT_CELLS2, abi.PIC_DEPOSIT_CELLS2_WIDE, abi.PIC_DEPOSIT_CELLS3, abi.PIC_DEPOSIT_CELLS3_WIDE,
                 abi.PIC_DEPOSIT_RUNS_SLAB)
CELLS_MODES = (abi.PIC_DEPOSIT_CELLS, abi.PIC_DEPOSIT_CELLS2, abi.PIC_DEPOSIT_CELLS2_WIDE, abi.PIC_DEPOSIT_CELLS3,
               abi.PIC_DEPOSIT_CELLS3_WIDE)


def deposit_mode_applies(mode, nox):
    """False where the mode would run the same kernel as another case (the library falls back)."""
    if nox == 4:
        return mode in (GLOBAL, abi.PIC_DEPOSIT_RUNS)           # order 4 with bins: the order-agnostic kernel
    if mode in (abi.PIC_DEPOSIT_RUNS4, abi.PIC_DEPOSIT_RUNS4_SLOTRED):
        return nox == 3
    if mode in CELLS_MODES:
        return nox in (1, 3)
    if mode in (abi.PIC_DEPOSIT_RUNS2, abi.PIC_DEPOSIT_RUNS2_SLOTRED):
        return nox in (1, 3)                                     # two lines per lane need N + 1 even
    return True


def device_bins(dev, s):
    cs = dev.t.from_numpy(s.cell_start.astype(np.int32)).cuda()
    bins = abi.pic_bins()
    bins.cell_start = cs.data_ptr()
    for d in range(3):
        bins.box_lo[d], bins.box_hi[d], bins.tile[d] = s.box_lo[d], s.box_hi[d], ps.TILE
    bins.np_binned = s.np
    dev.keep.append(cs)
    return bins


def deposit_both(orc, dev, s, nox, mode, offset=0, count=None, ng=None, with_bins=True):
    """Deposit particles [offset, offset + count) of set s on the GPU (deposition mode `mode`) and with the oracle into J
    that starts from the random background B.  Returns (rc, J_gpu, J_oracle, B) as lists of numpy arrays."""
    count = s.np - offset if count is None else count
    ng = (nox + 2,) * 3 if ng is None else ng
    xyzmin, lo = s.corner(ng)
    J = [orc.HostFab(s.box_lo, s.box_hi, ng, abi.YEE_STAG[c]) for c in (6, 7, 8)]
    P = orc.HostParticles(**s.arrays())
    args = (abi.dbl3(s.dinv), abi.dbl3(xyzmin), abi.int3(lo), s.q, s.dt, -0.5 * s.dt, nox)
    assert orc.lib().orc_deposit_esirkepov(C.byref(P.soa), offset, count, orc.fab_array(J), *args) == 0
    rng = np.random.default_rng(1000 + nox)
    scale = max(float(np.max(np.abs(f.a))) for f in J)
    B = [scale * rng.standard_normal(f.a.shape) for f in J]
    want = [f.a + b for f, b in zip(J, B)]
    for f, b in zip(J, B):
        f.a[...] = b
    arr, tens = dev.fabs(J)
    Pd, _ = dev.soa(P)
    bins = C.byref(device_bins(dev, s)) if with_bins and mode != GLOBAL else None
    dev.L.pic_set_deposit_mode(abi.PIC_DEPOSIT_RUNS if mode == GLOBAL else mode)
    try:
        rc = dev.L.pic_deposit_esirkepov(C.byref(Pd), offset, count, (abi.pic_fab * 3)(*arr), *args, bins, dev.stream)
        dev.sync()
    finally:
        dev.L.pic_set_deposit_mode(abi.PIC_DEPOSIT_RUNS)
    return rc, [t.cpu().numpy() for t in tens], want, B


def check_deposit(s, got, want, B, ng, nox):
    for c in range(3):
        name = "j" + "xyz"[c]
        dep = want[c] - B[c]
        assert np.max(np.abs(got[c] - want[c])) <= 1e-12 * np.max(np.abs(dep)), name
        untouched = ~ps.reach(s, got[c].shape, ng, nox)
        assert np.array_equal(got[c][untouched], B[c][untouched]), name + ": a node no stencil reaches changed"


@pytest.mark.parametrize("nox,mode", [(nox, mode) for nox in (1, 2, 3, 4) for mode in DEPOSIT_MODES
                                      if deposit_mode_applies(mode, nox)])
@pytest.mark.parametrize("case", CASES)
def test_deposit_sets_match_oracle(orc, dev, case, nox, mode):
    s = ps.get(case)
    rc, got, want, B = deposit_both(orc, dev, s, nox, mode)
    dev.ok(rc)
    check_deposit(s, got, want, B, (nox + 2,) * 3, nox)


def gather_both(orc, dev, s, nox, galerkin, mode, offset=0, count=None, with_bins=True):
    """PushPX then PushP of particles [offset, offset + count) on the GPU (gather mode `mode`) and with the oracle, on
    random fields.  Returns (rc, particles after the GPU push (7 x np), the oracle's HostParticles)."""
    count = s.np - offset if count is None else count
    ngEB = (4, 4, 4)
    xyzmin, lo = s.corner(ngEB)
    F = random_fields(orc, s.box_lo, s.box_hi, ngEB, 5, comps=range(6), scale=[1e10] * 3 + [30.0] * 3)
    arr, _ = dev.fabs(F)
    E, Bf = (abi.pic_fab * 3)(*arr[0:3]), (abi.pic_fab * 3)(*arr[3:6])
    P = orc.HostParticles(**s.arrays())
    Pd, buf = dev.soa(P)
    bins = C.byref(device_bins(dev, s)) if with_bins and mode != GLOBAL else None
    dt = s.dt
    args = (abi.dbl3(s.dinv), abi.dbl3(xyzmin), abi.int3(lo), s.q, s.m, dt, nox, galerkin, abi.PUSHER_BORIS)
    dev.L.pic_set_gather_mode(abi.PIC_GATHER_TILE if mode == GLOBAL else mode)
    rc = 0
    try:
        for push_position in (1, 0):
            rc = rc or dev.L.pic_gather_push(C.byref(Pd), offset, count, E, Bf, *args, push_position, bins, None, dev.stream)
            assert orc.lib().orc_gather_push(C.byref(P.soa), offset, count, orc.fab_array(F[0:3]), orc.fab_array(F[3:6]),
                                             *args, push_position) == 0
        dev.sync()
    finally:
        dev.L.pic_set_gather_mode(abi.PIC_GATHER_TILE)
    return rc, buf.cpu().numpy(), P


def check_gather(s, got, P, sl=slice(None)):
    lx = s.n[0] * s.dx[0]
    for i, k in enumerate(("x", "y", "z")):
        assert np.max(np.abs(got[i][sl] - getattr(P, k)[sl])) <= 1e-13 * lx, k
    for i, k in ((4, "ux"), (5, "uy"), (6, "uz")):
        assert rel_linf(got[i][sl], getattr(P, k)[sl]) <= 1e-13, k


@pytest.mark.parametrize("mode,galerkin", [(GLOBAL, 1), (GLOBAL, 0), (abi.PIC_GATHER_TILE, 1), (abi.PIC_GATHER_TILE, 0),
                                           (abi.PIC_GATHER_PAIRS, 1), (abi.PIC_GATHER_PAIRS_WIDE, 1),
                                           (abi.PIC_GATHER_PAIRS_192, 1)])
@pytest.mark.parametrize("nox", [1, 2, 3])
@pytest.mark.parametrize("case", CASES)
def test_gather_sets_match_oracle(orc, dev, case, nox, mode, galerkin):
    s = ps.get(case)
    rc, got, P = gather_both(orc, dev, s, nox, galerkin, mode)
    dev.ok(rc)
    check_gather(s, got, P)


# ---------------------------------------------------------------------------------------------------------------------
# A particle range inside the tile (offset > 0, fewer particles than the tile) through the C ABI
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [GLOBAL, abi.PIC_DEPOSIT_RUNS, abi.PIC_DEPOSIT_RUNS_SLAB, abi.PIC_DEPOSIT_CELLS])
@pytest.mark.parametrize("nox", [1, 3])
def test_deposit_partial_range_matches_oracle(orc, dev, nox, mode):
    """The run kernels and the order-agnostic kernel deposit exactly [offset, offset + np); PIC_DEPOSIT_CELLS needs the
    whole tile and hands a sub-range to the run kernels."""
    s = ps.get("steady")
    offset, count = 1000, 3000
    rc, got, want, B = deposit_both(orc, dev, s, nox, mode, offset=offset, count=count)
    dev.ok(rc)
    sub = ps.ParticleSet(s.name, s.n, s.dx, {k: v[offset:offset + count] for k, v in s.p.items()}, s.cell_start, s.dt)
    check_deposit(sub, got, want, B, (nox + 2,) * 3, nox)


def test_deposit_tile_refuses_a_partial_range(orc, dev):
    """PIC_DEPOSIT_TILE walks the bins of the whole tile: a sub-range is an error (PIC_ERR_RETURN), J is untouched."""
    s = ps.get("poisson")
    rc, got, _, B = deposit_both(orc, dev, s, 3, abi.PIC_DEPOSIT_TILE, offset=100, count=500)
    assert rc != 0 and b"offset 0" in dev.L.pic_last_error()
    for c in range(3):
        assert np.array_equal(got[c], B[c])


@pytest.mark.parametrize("nox", [1, 3, 4])
def test_gather_partial_range_matches_oracle(orc, dev, nox):
    """bins = NULL: particles [offset, offset + np) are pushed like the oracle pushes them, the others keep their bits;
    with bins the call must cover the whole tile and a sub-range is refused."""
    s = ps.get("steady")
    offset, count = 1000, 3000
    rc, got, P = gather_both(orc, dev, s, nox, 1, GLOBAL, offset=offset, count=count)
    dev.ok(rc)
    check_gather(s, got, P, slice(offset, offset + count))
    for i, k in enumerate(ps.NAMES):
        assert np.array_equal(got[i][:offset], s.p[k][:offset]) and np.array_equal(got[i][offset + count:],
                                                                                    s.p[k][offset + count:]), k
    if nox <= 3:
        rc, got, _ = gather_both(orc, dev, s, nox, 1, abi.PIC_GATHER_TILE, offset=offset, count=count)
        assert rc != 0 and b"whole tile" in dev.L.pic_last_error()
        for i, k in enumerate(ps.NAMES):
            assert np.array_equal(got[i], s.p[k]), k


# ---------------------------------------------------------------------------------------------------------------------
# The run kernels pack a cell into 10 bits per direction: J wider than that is refused, not deposited
# ---------------------------------------------------------------------------------------------------------------------
def wide_set(nx):
    """Particles in the lowest and highest cells along x of an nx x 8 x 8 box (plus a few in between)."""
    n, dx = (nx, 8, 8), (ps.DX_EXACT,) * 3
    rng = np.random.default_rng(nx)
    counts = np.zeros((n[2], n[1], n[0]), dtype=np.int64)
    counts[:, :, [0, 1, nx // 2, nx - 2, nx - 1]] = 2
    pos = ps._uniform_in_cells(rng, counts, n, dx)
    u = rng.normal(0.0, 0.1 * workloads.C, (len(pos[0]), 3))
    return ps._finish("wide%d" % nx, n, dx, pos, u, rng, ps.cfl_dt(dx))


@pytest.mark.parametrize("mode", [abi.PIC_DEPOSIT_RUNS, abi.PIC_DEPOSIT_RUNS_SLAB, abi.PIC_DEPOSIT_RUNS2,
                                  abi.PIC_DEPOSIT_CELLS])
def test_run_kernels_refuse_j_wider_than_their_keys(orc, dev, mode):
    """nox 3, ng 5: a box of 1010 cells gives Jy / Jz 1021 points along x, the widest the run kernels take (deposited
    like the oracle); 1011 cells give 1022 points: an error code, J untouched."""
    nox = 3
    s = wide_set(1010)
    rc, got, want, B = deposit_both(orc, dev, s, nox, mode)
    dev.ok(rc)
    check_deposit(s, got, want, B, (nox + 2,) * 3, nox)
    s = wide_set(1011)
    rc, got, _, B = deposit_both(orc, dev, s, nox, mode)
    assert rc != 0 and b"J extent" in dev.L.pic_last_error()
    for c in range(3):
        assert np.array_equal(got[c], B[c])


# ---------------------------------------------------------------------------------------------------------------------
# The whole loop from the steady state
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("deposit_mode,gather_mode", [(abi.PIC_DEPOSIT_RUNS, abi.PIC_GATHER_TILE),
                                                      (abi.PIC_DEPOSIT_RUNS_SLAB, abi.PIC_GATHER_TILE),
                                                      (abi.PIC_DEPOSIT_CELLS, abi.PIC_GATHER_TILE),
                                                      (abi.PIC_DEPOSIT_RUNS, abi.PIC_GATHER_PAIRS)])
def test_steady_state_loop_matches_oracle(orc, cuda, deposit_mode, gather_mode):
    """`steady` particles (with their log-uniform weights; 16^3 cells: the guard-cell exchange of order 3 needs more
    than 8 cells per axis) handed to the engine and to a fresh oracle, fields zero in both, 12 steps of order 3 with a
    cell sort every 4: the bar of test_order3_loop_matches_oracle."""
    from warpx_b200.lib import lib as piclib
    s = ps.steady(n=(16, 16, 16))
    wl = dict(n_cell=s.n, prob_lo=s.prob_lo, prob_hi=s.prob_hi,
              species=[dict(name="electrons", q=s.q, m=s.m, **s.arrays())])
    piclib().pic_set_deposit_mode(deposit_mode)
    piclib().pic_set_gather_mode(gather_mode)
    try:
        sim, osim = _run_both(orc, cuda, wl, 3, 12, sort_interval=4)
    finally:
        piclib().pic_set_deposit_mode(abi.PIC_DEPOSIT_RUNS)
        piclib().pic_set_gather_mode(abi.PIC_GATHER_TILE)
    for c in range(9):
        d, a = sim.field_numpy(c)
        _, oa = osim.fab(c)
        tol = 1e-9 if c not in (3, 4, 5) else 1e-7       # B: thermal-noise level, see test_order3_loop_matches_oracle
        assert rel_linf(a[d.valid_slices()], oa[d.valid_slices()]) <= tol, abi.COMP_NAMES[c]
    e, b = sim.field_energy()
    eo, bo = osim.field_energy()
    assert e == pytest.approx(eo, rel=1e-10) and b == pytest.approx(bo, rel=1e-8)
    A, B = _match_particles(sim, osim, 0)
    for k in ("x", "y", "z"):
        assert np.max(np.abs(A[k] - B[k])) / sim.dx[0] <= 1e-10
    for k in ("ux", "uy", "uz"):
        assert np.max(np.abs(A[k] - B[k])) / workloads.C <= 1e-10
