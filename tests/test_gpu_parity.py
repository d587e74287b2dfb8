"""GPU parity tests (-m gpu): every CUDA stage, called through the C ABI, against the CPU oracle
on identical seeded inputs; the whole loop against WarpX's golden checksums.

Tolerances (fp64; the CUDA code contracts a*b+c into FMAs and reorders sums, the oracle is built
with -ffp-contract=off):
    FDTD, gather+push, guard cells ........ rel-Linf <= 1e-13 after one application
    Esirkepov J ........................... |dJ| <= 1e-12 * max|J| after one deposition
    40-step Langmuir loop ................. WarpX checksums at WarpX's own rtol 1e-9;
                                            fields vs oracle rel-Linf <= 1e-9, field energy 1e-10,
                                            per-particle x/dx and u/c <= 1e-10
"""
import ctypes as C

import numpy as np
import pytest

from helpers import lower_corner, random_fields, rel_linf
from warpx_b200 import abi, workloads

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------
class Dev:
    """Device copies of HostFab / HostParticles with descriptors for the C ABI."""

    def __init__(self, torch):
        from warpx_b200.lib import lib
        self.t = torch
        self.L = lib()
        self.L.pic_set_error_mode(abi.PIC_ERR_RETURN)
        self.keep = []

    @property
    def stream(self):
        return self.t.cuda.current_stream().cuda_stream

    def fabs(self, hostfabs):
        arr = (abi.pic_fab * len(hostfabs))()
        tens = []
        for n, hf in enumerate(hostfabs):
            d = self.t.from_numpy(hf.a).cuda()
            arr[n] = hf.desc
            arr[n].p = d.data_ptr()
            tens.append(d)
        self.keep.append(tens)
        return arr, tens

    def soa(self, P, names=("x", "y", "z", "w", "ux", "uy", "uz")):
        buf = self.t.stack([self.t.from_numpy(getattr(P, n)) for n in names]).cuda()
        s = abi.pic_soa()
        for n, name in enumerate(names):
            setattr(s, name, buf[n].data_ptr())
        s.idcpu = None
        s.np = P.np
        self.keep.append(buf)
        return s, buf

    def sync(self):
        self.t.cuda.synchronize()

    def ok(self, rc):
        assert rc == 0, self.L.pic_last_error().decode()


@pytest.fixture()
def dev(cuda):
    return Dev(cuda)


def box(n):
    return (0, 0, 0), tuple(v - 1 for v in n)


# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("algo", [abi.SOLVER_YEE, abi.SOLVER_CKC])
@pytest.mark.parametrize("n", [(16, 12, 10), (70, 9, 5)])
def test_fdtd_matches_oracle(orc, dev, algo, n):
    L = orc.lib()
    box_lo, box_hi = box(n)
    dx = [1e-6, 1.5e-6, 0.8e-6]
    st = abi.pic_stencil()
    L.orc_stencil_coefs(algo, (C.c_double * 3)(*dx), C.byref(st))
    F = random_fields(orc, box_lo, box_hi, (2, 2, 2), 11, comps=range(9), scale=[1e9] * 3 + [3.0] * 3 + [1e12] * 3)
    arr, tens = dev.fabs(F)
    E, B, J = (abi.pic_fab * 3)(*arr[0:3]), (abi.pic_fab * 3)(*arr[3:6]), (abi.pic_fab * 3)(*arr[6:9])
    dt = 1.1e-15
    dev.ok(dev.L.pic_evolve_b(B, E, C.byref(st), 0.5 * dt, dev.stream))
    dev.ok(dev.L.pic_evolve_e(E, B, J, C.byref(st), dt, dev.stream))
    dev.ok(dev.L.pic_evolve_b(B, E, C.byref(st), 0.5 * dt, dev.stream))
    dev.sync()
    Eo, Bo, Jo = orc.fab_array(F[0:3]), orc.fab_array(F[3:6]), orc.fab_array(F[6:9])
    L.orc_evolve_b(Bo, Eo, C.byref(st), 0.5 * dt)
    L.orc_evolve_e(Eo, Bo, Jo, C.byref(st), dt)
    L.orc_evolve_b(Bo, Eo, C.byref(st), 0.5 * dt)
    for c in range(6):
        assert rel_linf(tens[c].cpu().numpy(), F[c].a) <= 1e-13, abi.COMP_NAMES[c]


def _particles(orc, n, ppc, u_th, lx, seed=1, shuffle=False):
    wl = workloads.uniform_plasma_3d(n_cell=n, ppc=ppc, u_th=u_th, lx=lx, seed=seed)
    sp = wl["species"][0]
    if shuffle:
        perm = np.random.default_rng(seed).permutation(len(sp["x"]))
        for k in orc.HostParticles.NAMES:
            sp[k] = sp[k][perm]
    return wl, sp


def _sorted_device_species(dev, sp_host, n, prob_lo, prob_hi, tile=(8, 8, 8)):
    """Counting-sort the particles on the device; returns (soa, buffer, bins, cell_start)."""
    t = dev.t
    P_in, buf_in = dev.soa(sp_host)
    buf_out = t.empty_like(buf_in)
    P_out = abi.pic_soa()
    for i, name in enumerate(("x", "y", "z", "w", "ux", "uy", "uz")):
        setattr(P_out, name, buf_out[i].data_ptr())
    P_out.idcpu = None
    P_out.np = P_in.np
    bins = abi.pic_bins()
    for d in range(3):
        bins.box_lo[d], bins.box_hi[d], bins.tile[d] = 0, n[d] - 1, tile[d]
    nb = dev.L.pic_bins_count(bins.box_lo, bins.box_hi, bins.tile)
    cell_start = t.empty(nb + 1, dtype=t.int32, device="cuda")
    work = t.empty(dev.L.pic_sort_workspace_bytes(P_in.np, nb), dtype=t.uint8, device="cuda")
    bins.cell_start = cell_start.data_ptr()
    bins.np_binned = P_in.np
    geom = abi.make_geom(n, prob_lo, prob_hi)
    dev.ok(dev.L.pic_sort_particles_by_cell(C.byref(P_in), C.byref(P_out), C.byref(geom), C.byref(bins),
                                            work.data_ptr(), dev.stream))
    dev.sync()
    dev.keep += [buf_out, cell_start, work]
    return P_out, buf_out, bins, cell_start, nb


def test_sort_bins_are_consistent(orc, dev):
    n = (20, 16, 12)
    lx = 1e-5
    wl, sp = _particles(orc, n, (2, 1, 2), 0.3, lx, shuffle=True)
    P = orc.HostParticles(**{k: sp[k] for k in orc.HostParticles.NAMES})
    Ps, buf, bins, cell_start, nb = _sorted_device_species(dev, P, n, wl["prob_lo"], wl["prob_hi"])
    cs = cell_start.cpu().numpy()
    out = buf.cpu().numpy()
    assert cs[0] == 0 and cs[-1] == P.np and np.all(np.diff(cs) >= 0)
    # permutation of the input (same multiset of particles)
    key_in = np.sort(P.x + 3.0 * P.y + 7.0 * P.z + 1e-12 * P.ux)
    key_out = np.sort(out[0] + 3.0 * out[1] + 7.0 * out[2] + 1e-12 * out[4])
    assert np.array_equal(key_in, key_out)
    # every particle sits in the bin of its cell (supercell-major numbering)
    dx = [(wl["prob_hi"][d] - wl["prob_lo"][d]) / n[d] for d in range(3)]
    cell = [np.clip(np.floor((out[d] - wl["prob_lo"][d]) / dx[d]).astype(int), 0, n[d] - 1) for d in range(3)]
    T = 8
    nt = [(n[d] + T - 1) // T for d in range(3)]
    tcell = [c // T for c in cell]
    lcell = [c % T for c in cell]
    binid = (tcell[0] + nt[0] * (tcell[1] + nt[1] * tcell[2])) * T ** 3 + lcell[0] + T * (lcell[1] + T * lcell[2])
    which = np.searchsorted(cs, np.arange(P.np), side="right") - 1
    assert np.array_equal(which, binid)


@pytest.mark.parametrize("nox,galerkin", [(1, 1), (1, 0), (2, 1), (3, 1), (3, 0)])
@pytest.mark.parametrize("pusher", [abi.PUSHER_BORIS, abi.PUSHER_VAY, abi.PUSHER_HC])
@pytest.mark.parametrize("path", ["global", "tile", "tile_drifted"])
def test_gather_push_matches_oracle(orc, dev, nox, galerkin, pusher, path):
    if pusher != abi.PUSHER_BORIS and (nox, galerkin) not in ((3, 1), (1, 1)):
        pytest.skip("pusher variants are covered at orders 1 and 3")
    L = orc.lib()
    n = (20, 16, 12)
    lx = 1e-5
    box_lo, box_hi = box(n)
    wl, sp = _particles(orc, n, (2, 1, 2), 0.3, lx, shuffle=(path == "global"))
    prob_lo = wl["prob_lo"]
    dx = [(wl["prob_hi"][d] - prob_lo[d]) / n[d] for d in range(3)]
    dinv = [1.0 / v for v in dx]
    ngEB = (4, 4, 4) if nox == 3 else (2, 2, 2)
    xyzmin, lo = lower_corner(prob_lo, dx, box_lo, ngEB)
    F = random_fields(orc, box_lo, box_hi, ngEB, 5, comps=range(6), scale=[1e10] * 3 + [30.0] * 3)
    P = orc.HostParticles(**{k: sp[k] for k in orc.HostParticles.NAMES})
    arr, _ = dev.fabs(F)
    E, B = (abi.pic_fab * 3)(*arr[0:3]), (abi.pic_fab * 3)(*arr[3:6])
    dt = 0.9 * dx[0] / workloads.C
    if path == "global":
        Pd, buf = dev.soa(P)
        bins = None
    else:
        Pd, buf, bins_s, _, _ = _sorted_device_species(dev, P, n, prob_lo, wl["prob_hi"])
        bins = C.byref(bins_s)
        if path == "tile_drifted":   # particles moved since the sort: bins are stale but must stay correct
            buf[0:3] += dev.t.tensor([[0.9 * dx[0]], [-0.7 * dx[1]], [0.8 * dx[2]]], device="cuda")
        host = buf.cpu().numpy()
        P = orc.HostParticles(**{k: host[i] for i, k in enumerate(orc.HostParticles.NAMES)})
    # by-product of the position push: the particles that left the periodic domain (pic_escape_list)
    geom = abi.make_geom(n, prob_lo, wl["prob_hi"])
    cap = P.np if pusher == abi.PUSHER_BORIS else 3          # 3: overflow -> the consumer sweeps everything
    esc_mem = dev.t.zeros(cap + 1, dtype=dev.t.int32, device="cuda")
    esc = abi.pic_escape_list()
    esc.count, esc.idx, esc.capacity = esc_mem.data_ptr(), esc_mem.data_ptr() + 4, cap
    for d in range(3):
        esc.lo[d], esc.hi[d] = prob_lo[d], wl["prob_hi"][d]
    for push_position in (1, 0):      # PushPX then PushP
        dev.ok(dev.L.pic_gather_push(C.byref(Pd), 0, P.np, E, B, abi.dbl3(dinv), abi.dbl3(xyzmin), abi.int3(lo),
                                     sp["q"], sp["m"], dt, nox, galerkin, pusher, push_position, bins,
                                     C.byref(esc), dev.stream))
        L.orc_gather_push(C.byref(P.soa), 0, P.np, orc.fab_array(F[0:3]), orc.fab_array(F[3:6]), abi.dbl3(dinv),
                          abi.dbl3(xyzmin), abi.int3(lo), sp["q"], sp["m"], dt, nox, galerkin, pusher, push_position)
        if push_position:
            dev.sync()
            got = buf.cpu().numpy()
            out = np.zeros(P.np, dtype=bool)
            for d in range(3):
                out |= (got[d] < prob_lo[d]) | (got[d] > wl["prob_hi"][d])
            listed = esc_mem.cpu().numpy()
            assert listed[0] == out.sum() > 0                 # PushP afterwards must not touch the list
            if cap >= listed[0]:
                assert np.array_equal(np.sort(listed[1:1 + listed[0]]), np.flatnonzero(out))
            # ... and the wrap that consumes it == amrex enforcePeriodic on every particle
            wrapped = buf.clone()
            Pw = abi.pic_soa.from_buffer_copy(Pd)
            for i, k in enumerate(orc.HostParticles.NAMES):
                setattr(Pw, k, wrapped[i].data_ptr())
            dev.ok(dev.L.pic_particles_wrap_listed(C.byref(Pw), C.byref(geom), C.byref(esc), dev.stream))
            dev.sync()
            Q = orc.HostParticles(**{k: got[i] for i, k in enumerate(orc.HostParticles.NAMES)})
            L.orc_wrap_periodic(C.byref(Q.soa), C.byref(geom))
            w = wrapped.cpu().numpy()
            assert np.array_equal(w[0], Q.x) and np.array_equal(w[1], Q.y) and np.array_equal(w[2], Q.z)
    dev.sync()
    assert int(esc_mem[0]) == listed[0]
    got = buf.cpu().numpy()
    for i, k in enumerate(("x", "y", "z")):
        assert np.max(np.abs(got[i] - getattr(P, k))) <= 1e-13 * lx, k
    for i, k in ((4, "ux"), (5, "uy"), (6, "uz")):
        assert rel_linf(got[i], getattr(P, k)) <= 1e-13, k


def add_background(dev, J, tens, seed):
    """J holds the oracle's deposition from zero.  Draw a random background B of the same magnitude, put it into the
    device arrays `tens` and add it to J, and return it: a kernel that stores where it should add is then wrong on
    every node it reaches."""
    rng = np.random.default_rng(500 + seed)
    scale = max(float(np.max(np.abs(f.a))) for f in J)
    B = [scale * rng.standard_normal(f.a.shape) for f in J]
    for f, b, t in zip(J, B, tens):
        f.a[...] += b
        t.copy_(dev.t.from_numpy(b))
    return B


def check_on_background(got, want, B):
    """|J_gpu - J_oracle| <= 1e-12 max|J_oracle - B|; nodes the oracle left at B (no stencil reaches them: a deposit adds
    nonzero values) keep B's bits on the GPU."""
    for c in range(3):
        dep = want[c] - B[c]
        assert np.max(np.abs(got[c] - want[c])) <= 1e-12 * np.max(np.abs(dep)), "j" + "xyz"[c]
        untouched = want[c] == B[c]
        assert np.any(untouched) and np.array_equal(got[c][untouched], B[c][untouched]), "j" + "xyz"[c]


@pytest.mark.parametrize("nox", [1, 2, 3])
@pytest.mark.parametrize("path", ["global", "tile", "tile_drifted", "tile_unsorted_bins",
                                  "runs", "runs_drifted", "runs_relativistic"])
def test_deposit_matches_oracle(orc, dev, nox, path):
    """global: order-agnostic kernel; tile*: shared-memory-block kernel; runs*: register-run kernel
    (the default with bins).  *_drifted: bins are stale; runs_relativistic: most particles change cell."""
    L = orc.lib()
    dev.L.pic_set_deposit_mode(1 if path.startswith("tile") else 0)
    kind = path
    path = {"runs": "tile", "runs_drifted": "tile_drifted", "runs_relativistic": "tile"}.get(path, path)
    n = (20, 16, 12)
    lx = 1e-5
    box_lo, box_hi = box(n)
    u_th = {"runs_relativistic": 3.0, "runs": 0.02, "tile": 0.02}.get(kind, 0.5)
    wl, sp = _particles(orc, n, (2, 2, 2), u_th, lx, shuffle=(path == "global"))
    prob_lo = wl["prob_lo"]
    dx = [(wl["prob_hi"][d] - prob_lo[d]) / n[d] for d in range(3)]
    dinv = [1.0 / v for v in dx]
    dt = 0.95 / (np.sqrt(sum(1.0 / v ** 2 for v in dx)) * workloads.C)
    ngJ = tuple(nox + 1 + (1 if path == "tile_drifted" else 0) for _ in range(3))
    xyzmin, lo = lower_corner(prob_lo, dx, box_lo, ngJ)
    J = [orc.HostFab(box_lo, box_hi, ngJ, abi.YEE_STAG[c]) for c in (6, 7, 8)]
    P = orc.HostParticles(**{k: sp[k] for k in orc.HostParticles.NAMES})
    arr, tens = dev.fabs(J)
    Jd = (abi.pic_fab * 3)(*arr)
    if path == "global":
        Pd, buf = dev.soa(P)
        bins = None
    else:
        tile = (8, 8, 8) if path != "tile_unsorted_bins" else (4, 8, 4)
        Pd, buf, bins_s, _, _ = _sorted_device_species(dev, P, n, prob_lo, wl["prob_hi"], tile=tile)
        bins = C.byref(bins_s)
        if path == "tile_drifted":
            buf[0:3] += dev.t.tensor([[0.8 * dx[0]], [-0.9 * dx[1]], [0.6 * dx[2]]], device="cuda")
        host = buf.cpu().numpy()
        P = orc.HostParticles(**{k: host[i] for i, k in enumerate(orc.HostParticles.NAMES)})
    L.orc_deposit_esirkepov(C.byref(P.soa), 0, P.np, orc.fab_array(J), abi.dbl3(dinv), abi.dbl3(xyzmin),
                            abi.int3(lo), sp["q"], dt, -0.5 * dt, nox)
    B = add_background(dev, J, tens, nox)
    dev.ok(dev.L.pic_deposit_esirkepov(C.byref(Pd), 0, P.np, Jd, abi.dbl3(dinv), abi.dbl3(xyzmin), abi.int3(lo),
                                       sp["q"], dt, -0.5 * dt, nox, bins, dev.stream))
    dev.sync()
    dev.L.pic_set_deposit_mode(0)
    check_on_background([t.cpu().numpy() for t in tens], [f.a for f in J], B)
    # Esirkepov identity (size independent): sum_cells J_x dV = sum_p q w (x_new - x_old)/dt
    gam = np.sqrt(1.0 + (P.ux ** 2 + P.uy ** 2 + P.uz ** 2) / workloads.C ** 2)
    dV = dx[0] * dx[1] * dx[2]
    for c, u in enumerate((P.ux, P.uy, P.uz)):
        lhs = float((tens[c].cpu() - dev.t.from_numpy(B[c])).sum()) * dV
        rhs = float(np.sum(sp["q"] * P.w * u / gam))
        assert lhs == pytest.approx(rhs, rel=1e-10, abs=1e-12 * float(np.sum(np.abs(sp["q"] * P.w * u / gam))))


@pytest.mark.parametrize("stag_comp", [0, 3, 6, 8])
def test_local_guard_cells_match_oracle(orc, dev, stag_comp):
    L = orc.lib()
    n = (12, 10, 14)
    box_lo, box_hi = box(n)
    geom = abi.make_geom(n, (0, 0, 0), (1, 1, 1))
    ng = (4, 4, 4)
    F = random_fields(orc, box_lo, box_hi, ng, 21, comps=[stag_comp])[0]
    # nodal duplicates (index N == index 0) hold equal values in a real run
    v = F.valid()
    for ax, d in ((2, 0), (1, 1), (0, 2)):
        if abi.YEE_STAG[stag_comp][d]:
            idx_lo = [slice(None)] * 3; idx_hi = [slice(None)] * 3
            idx_lo[ax] = 0; idx_hi[ax] = -1
            v[tuple(idx_hi)] = v[tuple(idx_lo)]
    # FillBoundary with fewer guards than allocated
    arr, tens = dev.fabs([F])
    for dim in range(3):
        dev.ok(dev.L.pic_fill_boundary_local(C.byref(arr[0]), dim, 2, C.byref(geom), dev.stream))
    dev.sync()
    L.orc_fill_boundary(orc.fab_array([F]), 1, abi.int3((2, 2, 2)), C.byref(geom))
    got = tens[0].cpu().numpy()
    sl = tuple(slice(2, -2) for _ in range(3))       # guards beyond ng = 2 are untouched by both
    assert np.array_equal(got[sl], F.a[sl])
    # SumBoundary(src = 3, dst = all)
    F2 = random_fields(orc, box_lo, box_hi, ng, 22, comps=[stag_comp])[0]
    arr, tens = dev.fabs([F2])
    for dim in range(3):
        dev.ok(dev.L.pic_sum_boundary_local(C.byref(arr[0]), dim, 3, C.byref(geom), dev.stream))
    for dim in range(3):
        dev.ok(dev.L.pic_fill_boundary_local(C.byref(arr[0]), dim, 4, C.byref(geom), dev.stream))
    dev.sync()
    L.orc_sum_boundary(orc.fab_array([F2]), 1, abi.int3((3, 3, 3)), abi.int3(ng), C.byref(geom))
    assert rel_linf(tens[0].cpu().numpy(), F2.a) <= 1e-14


@pytest.mark.parametrize("npass", [(1, 1, 1), (2, 1, 3), (0, 4, 0), (0, 0, 0)])
@pytest.mark.parametrize("stag_comp", [6, 8])
def test_bilinear_filter_matches_oracle(orc, dev, stag_comp, npass):
    """pic_apply_filter against the restated Filter::DoFilter over the grown box, zero padding at
    the array edge included; the GPU folds the mirrored reads into the weights, so the tolerance
    is a few ulp of the local magnitude (1e-14 relative to the field's max)."""
    L = orc.lib()
    n = (70, 9, 6)                                           # > one 64-wide block in i, ragged in j
    box_lo, box_hi = box(n)
    ng = (5, 5, 5)
    src = random_fields(orc, box_lo, box_hi, ng, 31, comps=[stag_comp])[0]
    dst = orc.HostFab(box_lo, box_hi, ng, abi.YEE_STAG[stag_comp])
    L.orc_apply_filter(C.byref(src.desc), C.byref(dst.desc), abi.int3(npass))
    arr, tens = dev.fabs([src, dst])
    tens[1].fill_(7.0)                                       # every point of dst must be overwritten
    dev.ok(dev.L.pic_apply_filter(C.byref(arr[0]), C.byref(arr[1]), abi.int3(npass), dev.stream))
    dev.sync()
    got = tens[1].cpu().numpy()
    assert rel_linf(got, dst.a) <= 1e-14
    assert np.array_equal(tens[0].cpu().numpy(), src.a)      # the source is read-only
    if npass == (0, 0, 0):
        assert np.array_equal(got, src.a)
    # in-place use is refused (the reference filters into a temporary)
    assert dev.L.pic_apply_filter(C.byref(arr[0]), C.byref(arr[0]), abi.int3(npass), dev.stream) != 0


def test_bilinear_filter_three_components_in_one_launch(orc, dev):
    """pic_apply_filter_multi (Jx, Jy, Jz of ApplyFilterJ in one launch; the streaming kernel of npass = (1,1,1)) against
    the oracle, on a box longer than one chunk of planes and ragged against the CTA; PIC-internal consistency: the
    single-component call gives the same bits."""
    L = orc.lib()
    n = (70, 21, 40)
    box_lo, box_hi = box(n)
    ng = (5, 5, 5)
    src = random_fields(orc, box_lo, box_hi, ng, 17, comps=[6, 7, 8])
    want = [orc.HostFab(box_lo, box_hi, ng, abi.YEE_STAG[c]) for c in (6, 7, 8)]
    for a, b in zip(src, want):
        L.orc_apply_filter(C.byref(a.desc), C.byref(b.desc), abi.int3((1, 1, 1)))
    arr, tens = dev.fabs(list(src) + want)
    for t in tens[3:]:
        t.fill_(7.0)
    dev.ok(dev.L.pic_apply_filter_multi((abi.pic_fab * 3)(*arr[0:3]), (abi.pic_fab * 3)(*arr[3:6]), 3, abi.int3((1, 1, 1)), dev.stream))
    dev.sync()
    for c in range(3):
        assert rel_linf(tens[3 + c].cpu().numpy(), want[c].a) <= 1e-14, c
    keep = tens[4].clone()
    dev.ok(dev.L.pic_apply_filter(C.byref(arr[1]), C.byref(arr[4]), abi.int3((1, 1, 1)), dev.stream))
    dev.sync()
    assert bool((tens[4] == keep).all())


def test_wrap_periodic_and_field_energy(orc, dev):
    L = orc.lib()
    n = (8, 8, 8)
    geom = abi.make_geom(n, (-1.0, -2.0, 0.0), (1.0, 2.0, 3.0))
    rng = np.random.default_rng(3)
    arrs = {k: rng.uniform(-1, 1, 5000) for k in ("w", "ux", "uy", "uz")}
    arrs["x"] = rng.uniform(-2.9, 2.9, 5000); arrs["y"] = rng.uniform(-5.9, 5.9, 5000); arrs["z"] = rng.uniform(-2.9, 5.9, 5000)
    arrs["x"][:3] = (-1.0, 1.0, 1.0 + 1e-17)
    P = orc.HostParticles(**arrs)
    Pd, buf = dev.soa(P)
    dev.ok(dev.L.pic_particles_wrap_periodic(C.byref(Pd), C.byref(geom), dev.stream))
    L.orc_wrap_periodic(C.byref(P.soa), C.byref(geom))
    dev.sync()
    got = buf.cpu().numpy()
    assert np.array_equal(got[0], P.x) and np.array_equal(got[1], P.y) and np.array_equal(got[2], P.z)
    F = random_fields(orc, (0, 0, 0), (7, 7, 7), (2, 2, 2), 9, comps=[0, 5, 2])
    arr, _ = dev.fabs(F)
    out = dev.t.zeros(1, dtype=dev.t.float64, device="cuda")
    for i, f in enumerate(F):
        dev.ok(dev.L.pic_sum_squares_unique(C.byref(arr[i]), C.byref(geom), out.data_ptr(), dev.stream))
        dev.sync()
        ref = L.orc_sum_squares_unique(orc.fab_array([f]), 1, C.byref(geom))
        assert float(out.cpu()) == pytest.approx(ref, rel=1e-13)


def test_preconditions_raise_like_the_reference_aborts(dev, orc):
    F = random_fields(orc, (0, 0, 0), (7, 7, 7), (0, 0, 0), 9, comps=range(6))
    arr, _ = dev.fabs(F)
    st = abi.pic_stencil(); st.algo = 0
    rc = dev.L.pic_evolve_b((abi.pic_fab * 3)(*arr[3:6]), (abi.pic_fab * 3)(*arr[0:3]), C.byref(st), 1e-15, dev.stream)
    assert rc != 0 and b"guard" in dev.L.pic_last_error()
    P = orc.HostParticles(**{k: np.zeros(4) for k in orc.HostParticles.NAMES})
    Pd, _ = dev.soa(P)
    rc = dev.L.pic_gather_push(C.byref(Pd), 0, 4, (abi.pic_fab * 3)(*arr[0:3]), (abi.pic_fab * 3)(*arr[3:6]),
                               abi.dbl3((1, 1, 1)), abi.dbl3((0, 0, 0)), abi.int3((0, 0, 0)), 1.0, 1.0, 1.0,
                               7, 1, 0, 1, None, None, dev.stream)
    assert rc != 0 and b"shape order" in dev.L.pic_last_error()


# ---------------------------------------------------------------------------------------------
def _run_both(orc, cuda, wl, nox, nsteps, **kw):
    from warpx_b200.engine import Simulation
    sim = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=nox, **kw)
    osim = orc.OracleSim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=nox, solver=kw.get("solver", 0),
                         pusher=kw.get("pusher", 0), use_filter=kw.get("use_filter", False),
                         filter_npass=kw.get("filter_npass", (1, 1, 1)))
    for s in wl["species"]:
        sim.add_species(s["name"], s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
        osim.add_species(s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    sim.Evolve(nsteps)
    osim.evolve(nsteps)
    cuda.cuda.synchronize()
    return sim, osim


def _match_particles(sim, osim, isp):
    """Pair GPU and oracle particles by the 64-bit particle id (the reference's idcpu): the engine
    carries it through every sort, the single-box oracle never reorders particles."""
    a = sim.species_numpy(isp, sort_by_id=True)
    b = osim.particles(isp)
    assert np.array_equal(a["id"], np.arange(len(b["x"])))
    return a, b


@pytest.mark.parametrize("use_bins", [True, False])
def test_langmuir_loop_golden_and_oracle(orc, cuda, golden, use_bins):
    """Config 1, 40 steps: WarpX's regression checksums (rtol 1e-9) and the oracle's fields."""
    wl = workloads.langmuir_3d()
    sim, osim = _run_both(orc, cuda, wl, 1, 40, use_bins=use_bins, sort_interval=4)
    g = golden["test_3d_langmuir_multi"]
    L = orc.lib()
    dx = sim.dx
    for c, name in enumerate(abi.COMP_NAMES):
        d, a = sim.field_numpy(c)
        hf = orc.HostFab(sim.box_lo, sim.box_hi, d.ng, abi.YEE_STAG[c], data=a)
        cs = L.orc_checksum_cell_centered(C.byref(hf.desc), abi.int3(sim.box_lo), abi.int3(sim.box_hi))
        assert abs(cs - g["lev=0"][name]) <= 1e-9 * abs(g["lev=0"][name]), name
        _, oa = osim.fab(c)
        # B is at round-off level in this electrostatic mode (|B| c / |E| ~ 1e-5): looser bound
        tol = 1e-9 if c not in (3, 4, 5) else 1e-7
        assert rel_linf(a[d.valid_slices()], oa[d.valid_slices()]) <= tol, name
    for isp, sname in enumerate(("electrons", "positrons")):
        P = sim.species_numpy(isp)
        vals = {"particle_position_x": P["x"], "particle_position_y": P["y"], "particle_position_z": P["z"],
                "particle_momentum_x": P["ux"] * workloads.M_E, "particle_momentum_z": P["uz"] * workloads.M_E,
                "particle_weight": P["w"]}
        for key, gv in g[sname].items():
            assert abs(float(np.sum(np.abs(vals[key]))) - gv) <= 1e-9 * abs(gv), (sname, key)
        A, B = _match_particles(sim, osim, isp)
        for k in ("x", "y", "z"):
            assert np.max(np.abs(A[k] - B[k])) / dx[0] <= 1e-10
        for k in ("ux", "uy", "uz"):
            assert np.max(np.abs(A[k] - B[k])) / workloads.C <= 1e-10
    e, b = sim.field_energy()
    eo, bo = osim.field_energy()
    assert e == pytest.approx(eo, rel=1e-10)
    assert b == pytest.approx(bo, rel=1e-7)     # B is at round-off level in this electrostatic mode


def test_plotfile_golden_checksums(orc, cuda, golden, tmp_path):
    """The reference's own regression loop, closed through files: config 1 for 40 steps on the GPU, dumped with
    warpx_b200.diagnostics.write_plotfile in the layout of `diag.format = plotfile`, read back the way
    Regression/Checksum/checksum.py reads a plotfile (tests/plotfile_reader.py stands in for yt), compared with every
    key of test_3d_langmuir_multi.json at WarpX's rtol 1e-9 (rho and part_per_cell are separate diagnostics functors)."""
    from warpx_b200 import diagnostics
    from warpx_b200.engine import Simulation
    import plotfile_reader
    wl = workloads.langmuir_3d()
    sim = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=1, sort_interval=4)
    for s in wl["species"]:
        sim.add_species(s["name"], s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    sim.Evolve(40)
    cuda.cuda.synchronize()
    root = diagnostics.write_plotfile(sim, str(tmp_path / "diags" / "plt"))
    got = plotfile_reader.checksums(root, species=("electrons", "positrons"))
    g = golden["test_3d_langmuir_multi"]
    for name in abi.COMP_NAMES:
        assert abs(got["lev=0"][name] - g["lev=0"][name]) <= 1e-9 * abs(g["lev=0"][name]), name
    for sname in ("electrons", "positrons"):
        for key, gv in g[sname].items():
            assert abs(got[sname][key] - gv) <= 1e-9 * abs(gv), (sname, key)
    sim.close()


@pytest.mark.parametrize("solver,pusher,native", [(abi.SOLVER_YEE, abi.PUSHER_BORIS, True),
                                                  (abi.SOLVER_YEE, abi.PUSHER_BORIS, False),
                                                  (abi.SOLVER_CKC, abi.PUSHER_VAY, True)])
def test_order3_loop_matches_oracle(orc, cuda, solver, pusher, native):
    """Config 2 / 3 physics (order-3 Esirkepov, 8 ppc, Yee or CKC) at 32^3, 10 steps, with a
    Langmuir perturbation on top of the thermal spread so that the fields are well above noise."""
    wl = workloads.uniform_plasma_3d(n=32, ppc=(2, 2, 2), u_th=0.01, lx=5e-6, perturbation=0.01)
    # native: the library's C++ step driver (csrc/engine.cu); otherwise the Python sequencer
    sim, osim = _run_both(orc, cuda, wl, 3, 10, solver=solver, pusher=pusher, sort_interval=4, native_driver=native)
    assert bool(sim.native) == native
    for c in range(9):
        d, a = sim.field_numpy(c)
        _, oa = osim.fab(c)
        tol = 1e-9 if c not in (3, 4, 5) else 1e-7
        assert rel_linf(a[d.valid_slices()], oa[d.valid_slices()]) <= tol, abi.COMP_NAMES[c]
    e, b = sim.field_energy()
    eo, bo = osim.field_energy()
    assert e == pytest.approx(eo, rel=1e-10) and b == pytest.approx(bo, rel=1e-8)
    A, B = _match_particles(sim, osim, 0)
    for k in ("x", "y", "z"):
        assert np.max(np.abs(A[k] - B[k])) / sim.dx[0] <= 1e-10
    for k in ("ux", "uy", "uz"):
        assert np.max(np.abs(A[k] - B[k])) / workloads.C <= 1e-10


@pytest.mark.parametrize("n,deposit_mode", [(128, abi.PIC_DEPOSIT_RUNS), (128, abi.PIC_DEPOSIT_CELLS), (256, abi.PIC_DEPOSIT_CELLS)])
def test_config2_at_benchmark_size_matches_oracle(orc, cuda, n, deposit_mode):
    """BASELINE configs[1] itself -- same cell size (40 um / 256), 8 ppc on the lattice, u_th = 0.01 c from the
    counter-based generator, Yee, Boris, order 3, cell sort every 4 steps -- for the first 10 steps against the
    oracle (SURVEY.md 8d: "parity on first 10"), at the tolerance north_star states: fields 1e-9, field energy
    1e-10, every particle by id x/dx and u/c 1e-10.  128^3 (2 s of oracle time); 256^3, the full benchmark
    box, when PIC_TEST_FULL_SIZE=1 (a minute of oracle time and ~40 GB of host memory)."""
    import os
    if n == 256 and os.environ.get("PIC_TEST_FULL_SIZE", "0") != "1":
        pytest.skip("set PIC_TEST_FULL_SIZE=1 for the 256^3 run")
    from warpx_b200.lib import lib
    wl = workloads.uniform_plasma_3d(n=n, ppc=(2, 2, 2), u_th=0.01, lx=40.0e-6 * n / 256.0, perturbation=0.01)
    lib().pic_set_deposit_mode(deposit_mode)
    try:
        sim, osim = _run_both(orc, cuda, wl, 3, 10, sort_interval=4)
    finally:
        lib().pic_set_deposit_mode(abi.PIC_DEPOSIT_RUNS)
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
    sim.close()


@pytest.mark.parametrize("native,npass", [(True, (1, 1, 1)), (False, (1, 1, 1)), (True, (2, 1, 3))])
def test_filtered_loop_matches_oracle(orc, cuda, native, npass):
    """warpx.use_filter = 1 (the reference's default): J gets npass more guard cells, the bilinear
    filter runs before SumBoundaryJ.  Same bar as the unfiltered order-3 loop."""
    wl = workloads.uniform_plasma_3d(n=32, ppc=(2, 2, 2), u_th=0.01, lx=5e-6, perturbation=0.01)
    sim, osim = _run_both(orc, cuda, wl, 3, 10, sort_interval=4, native_driver=native, use_filter=True,
                          filter_npass=npass)
    assert bool(sim.native) == native
    assert sim.ng_J == osim.guards()["ng_J"] == [4 + v for v in npass]
    for c in range(9):
        d, a = sim.field_numpy(c)
        _, oa = osim.fab(c)
        tol = 1e-9 if c not in (3, 4, 5) else 1e-7
        assert rel_linf(a[d.valid_slices()], oa[d.valid_slices()]) <= tol, abi.COMP_NAMES[c]
    A, B = _match_particles(sim, osim, 0)
    for k in ("x", "y", "z"):
        assert np.max(np.abs(A[k] - B[k])) / sim.dx[0] <= 1e-10
    for k in ("ux", "uy", "uz"):
        assert np.max(np.abs(A[k] - B[k])) / workloads.C <= 1e-10


def test_full_size_properties(cuda):
    """BASELINE config-2 size (256^3, 8 ppc, order 3) through size-independent properties:
    the Esirkepov identity sum J dV = sum q w v, div B = 0 after the solve, particle count and
    weight conservation through sort + wrap, and field-energy growth bounded (no blow-up)."""
    from warpx_b200.engine import Simulation
    t = cuda
    free, _ = t.cuda.mem_get_info()
    n = 256 if free > 40e9 else 128
    wl = workloads.uniform_plasma_3d(n=n, ppc=(2, 2, 2), u_th=0.01)
    sim = Simulation(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=3, sort_interval=4)
    s = wl["species"][0]
    sp = sim.add_species(s["name"], s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
    np0, w0 = sp.np, float(sp.array("w").sum())
    sim.Evolve(5, synchronize_last=False)
    t.cuda.synchronize()
    assert sp.np == np0 and float(sp.array("w").sum()) == pytest.approx(w0, rel=1e-14)
    # J of the last step (valid points, duplicates counted once) vs particle momenta at u^{n+1/2}
    dV = sim.dx[0] * sim.dx[1] * sim.dx[2]
    u = [sp.array(k) for k in ("ux", "uy", "uz")]
    gam = t.sqrt(1.0 + (u[0] ** 2 + u[1] ** 2 + u[2] ** 2) / workloads.C ** 2)
    for c in range(3):
        d = sim.fab[6 + c]
        v = sim.data[6 + c][d.valid_slices()]
        # drop the upper duplicate layer along the nodal directions
        sl = tuple(slice(0, -1) if d.stag[dd] else slice(None) for dd in (2, 1, 0))
        lhs = float(v[sl].sum()) * dV
        rhs = float((s["q"] * sp.array("w") * u[c] / gam).sum())
        scale = float((abs(s["q"]) * sp.array("w") * u[c].abs() / gam).sum())
        assert abs(lhs - rhs) <= 1e-9 * scale
    # div B = 0 to round-off on the Yee grid
    bx, by, bz = (sim.data[3 + c] for c in range(3))
    g = sim.ng_EB[0]
    N = n
    BX = bx[g:g + N, g:g + N, g:g + N + 1]
    BY = by[g:g + N, g:g + N + 1, g:g + N]
    BZ = bz[g:g + N + 1, g:g + N, g:g + N]
    div = (BX[:, :, 1:] - BX[:, :, :-1]) / sim.dx[0] + (BY[:, 1:, :] - BY[:, :-1, :]) / sim.dx[1] \
        + (BZ[1:, :, :] - BZ[:-1, :, :]) / sim.dx[2]
    scale = float(BX.abs().max()) / sim.dx[0] + 1e-300
    assert float(div.abs().max()) <= 1e-9 * scale
    e, b = sim.field_energy()
    assert np.isfinite(e) and np.isfinite(b) and e > 0


def test_two_gpu_halo_and_migration(cuda):
    """N > 1 on real GPUs (skipped on a single-GPU box): tests/multi_gpu_check.py under torchrun."""
    import os
    import subprocess
    import sys
    if cuda.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29533",
                        os.path.join(root, "tests", "multi_gpu_check.py")], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "MULTI_GPU_CHECK PASS" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
