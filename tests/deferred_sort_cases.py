"""TEST INFRASTRUCTURE -- the deferred cell sort through the C ABI, written once for two libraries: the device library
(tests/test_gpu_deferred_sort.py) and the same sources under host emulation (tests/test_deferred_sort_host.py).

The sort is two halves (pic_sort_index_by_cell: cell_start + permutation; pic_sort_apply_permutation: the move) and
pic_gather_push_permuted carries out the move inside the push.  Gather + push is a function of one particle and the
fields, so the carried move is checked bit for bit by particle id."""
import ctypes as C

import numpy as np

import particle_sets as ps
from warpx_b200 import abi

NAMES = ps.NAMES
STAGGERINGS = {"yee": abi.YEE_STAG, "nodal": [(1, 1, 1)] * 6}


class Backend:
    """One library and the memory it works on: torch tensors on `device`, pointers for the C ABI."""

    def __init__(self, torch, L, device):
        self.t, self.L, self.device = torch, L, torch.device(device)
        L.pic_set_error_mode(abi.PIC_ERR_RETURN)

    @property
    def stream(self):
        return self.t.cuda.current_stream().cuda_stream if self.device.type == "cuda" else None

    def sync(self):
        if self.device.type == "cuda":
            self.t.cuda.synchronize()

    def ok(self, rc):
        assert rc == 0, self.L.pic_last_error().decode()

    def particles(self, arrays, ids):
        buf = self.t.stack([self.t.from_numpy(np.ascontiguousarray(arrays[k])) for k in NAMES]).to(self.device)
        return Particles(self, buf, self.t.from_numpy(np.asarray(ids, dtype=np.int64)).to(self.device))

    def ints(self, n):
        return self.t.zeros(n, dtype=self.t.int32, device=self.device)


class Particles:
    def __init__(self, be, buf, ids):
        self.be, self.buf, self.ids = be, buf, ids
        self.np = buf.shape[1]
        self.soa = abi.pic_soa()
        for i, k in enumerate(NAMES):
            setattr(self.soa, k, buf[i].data_ptr())
        self.soa.idcpu = ids.data_ptr()
        self.soa.np = self.np

    def like(self):
        t = self.be.t
        return Particles(self.be, t.full_like(self.buf, float("nan")), t.full_like(self.ids, -1))

    def numpy(self):
        self.be.sync()
        out = {k: self.buf[i].cpu().numpy() for i, k in enumerate(NAMES)}
        out["id"] = self.ids.cpu().numpy()
        return out


def by_id(p):
    order = np.argsort(p["id"], kind="stable")
    return {k: v[order] for k, v in p.items()}


class Sorter:
    """Bins, workspace and geometry of the box of particle set s."""

    def __init__(self, be, s):
        self.be, self.s = be, s
        self.bins = abi.pic_bins()
        for d in range(3):
            self.bins.box_lo[d], self.bins.box_hi[d], self.bins.tile[d] = s.box_lo[d], s.box_hi[d], ps.TILE
        self.nb = be.L.pic_bins_count(self.bins.box_lo, self.bins.box_hi, self.bins.tile)
        self.cell_start = be.ints(self.nb + 1)
        self.work = be.t.zeros(be.L.pic_sort_workspace_bytes(s.np, self.nb), dtype=be.t.uint8, device=be.device)
        self.bins.cell_start = self.cell_start.data_ptr()
        self.bins.np_binned = s.np
        self.geom = abi.make_geom(s.n, s.prob_lo, s.prob_hi)

    def index(self, P):
        src = C.c_void_p()
        self.be.ok(self.be.L.pic_sort_index_by_cell(C.byref(P.soa), C.byref(self.geom), C.byref(self.bins),
                                                    self.work.data_ptr(), C.byref(src), self.be.stream))
        return src

    def apply(self, P, src):
        out = P.like()
        self.be.ok(self.be.L.pic_sort_apply_permutation(C.byref(P.soa), C.byref(out.soa), src, self.be.stream))
        return out

    def whole(self, P):
        out = P.like()
        self.be.ok(self.be.L.pic_sort_particles_by_cell(C.byref(P.soa), C.byref(out.soa), C.byref(self.geom),
                                                        C.byref(self.bins), self.work.data_ptr(), self.be.stream))
        return out


def shuffled(s, seed):
    """The set's particles in an order that is sorted except for a tenth of them (what a sort finds after a few
    steps), with ids."""
    p = s.arrays()
    rng = np.random.default_rng(seed)
    order = np.arange(s.np)
    movers = rng.choice(s.np, max(s.np // 10, min(s.np, 2)), replace=False)
    order[np.sort(movers)] = movers
    return {k: v[order] for k, v in p.items()}, rng.permutation(s.np) + 1000


def check_index_apply_is_the_sort(be, name):
    """index + apply gives what the one-call sort gives: same cell_start, the same particles in every cell."""
    s = ps.get(name)
    arrays, ids = shuffled(s, 11)
    P = be.particles(arrays, ids)
    so = Sorter(be, s)
    whole = so.whole(P).numpy()
    cs_whole = so.cell_start.cpu().numpy().copy()
    so.cell_start.zero_()
    halves = so.apply(P, so.index(P)).numpy()
    cs = so.cell_start.cpu().numpy()
    assert np.array_equal(cs, cs_whole) and cs[0] == 0 and cs[-1] == s.np
    assert np.array_equal(P.numpy()["id"], ids)                              # the input is left alone
    bin_of_slot = np.searchsorted(cs, np.arange(s.np), side="right") - 1
    expect = ps.bin_of(halves["x"], halves["y"], halves["z"], s.origin, s.dx, s.n)
    assert np.array_equal(bin_of_slot, expect)
    for p in (whole, halves):                                               # order inside a cell is free
        o = np.lexsort((p["id"], bin_of_slot))
        for k in p:
            p[k] = p[k][o]
    for k in whole:
        assert np.array_equal(whole[k], halves[k]), k


def _fields(be, orc, s, ng, stag):
    rng = np.random.default_rng(5)
    keep, arr = [], (abi.pic_fab * 6)()
    for c in range(6):
        f = orc.HostFab(s.box_lo, s.box_hi, ng, stag[c])
        f.a[...] = (1e10 if c < 3 else 30.0) * rng.standard_normal(f.a.shape)
        d = be.t.from_numpy(f.a).to(be.device)
        arr[c] = f.desc
        arr[c].p = d.data_ptr()
        keep.append(d)
    return (abi.pic_fab * 3)(*arr[0:3]), (abi.pic_fab * 3)(*arr[3:6]), keep


def _escape_list(be, s, cap):
    mem = be.ints(cap + 1)
    esc = abi.pic_escape_list()
    esc.count, esc.idx, esc.capacity = mem.data_ptr(), mem.data_ptr() + 4, cap
    for d in range(3):
        esc.lo[d], esc.hi[d] = s.prob_lo[d], s.prob_hi[d]
    return esc, mem


def _escaped_ids(be, mem, P):
    be.sync()
    m = mem.cpu().numpy()
    assert m[0] <= len(m) - 1
    return np.sort(P.numpy()["id"][m[1:1 + m[0]]])


def check_permuting_push_is_apply_then_push(be, orc, name, nox, galerkin, pusher, stag, stale_bins=False):
    """pic_gather_push_permuted == pic_sort_apply_permutation + pic_gather_push, bit for bit by id, and both list the
    same escaped particles.  stale_bins: the permutation leads to the set's own order, whose bins are a few steps old
    (particles outside their bin's cell, row and supercell: the kernel's hand-on lists, which a fresh sort leaves
    almost empty)."""
    s = ps.get(name)
    so = Sorter(be, s)
    if stale_bins:
        rng = np.random.default_rng(3)
        where = rng.permutation(s.np)                   # particle `slot` of the set lies at where[slot] of the input
        arrays, ids = s.arrays(), np.arange(s.np) + 1000
        P = be.particles({k: _scatter(v, where) for k, v in arrays.items()}, _scatter(ids, where))
        so.cell_start.copy_(be.t.from_numpy(s.cell_start.astype(np.int32)))
        src_t = be.t.from_numpy(where.astype(np.int32)).to(be.device)
        src = C.c_void_p(src_t.data_ptr())
    else:
        arrays, ids = shuffled(s, 12)
        P = be.particles(arrays, ids)
        src = so.index(P)
    ng = (4, 4, 4)
    xyzmin, lo = s.corner(ng)
    E, B, keep = _fields(be, orc, s, ng, STAGGERINGS[stag])
    geo = (abi.dbl3(s.dinv), abi.dbl3(xyzmin), abi.int3(lo), s.q, s.m, s.dt, nox, galerkin, pusher)
    # the two-pass way
    A = so.apply(P, src)
    esc_a, mem_a = _escape_list(be, s, s.np)
    be.ok(be.L.pic_gather_push(C.byref(A.soa), 0, A.np, E, B, *geo, 1, C.byref(so.bins), C.byref(esc_a), be.stream))
    # the carried move
    before = P.numpy()
    Bp = P.like()
    esc_b, mem_b = _escape_list(be, s, s.np)
    be.ok(be.L.pic_gather_push_permuted(C.byref(P.soa), C.byref(Bp.soa), src, E, B, *geo, C.byref(so.bins),
                                        C.byref(esc_b), be.stream))
    a, b = A.numpy(), Bp.numpy()
    assert np.array_equal(np.sort(b["id"]), np.sort(ids))
    for k in a:
        assert np.array_equal(a[k], b[k]), k            # same slots, not only the same particles
    after = P.numpy()
    for k in before:
        assert np.array_equal(before[k], after[k]), k   # the source buffer is read only
    moved = by_id(b)
    start = by_id(before)
    assert np.array_equal(moved["w"], start["w"]) and not np.array_equal(moved["x"], start["x"])
    assert np.array_equal(_escaped_ids(be, mem_a, A), _escaped_ids(be, mem_b, Bp))


def _scatter(v, where):
    out = np.empty_like(v)
    out[where] = v
    return out
