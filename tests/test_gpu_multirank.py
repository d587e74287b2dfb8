"""GPU tests (-m gpu): the multi-rank paths of the library on ONE device.

Kernel level: the halo slab pack / unpack (pic_halo_*, every mode, thin and wide boxes), the local multi-component
sweeps, the particle migration kernels (classify, pack, unpack, the candidate list) and the antenna's owned weights,
each against a numpy restatement of what it should do.  Engine level: brick and slab decompositions of the C++ step
driver, the ranks being THREADS of this process, each driving warpx_b200.engine.Simulation on its own CUDA stream and
exchanging through the device build of the NCCL stand-in (tests/host_harness/fake_nccl.cpp, -DPIC_STANDIN_DEVICE),
against the single-box oracle and WarpX's golden checksums -- the scenarios of test_host_multirank.py, here with real
launch geometry, device memory and concurrent thread blocks.  TEST INFRASTRUCTURE; no product code runs this way."""
import ctypes as C
import os
import threading

import numpy as np
import pytest

from warpx_b200 import abi, parallel, workloads

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]


@pytest.fixture(scope="module")
def L(cuda):
    from warpx_b200.lib import lib
    L = lib()
    L.pic_set_error_mode(abi.PIC_ERR_RETURN)
    return L


def _bits(a):
    return np.ascontiguousarray(a).view(np.int64)


def _same_bits(a, b):
    return np.array_equal(_bits(a), _bits(b))


# ---------------------------------------------------------------------------------------------------------------------
# Ranks as threads on one GPU
# ---------------------------------------------------------------------------------------------------------------------
def _harness():
    from host_harness import harness
    return harness


class DeviceThreadDist:
    """The torch.distributed calls Simulation makes, between threads that each work on their own stream.  Tensors pass
    through the host: a device-side clone would be read by another rank's stream before it is finished."""

    class ReduceOp:
        SUM, MAX = "sum", "max"

    def __init__(self, shared, rank):
        self.shared, self.rank = shared, rank

    def get_rank(self):
        return self.rank

    def get_world_size(self):
        return self.shared.world

    def barrier(self):
        self.shared.barrier.wait()

    def broadcast(self, tensor, src):
        sh = self.shared
        if self.rank == src:
            sh.slots[src] = tensor.cpu().clone()
        sh.barrier.wait()
        if self.rank != src:
            tensor.copy_(sh.slots[src])
        sh.barrier.wait()

    def all_reduce(self, tensor, op=None):
        import torch
        sh = self.shared
        sh.slots[self.rank] = tensor.cpu().clone()
        sh.barrier.wait()
        stack = torch.stack(sh.slots)
        res = stack.max(dim=0).values if op == self.ReduceOp.MAX else stack.sum(dim=0)
        sh.barrier.wait()
        tensor.copy_(res)


_STANDIN = None


def standin():
    """The device stand-in (built once per process)."""
    global _STANDIN
    if _STANDIN is None:
        S = C.CDLL(_harness().build_device_nccl())
        for name in ("standin_sends", "standin_recvs", "standin_allreduces"):
            getattr(S, name).restype = C.c_long
        _STANDIN = S
    return _STANDIN


def run_ranks(world, fn):
    """fn(rank, dist) on `world` threads, each under its own torch.cuda.Stream() (torch's current stream is per
    thread); returns the results, re-raises the first exception.  Checks that the ranks exchanged through the stand-in."""
    import torch
    from warpx_b200.lib import lib
    S = standin()
    lib()
    sends0, ar0 = S.standin_sends(), S.standin_allreduces()
    device = torch.cuda.current_device()
    shared = _harness().ThreadDist._Shared(world)
    out, err = [None] * world, [None] * world

    def target(r):
        try:
            torch.cuda.set_device(device)
            stream = torch.cuda.Stream()
            with torch.cuda.stream(stream):
                out[r] = fn(r, DeviceThreadDist(shared, r))
            stream.synchronize()
        except BaseException as e:       # noqa: BLE001 -- reported to the caller below
            err[r] = e
            shared.barrier.abort()
    # The library binds PIC_NCCL_LIBRARY at its first communicator call and keeps the handle (nothing in this process
    # may have bound another NCCL before); the variable is not left behind for child processes.
    before = os.environ.get("PIC_NCCL_LIBRARY")
    os.environ["PIC_NCCL_LIBRARY"] = S._name
    try:
        threads = [threading.Thread(target=target, args=(r,)) for r in range(world)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
    finally:
        if before is None:
            del os.environ["PIC_NCCL_LIBRARY"]
        else:
            os.environ["PIC_NCCL_LIBRARY"] = before
    torch.cuda.synchronize()
    for e in err:
        if e is not None and not isinstance(e, threading.BrokenBarrierError):
            raise e
    for e in err:
        if e is not None:
            raise e
    sends, ar = S.standin_sends() - sends0, S.standin_allreduces() - ar0
    print(f"[device NCCL stand-in] {world} ranks: {sends} sends, {ar} all-reduces")
    assert sends > 0, "the ranks did not exchange through the stand-in"
    return out


class DeviceRanks:
    """What the scenarios of test_host_multirank.py take of the host harness (`hh`), on the device: the real
    Simulation, the real library, threads on one GPU."""

    @staticmethod
    def host_simulation_class():
        from warpx_b200.engine import Simulation
        return Simulation

    @staticmethod
    def host_library():
        from warpx_b200.lib import lib
        return lib()

    run_ranks = staticmethod(run_ranks)


@pytest.fixture(scope="module")
def ranks(L):
    return DeviceRanks()


@pytest.fixture(scope="module")
def scenarios():
    import test_host_multirank
    return test_host_multirank


# ---------------------------------------------------------------------------------------------------------------------
# Halo slabs: pic_halo_pack / pic_halo_unpack and the _multi forms against a numpy restatement of slab_range
# ---------------------------------------------------------------------------------------------------------------------
HALO_COMPS = (0, 4, 6, 8)                       # Ex, By, jx, jz: every staggering along every axis
# (box_lo, box_hi, allocated guards): 8 cells with 5 guards -- SumBoundary's two slabs overlap -- and a wide box
HALO_BOXES = {"thin": ((8, 16, 0), (15, 23, 7), (5, 5, 5)),
              "wide": ((0, 8, 4), (23, 23, 19), (3, 4, 5))}


def np_slab_range(d, dim, side, ng, mode, unpack):
    """(first global index, count) along dim of the slab exchanged with the neighbour on `side` (halo.cu: slab_range)."""
    st = d.stag[dim]
    lc = d.lo[dim] + d.ng[dim]                 # first cell
    hc = d.hi[dim] - d.ng[dim] - st            # last cell
    if mode == 0:                               # copy: valid layers out, guards in
        return ((hc + 1 - ng) if side else (lc + st)) if not unpack else ((hc + 1 + st) if side else (lc - ng)), ng
    if mode == 1:                               # sum: guards (+ shared node) out, added into valid
        return ((hc + 1) if side else (lc - ng)) if not unpack else ((hc + 1 - ng) if side else lc), ng + st
    return ((hc + 1 - ng) if side else (lc - ng)), 2 * ng + st      # sum + refresh: the whole overlap zone


def np_slab(d, dim, first, count):
    """numpy index [k, j, i] of a slab: [first, first + count) along dim, the allocated extent across."""
    sl = [slice(None)] * 3
    sl[2 - dim] = slice(first - d.lo[dim], first - d.lo[dim] + count)
    return tuple(sl)


def halo_ok(d, dim, ng, mode):
    """Whether the library accepts the slab (ng <= cells; the fused mode needs 2 ng + stag <= cells)."""
    cells = d.hi[dim] - d.lo[dim] + 1 - 2 * d.ng[dim] - d.stag[dim]
    return 2 * ng + d.stag[dim] <= cells if mode == 2 else ng <= cells


def halo_ngs(ngalloc, dim):
    return sorted({0, 1, 4, ngalloc[dim]} & set(range(ngalloc[dim] + 1)))


class DevFabs:
    """Components on one box: numpy start values, device copies, descriptors."""

    def __init__(self, torch, box, comps, seed):
        lo, hi, ng = box
        rng = np.random.default_rng(seed)
        self.torch, self.descs, self.start, self.dev = torch, [], [], []
        for c in comps:
            d = abi.make_fab(None, lo, hi, ng, abi.YEE_STAG[c])
            a = rng.standard_normal(d.shape)
            t = torch.from_numpy(a).cuda()
            d.p = t.data_ptr()
            self.descs.append(d)
            self.start.append(a)
            self.dev.append(t)
        self.arr = (abi.pic_fab * len(self.descs))(*self.descs)

    def reset(self):
        for a, t in zip(self.start, self.dev):
            t.copy_(self.torch.from_numpy(a))

    def now(self, k):
        self.torch.cuda.synchronize()
        return self.dev[k].cpu().numpy()


def _stream(torch):
    return torch.cuda.current_stream().cuda_stream


def _sentinel_buf(torch, n, pad=9):
    return torch.full((n + pad,), 1.0e300, dtype=torch.float64, device="cuda")


@pytest.mark.parametrize("which", sorted(HALO_BOXES))
def test_halo_pack_unpack_one_side_match_numpy(L, cuda, which):
    """pic_halo_pack writes exactly pic_halo_slab_count doubles, i fastest, and nothing else; pic_halo_unpack copies
    (mode 0) / adds (mode 1) into its slab only, every other point keeps its bits.  Every staggering, axis and side;
    ng from 0 to the allocated width."""
    torch = cuda
    box = HALO_BOXES[which]
    F = DevFabs(torch, box, HALO_COMPS, seed=11)
    rng = np.random.default_rng(12)
    s = _stream(torch)
    cases = 0
    for k, c in enumerate(HALO_COMPS):
        d = F.descs[k]
        for dim in range(3):
            for ng in halo_ngs(box[2], dim):
                for mode in (0, 1):
                    for side in (0, 1):
                        what = (abi.COMP_NAMES[c], dim, ng, mode, side)
                        assert halo_ok(d, dim, ng, mode)
                        first, count = np_slab_range(d, dim, side, ng, mode, 0)
                        sl = np_slab(d, dim, first, count)
                        n = int(np.prod(F.start[k][sl].shape))
                        assert L.pic_halo_slab_count(C.byref(d), dim, ng, mode) == n, what
                        buf = _sentinel_buf(torch, n)
                        assert L.pic_halo_pack(C.byref(d), dim, side, ng, mode, buf.data_ptr(), s) == 0, L.pic_last_error()
                        got = buf.cpu().numpy()
                        assert _same_bits(got[:n], F.start[k][sl].ravel()), what
                        assert np.all(got[n:] == 1.0e300), what
                        assert _same_bits(F.now(k), F.start[k]), what                     # pack reads only
                        first, count = np_slab_range(d, dim, side, ng, mode, 1)
                        sl = np_slab(d, dim, first, count)
                        vals = rng.standard_normal(n)
                        buf = torch.from_numpy(vals).cuda()
                        assert L.pic_halo_unpack(C.byref(d), dim, side, ng, mode, buf.data_ptr(), s) == 0, L.pic_last_error()
                        want = F.start[k].copy()
                        if mode == 0:
                            want[sl] = vals.reshape(want[sl].shape)
                        else:
                            want[sl] += vals.reshape(want[sl].shape)
                        assert _same_bits(F.now(k), want), what
                        F.reset()
                        cases += 1
    assert cases > 100


@pytest.mark.parametrize("which", sorted(HALO_BOXES))
def test_halo_multi_matches_one_side_calls(L, cuda, which):
    """pic_halo_pack_multi / pic_halo_unpack_multi over Ex, By, jx, jz at once: the packed messages are the
    components' slabs back to back; the unpack equals numpy's low side then high side and -- modes 0 and 1 -- the
    one-side calls run low then high, bit for bit.  On the thin box SumBoundary's two slabs share points (cells <=
    2 ng + stag - 1): a launch in which both sides' threads add into them would lose or reorder adds.  The fused
    mode 2 is refused where the box is too thin for it, and the arrays are left alone."""
    torch = cuda
    box = HALO_BOXES[which]
    F = DevFabs(torch, box, HALO_COMPS, seed=21)
    G = DevFabs(torch, box, HALO_COMPS, seed=21)
    rng = np.random.default_rng(22)
    s = _stream(torch)
    nf = len(HALO_COMPS)
    overlapped = 0
    for dim in range(3):
        for ng in halo_ngs(box[2], dim):
            for mode in (0, 1, 2):
                what = (dim, ng, mode)
                ok = all(halo_ok(d, dim, ng, mode) for d in F.descs)
                counts = [L.pic_halo_slab_count(C.byref(d), dim, ng, mode) for d in F.descs]
                total = sum(counts)
                bufs = [_sentinel_buf(torch, total) for _ in range(2)]
                rc = L.pic_halo_pack_multi(F.arr, nf, dim, ng, mode, bufs[0].data_ptr(), bufs[1].data_ptr(), s)
                if not ok:
                    assert rc != 0 and mode == 2, what
                    vals = [torch.zeros(total + 1, dtype=torch.float64, device="cuda") for _ in range(2)]
                    assert L.pic_halo_unpack_multi(F.arr, nf, dim, ng, mode, vals[0].data_ptr(), vals[1].data_ptr(), s) != 0
                    assert b"too thin" in L.pic_last_error()
                    assert all(_same_bits(F.now(k), F.start[k]) for k in range(nf)), what
                    continue
                assert rc == 0, L.pic_last_error()
                for side in (0, 1):
                    got = bufs[side].cpu().numpy()
                    want = np.concatenate([F.start[k][np_slab(F.descs[k], dim, *np_slab_range(F.descs[k], dim, side, ng, mode, 0))].ravel()
                                           for k in range(nf)])
                    assert len(want) == total and _same_bits(got[:total], want), what + (side,)
                    assert np.all(got[total:] == 1.0e300), what
                assert all(_same_bits(F.now(k), F.start[k]) for k in range(nf)), what
                # unpack: numpy low then high
                vals = [rng.standard_normal(total) for _ in range(2)]
                dv = [torch.from_numpy(v).cuda() for v in vals]
                assert L.pic_halo_unpack_multi(F.arr, nf, dim, ng, mode, dv[0].data_ptr(), dv[1].data_ptr(), s) == 0, L.pic_last_error()
                want = [a.copy() for a in F.start]
                shared = False
                for side in (0, 1):
                    off = 0
                    for k in range(nf):
                        d = F.descs[k]
                        sl = np_slab(d, dim, *np_slab_range(d, dim, side, ng, mode, 1))
                        v = vals[side][off:off + counts[k]].reshape(want[k][sl].shape)
                        if mode == 0:
                            want[k][sl] = v
                        else:
                            want[k][sl] += v
                        off += counts[k]
                for k in range(nf):
                    d = F.descs[k]
                    f0, n0 = np_slab_range(d, dim, 0, ng, mode, 1)
                    f1, n1 = np_slab_range(d, dim, 1, ng, mode, 1)
                    shared |= n0 > 0 and n1 > 0 and f0 + n0 > f1
                for k in range(nf):
                    assert _same_bits(F.now(k), want[k]), what + (abi.COMP_NAMES[HALO_COMPS[k]], "multi vs numpy")
                overlapped += shared
                # the one-side calls, low side then high side, on the second copy
                if mode != 2:
                    for side in (0, 1):
                        off = 0
                        for k in range(nf):
                            assert L.pic_halo_unpack(C.byref(G.descs[k]), dim, side, ng, mode, dv[side][off:].data_ptr(), s) == 0
                            off += counts[k]
                    for k in range(nf):
                        assert _same_bits(G.now(k), F.now(k)), what + (abi.COMP_NAMES[HALO_COMPS[k]], "multi vs one side")
                F.reset()
                G.reset()
    if which == "thin":
        assert overlapped > 0                   # the regime of the two-launch unpack was reached


def test_halo_refuses_slab_wider_than_box(L, cuda):
    """ng larger than the box's cells (modes 0 and 1) would reach through the valid points into the guards of the
    other face: every entry point refuses it, and the arrays keep their bits.  ng = cells is still accepted."""
    torch = cuda
    box = ((0, 0, 0), (2, 7, 7), (5, 5, 5))           # 3 cells along x, 5 guards
    F = DevFabs(torch, box, HALO_COMPS, seed=31)
    s = _stream(torch)
    buf = [torch.zeros(1 << 16, dtype=torch.float64, device="cuda") for _ in range(2)]
    nf = len(HALO_COMPS)
    for mode in (0, 1):
        for ng in (4, 5):
            for k in range(nf):
                for side in (0, 1):
                    assert L.pic_halo_pack(C.byref(F.descs[k]), 0, side, ng, mode, buf[0].data_ptr(), s) != 0
                    assert b"exceeds the 3 cells" in L.pic_last_error()
                    assert L.pic_halo_unpack(C.byref(F.descs[k]), 0, side, ng, mode, buf[0].data_ptr(), s) != 0
            assert L.pic_halo_pack_multi(F.arr, nf, 0, ng, mode, buf[0].data_ptr(), buf[1].data_ptr(), s) != 0
            assert L.pic_halo_unpack_multi(F.arr, nf, 0, ng, mode, buf[0].data_ptr(), buf[1].data_ptr(), s) != 0
            assert b"exceeds the 3 cells" in L.pic_last_error()
        assert all(_same_bits(F.now(k), F.start[k]) for k in range(nf)), mode
        assert L.pic_halo_pack_multi(F.arr, nf, 0, 3, mode, buf[0].data_ptr(), buf[1].data_ptr(), s) == 0
        assert L.pic_halo_unpack(C.byref(F.descs[0]), 0, 1, 3, mode, buf[0].data_ptr(), s) == 0
        F.reset()


@pytest.mark.parametrize("periodic", [(1, 1, 1), (1, 0, 1)])
def test_boundary_local_multi_matches_per_component(L, cuda, periodic):
    """pic_boundary_local_multi (all components of a local sweep in one launch) against pic_fill_boundary_local /
    pic_sum_boundary_local one component at a time, bit for bit: every staggering, every periodic axis, ng from 0 to
    the allocated width, a non-periodic transverse axis."""
    torch = cuda
    n = (8, 12, 16)
    box = ((0, 0, 0), tuple(v - 1 for v in n), (3, 3, 3))
    geom = abi.make_geom(n, (0.0, 0.0, 0.0), tuple(float(v) for v in n), periodic=periodic)
    F = DevFabs(torch, box, HALO_COMPS, seed=41)
    G = DevFabs(torch, box, HALO_COMPS, seed=41)
    s = _stream(torch)
    nf = len(HALO_COMPS)
    for dim in range(3):
        if not periodic[dim]:
            continue
        for mode in (0, 1):
            for ng in (0, 1, 3):
                what = (dim, mode, ng)
                assert L.pic_boundary_local_multi(F.arr, nf, dim, ng, mode, C.byref(geom), s) == 0, L.pic_last_error()
                for k in range(nf):
                    one = L.pic_fill_boundary_local if mode == 0 else L.pic_sum_boundary_local
                    assert one(C.byref(G.descs[k]), dim, ng, C.byref(geom), s) == 0, L.pic_last_error()
                changed = False
                for k in range(nf):
                    a = F.now(k)
                    assert _same_bits(a, G.now(k)), what + (abi.COMP_NAMES[HALO_COMPS[k]],)
                    changed |= not _same_bits(a, F.start[k])
                assert changed == (ng > 0 or (mode == 1 and any(F.descs[k].stag[dim] for k in range(nf)))), what
                F.reset()
                G.reset()


# ---------------------------------------------------------------------------------------------------------------------
# Particle migration kernels against a numpy model
# ---------------------------------------------------------------------------------------------------------------------
MSG_HEADER, MSG_ROWS = 8, 8


class DevParticles:
    """A particle tile on the device: rows x y z w ux uy uz, 64-bit ids; `capacity` entries plus a sentinel pad."""
    PAD = 64

    def __init__(self, torch, rows, ids, capacity):
        self.torch, self.capacity = torch, capacity
        n = rows.shape[1]
        self.rows = torch.full((7, capacity + self.PAD), -777.0, dtype=torch.float64, device="cuda")
        self.ids = torch.full((capacity + self.PAD,), -7, dtype=torch.int64, device="cuda")
        self.rows[:, :n] = torch.from_numpy(rows).cuda()
        self.ids[:n] = torch.from_numpy(ids).cuda()
        self.soa = abi.pic_soa()
        for r, name in enumerate(("x", "y", "z", "w", "ux", "uy", "uz")):
            setattr(self.soa, name, self.rows[r].data_ptr())
        self.soa.idcpu = self.ids.data_ptr()
        self.soa.np = n

    def host(self):
        self.torch.cuda.synchronize()
        return self.rows.cpu().numpy(), self.ids.cpu().numpy()


def make_message(rows, ids, count, cap):
    """A migration message: header [0] = the sender's count (may exceed cap), then MSG_ROWS rows of cap entries."""
    msg = np.zeros(MSG_HEADER + MSG_ROWS * cap)
    msg[0] = count
    n = min(count, cap)
    body = msg[MSG_HEADER:].reshape(MSG_ROWS, cap)
    body[:7, :n] = rows[:, :n]
    body[7, :n] = ids[:n].view(np.float64)
    return msg


def _rows(rng, n, id0):
    return rng.standard_normal((7, n)), np.arange(id0, id0 + n, dtype=np.int64) * 3 + (1 << 40)


def test_migrate_pack_matches_message_format(L, cuda):
    """pic_migrate_pack: header = the true leaver count; the first min(count, cap) listed particles, row by row, the
    id as its bit pattern; nothing past them.  Counts below, at and above cap."""
    torch = cuda
    rng = np.random.default_rng(51)
    n, cap = 3000, 256
    rows, ids = _rows(rng, n, 0)
    P = DevParticles(torch, rows, ids, n)
    s = _stream(torch)
    nmsg = L.pic_migrate_message_doubles(cap)
    assert nmsg == MSG_HEADER + MSG_ROWS * cap
    for count in (0, 1, 97, cap, cap + 41):
        idx = rng.choice(n, size=cap, replace=False).astype(np.int32)
        d_idx = torch.from_numpy(idx).cuda()
        d_cnt = torch.tensor([count], dtype=torch.int32, device="cuda")
        msg = _sentinel_buf(torch, nmsg)
        assert L.pic_migrate_pack(C.byref(P.soa), d_idx.data_ptr(), d_cnt.data_ptr(), cap, msg.data_ptr(), s) == 0
        got = msg.cpu().numpy()
        m = min(count, cap)
        assert got[0] == count
        body = got[MSG_HEADER:nmsg].reshape(MSG_ROWS, cap)
        assert _same_bits(body[:7, :m], rows[:, idx[:m]]), count
        assert np.array_equal(body[7, :m].view(np.int64), ids[idx[:m]]), count
        assert np.all(body[:, m:] == 1.0e300) and np.all(got[nmsg:] == 1.0e300), count
        assert np.all(got[1:MSG_HEADER] == 1.0e300), count


def unpack_case(L, torch, rng, np_old, capacity, cap, holes, arrivals, counts=None, alias=False):
    """Run pic_migrate_unpack on a constructed tile and check it against the model of migrate.cu: arrival j fills
    hole j (low list first), the rest are appended at np_old in order; when more left than arrived, the tail
    [np_new, np_old) is compacted into the open holes below np_new.  holes: (low, high) index lists as the classify
    left them (cap entries at most), counts: the true leaver counts (default: the list lengths); arrivals: (low, high)
    as (count in the header, number of particles in the message).  Returns (np_new, status)."""
    rows, ids = _rows(rng, np_old, 0)
    P = DevParticles(torch, rows, ids, capacity)
    counts = counts or (len(holes[0]), len(holes[1]))
    idx = []
    for h in holes:
        a = np.full(cap, -1, dtype=np.int32)
        a[:len(h)] = h
        idx.append(torch.from_numpy(a).cuda())
    arr_rows, arr_ids, msgs = [], [], []
    for side, (hdr, n) in enumerate(arrivals):
        r, i = _rows(rng, n, 10_000_000 * (side + 1))
        arr_rows.append(r)
        arr_ids.append(i)
        msgs.append(torch.from_numpy(make_message(r, i, hdr, cap)).cuda())
    d_counts = torch.tensor(list(counts), dtype=torch.int32, device="cuda")
    work = torch.zeros(L.pic_migrate_workspace_bytes(cap) // 4, dtype=torch.int32, device="cuda")
    if alias:                               # the engine's way: the count lives in work[0], the soa's np is a launch bound
        work[0] = np_old
        P.soa.np = capacity
        np_dev = work.data_ptr()
    else:
        np_dev = None
    assert L.pic_migrate_unpack(C.byref(P.soa), d_counts.data_ptr(), idx[0].data_ptr(), idx[1].data_ptr(),
                                msgs[0].data_ptr(), msgs[1].data_ptr(), cap, capacity, work.data_ptr(), np_dev,
                                _stream(torch)) == 0, L.pic_last_error()
    got_rows, got_ids = P.host()
    w = work.cpu().numpy()
    # the model
    n0, n1 = min(counts[0], cap), min(counts[1], cap)
    hole = np.concatenate([np.asarray(holes[0][:n0]), np.asarray(holes[1][:n1])]).astype(np.int64)
    a_rows = np.concatenate([arr_rows[s][:, :min(arrivals[s][0], cap)] for s in (0, 1)], axis=1)
    a_ids = np.concatenate([arr_ids[s][:min(arrivals[s][0], cap)] for s in (0, 1)])
    n_arr = a_ids.size
    np_new = np_old + n_arr - len(hole)
    status = (1 if max(counts[0], counts[1], arrivals[0][0], arrivals[1][0]) > cap else 0) | (2 if np_new > capacity else 0)
    assert w[0] == np_new and w[5] == np_new and w[4] == np_old and w[1] == status, (w[:8], np_new, status)
    assert np.all(got_rows[:, capacity:] == -777.0) and np.all(got_ids[capacity:] == -7)     # nothing past the capacity
    if status & 2:
        return np_new, status
    if n_arr >= len(hole):                  # every hole filled in list order, the rest appended in order
        want_rows, want_ids = rows.copy(), ids.copy()
        want_rows[:, hole] = a_rows[:, :len(hole)]
        want_ids[hole] = a_ids[:len(hole)]
        want_rows = np.concatenate([want_rows, a_rows[:, len(hole):]], axis=1)
        want_ids = np.concatenate([want_ids, a_ids[len(hole):]])
        assert _same_bits(got_rows[:, :np_new], want_rows) and np.array_equal(got_ids[:np_new], want_ids)
    else:
        # who is where: the multiset by id, every particle with its own values; what stayed below np_new kept its slot
        keep = np.ones(np_old, dtype=bool)
        keep[hole] = False
        want_ids = np.concatenate([ids[keep], a_ids])
        assert np.array_equal(np.sort(got_ids[:np_new]), np.sort(want_ids))
        src = {int(i): rows[:, k] for k, i in enumerate(ids)}
        src.update({int(i): a_rows[:, k] for k, i in enumerate(a_ids)})
        for k in range(np_new):
            assert _same_bits(got_rows[:, k], src[int(got_ids[k])]), k
        stay = np.nonzero(keep[:np_new])[0]
        assert np.array_equal(got_ids[stay], ids[stay]) and _same_bits(got_rows[:, stay], rows[:, stay])
    return np_new, status


@pytest.mark.parametrize("alias", [False, True])
def test_migrate_unpack_matches_model(L, cuda, alias):
    """pic_migrate_unpack on constructed lists: arrivals equal to departures, more arrivals, more departures with open
    holes inside and outside the tail, lists and messages longer than cap (status 1), the tile's capacity exceeded
    (status 2); the particle count read from the host's np or from np_dev aliasing work[0]."""
    torch = cuda
    rng = np.random.default_rng(61 + alias)
    cap, np_old, capacity = 512, 6000, 8000

    def holes(nlo, nhi, tail=0, m=None):
        """nlo + nhi distinct hole indices; `tail` of them inside [np_old - m, np_old)."""
        pool_tail = np.arange(np_old - m, np_old) if m else np.empty(0, dtype=np.int64)
        t = rng.choice(pool_tail, size=tail, replace=False) if tail else np.empty(0, dtype=np.int64)
        rest = rng.choice(np.setdiff1d(np.arange(np_old), pool_tail), size=nlo + nhi - tail, replace=False)
        allh = np.concatenate([t, rest]).astype(np.int32)
        rng.shuffle(allh)
        return allh[:nlo], allh[nlo:]

    # equal
    assert unpack_case(L, torch, rng, np_old, capacity, cap, holes(100, 80), ((120, 120), (60, 60)), alias=alias) == (np_old, 0)
    # more arrivals than departures
    assert unpack_case(L, torch, rng, np_old, capacity, cap, holes(50, 30), ((200, 200), (150, 150)), alias=alias)[1] == 0
    # more departures: m = 350 open holes, 120 of them in the tail [np_new, np_old), the tail's other slots survivors
    assert unpack_case(L, torch, rng, np_old, capacity, cap, holes(300, 200, tail=120, m=350), ((100, 100), (50, 50)),
                       alias=alias) == (np_old - 350, 0)
    # every departure in the tail, no arrival
    assert unpack_case(L, torch, rng, np_old, capacity, cap, holes(200, 100, tail=300, m=300), ((0, 0), (0, 0)),
                       alias=alias) == (np_old - 300, 0)
    # no departure from the tail: all tail slots survive into the holes below
    assert unpack_case(L, torch, rng, np_old, capacity, cap, holes(200, 100, tail=0, m=300), ((0, 0), (0, 0)),
                       alias=alias) == (np_old - 300, 0)
    # lists longer than cap: the first cap leavers and arrivals move, the status says overflow
    lo, hi = holes(cap, 40)
    assert unpack_case(L, torch, rng, np_old, capacity, cap, (lo, hi), ((cap + 5, cap), (10, 10)),
                       counts=(cap + 77, 40), alias=alias)[1] == 1
    # the tile's capacity
    assert unpack_case(L, torch, rng, np_old, np_old + 100, cap, holes(10, 10), ((cap, cap), (cap, cap)), alias=alias)[1] == 2


def test_classify_and_candidate_list_match_numpy(L, cuda):
    """pic_particles_classify / pic_particles_classify_listed against numpy's restatement of classify_one (periodic
    ownership, two ranks along an axis, a non-periodic axis; positions on cell faces and outside the domain), the same
    leavers as a set; counts past the index capacity; the listed sweep with dead entries, and the full sweep once the
    list overflowed; pic_migrate_note_appended."""
    torch = cuda
    rng = np.random.default_rng(71)
    n, npart = 16, 5000
    plo, phi = -0.3, 1.7
    geom = abi.make_geom((n, n, n), (plo,) * 3, (phi,) * 3)
    dinv = 1.0 / ((phi - plo) / n)
    y = rng.uniform(plo - 0.05, phi + 0.05, npart)
    y[:200] = plo + (phi - plo) * rng.integers(0, n + 1, 200) / n             # on cell faces
    rows = rng.standard_normal((7, npart))
    rows[1] = y
    P = DevParticles(torch, rows, np.arange(npart, dtype=np.int64), npart)
    s = _stream(torch)
    lo, hi = 4, 11
    cell = np.clip(np.floor((y - plo) * dinv).astype(int), 0, n - 1)
    leave = (cell < lo) | (cell > hi)

    def model(both_up):
        width = hi - lo + 1
        up_lo = (hi + 1) % n
        up = (cell > hi) if both_up == 2 else (np.ones(npart, bool) if both_up == 1 else (cell >= up_lo) & (cell < up_lo + width))
        return set(np.nonzero(leave & ~up)[0].tolist()), set(np.nonzero(leave & up)[0].tolist())

    np_dev = torch.tensor([npart], dtype=torch.int32, device="cuda")

    def run(both_up, cap, cand=None, use_np_dev=False):
        counts = torch.zeros(2, dtype=torch.int32, device="cuda")
        idx = [torch.full((cap,), -7, dtype=torch.int32, device="cuda") for _ in range(2)]
        args = [C.byref(P.soa), C.byref(geom), 1, lo, hi, both_up, counts.data_ptr(), idx[0].data_ptr(), idx[1].data_ptr(), cap,
                np_dev.data_ptr() if use_np_dev else None]
        if cand is not None:
            assert L.pic_particles_classify_listed(*args, C.byref(cand), s) == 0, L.pic_last_error()
        else:
            assert L.pic_particles_classify(*args, s) == 0, L.pic_last_error()
        c = counts.cpu().numpy()
        got = [idx[k].cpu().numpy() for k in range(2)]
        for k in range(2):
            assert np.all(got[k][min(c[k], cap):] == -7)
        return [set(got[k][:min(c[k], cap)].tolist()) for k in range(2)], [int(v) for v in c]

    for both_up in (0, 1, 2):
        want = model(both_up)
        for use_np_dev in (False, True):
            got, c = run(both_up, 4096, use_np_dev=use_np_dev)
            assert got == list(want) and c == [len(want[0]), len(want[1])], both_up
        # index lists shorter than the leavers: true counts, the stored entries a subset
        got, c = run(both_up, 64)
        assert c == [len(want[0]), len(want[1])]
        assert all(len(got[k]) == min(64, c[k]) and got[k] <= want[k] for k in range(2))
    assert all(len(v) > 100 for v in model(0))
    # the candidate list: every leaver, some stayers, entries past the particle count, one dropped earlier
    leavers = np.nonzero(leave)[0]
    stay = np.nonzero(~leave)[0][:50]
    entries = np.concatenate([leavers, stay, [npart + 5, npart], [-1]]).astype(np.int32)
    rng.shuffle(entries)
    store = torch.from_numpy(np.concatenate([entries, np.full(64, -9, dtype=np.int32)])).cuda()
    count = torch.tensor([len(entries)], dtype=torch.int32, device="cuda")
    cand = abi.pic_escape_list()
    cand.idx, cand.count, cand.capacity = store.data_ptr(), count.data_ptr(), store.numel()
    want = model(0)
    got, c = run(0, 4096, cand)
    assert got == list(want) and c == [len(want[0]), len(want[1])]
    st = store.cpu().numpy()
    assert set(st[:len(entries)][entries >= npart].tolist()) == {-1}            # dead entries are dropped for good
    # appended arrivals of an unpack (work[4] = count before, work[5] = after) become candidates
    work = torch.zeros(8, dtype=torch.int32, device="cuda")

    def note(before, after):
        work[4], work[5] = before, after
        assert L.pic_migrate_note_appended(work.data_ptr(), C.byref(cand), s) == 0, L.pic_last_error()
        return int(count.cpu()[0]), store.cpu().numpy()

    c, st = note(npart - 10, npart)
    assert c == len(entries) + 10 and st[len(entries):len(entries) + 10].tolist() == list(range(npart - 10, npart))
    assert note(npart, npart - 3)[0] == len(entries) + 10                      # a net loss appends nothing
    assert note(0, 1000)[0] == store.numel() + 1                               # more than the list holds: overflow mark
    got, c = run(0, 4096, cand, use_np_dev=True)                              # overflowed list: every particle is visited
    assert got == list(want) and c == [len(want[0]), len(want[1])]


def test_owned_weights_match_numpy(L, cuda):
    """pic_particles_owned_weights: w inside the half-open brick [own_lo, own_hi), 0 outside; infinite faces; particles
    exactly on a face."""
    torch = cuda
    rng = np.random.default_rng(81)
    n = 5003
    rows = rng.uniform(-1.0, 2.0, (7, n))
    rows[3] = rng.uniform(0.5, 2.0, n)
    own_lo, own_hi = (0.0, -np.inf, 0.25), (1.0, 0.5, np.inf)
    for d in (0, 2):
        rows[d, :100] = own_lo[d]
        rows[d, 100:200] = own_hi[d] if np.isfinite(own_hi[d]) else 1.0
    P = DevParticles(torch, rows, np.arange(n, dtype=np.int64), n)
    out = torch.full((n + 5,), 3.0, dtype=torch.float64, device="cuda")
    assert L.pic_particles_owned_weights(C.byref(P.soa), abi.dbl3(own_lo), abi.dbl3(own_hi), out.data_ptr(), _stream(torch)) == 0
    inside = np.ones(n, dtype=bool)
    for d in range(3):
        inside &= (rows[d] >= own_lo[d]) & (rows[d] < own_hi[d])
    got = out.cpu().numpy()
    assert 0 < inside.sum() < n
    assert _same_bits(got[:n], np.where(inside, rows[3], 0.0)) and np.all(got[n:] == 3.0)


# ---------------------------------------------------------------------------------------------------------------------
# The step driver on bricks and slabs (the scenarios of test_host_multirank.py on the device)
# ---------------------------------------------------------------------------------------------------------------------
def test_two_bricks_periodic_loop_matches_oracle(orc, ranks, scenarios):
    scenarios.test_two_bricks_periodic_loop_matches_oracle(orc, ranks)


def test_eight_bricks_order3_thermal_loop_matches_oracle(orc, ranks, scenarios):
    """8^3 bricks, order 3, filter: ng_J = 5, so every SumBoundary of J along every axis is the thin-box unpack whose two
    slabs overlap; the migration classifies from the push's list (the listed-sweep counter)."""
    scenarios.test_eight_bricks_order3_thermal_loop_matches_oracle(orc, ranks)


def test_two_wide_bricks_order3_fused_current_exchange_matches_oracle(orc, ranks, scenarios):
    scenarios.test_two_wide_bricks_order3_fused_current_exchange_matches_oracle(orc, ranks)


@pytest.mark.parametrize("world", [4])
def test_z_slabs_with_moving_window_match_oracle(orc, ranks, scenarios, world):
    """(On two slabs the deck's plasma stays inside the upper slab for the scenario's 10 steps, and its check that
    particles crossed a slab boundary cannot hold; four slabs split the plasma.)"""
    scenarios.test_z_slabs_with_moving_window_match_oracle(orc, ranks, world)


def test_boosted_frame_z_slabs_match_oracle(orc, ranks, scenarios):
    scenarios.test_boosted_frame_z_slabs_match_oracle(orc, ranks)


def test_two_bricks_keep_gauss_law(orc, ranks, scenarios):
    full = workloads.uniform_plasma_3d(n=16, ppc=(2, 1, 1), u_th=0.3, perturbation=0.01)
    assert scenarios.gauss_bricks(orc, ranks, full, 2, 1, (1, 4, 5, 12))


def test_eight_bricks_keep_gauss_law(orc, ranks, scenarios):
    full = workloads.uniform_plasma_3d(n=16, ppc=(2, 1, 1), u_th=0.3, perturbation=0.01)
    assert scenarios.gauss_bricks(orc, ranks, full, 8, 3, (1, 4, 5, 8), use_filter=True)


@pytest.mark.parametrize("world", [2, 8])
def test_redistribute_moves_every_particle_to_its_owner(orc, ranks, world):
    """pic_engine_redistribute: particles displaced by up to 0.9 cell in every direction -- across brick faces, edges,
    corners and the periodic domain boundary -- end up on the rank that owns their cell, wrapped exactly like the
    oracle's enforcePeriodic, none lost, none duplicated."""
    import torch
    from warpx_b200.engine import Simulation
    n = 16
    full = workloads.uniform_plasma_3d(n=n, ppc=(1, 1, 2), u_th=0.0)
    s = full["species"][0]
    dx = [(full["prob_hi"][d] - full["prob_lo"][d]) / n for d in range(3)]
    rng = np.random.default_rng(8)
    shift = [rng.uniform(-0.9, 0.9, len(s["x"])) * dx[d] for d in range(3)]
    gid = np.arange(len(s["x"]), dtype=np.float64)          # carried in uz: identifies a particle after the move

    def rank_fn(rank, dist):
        dec = parallel.Decomposition((n, n, n), parallel.brick_grid(world), rank)
        sim = Simulation(full["n_cell"], full["prob_lo"], full["prob_hi"], nox=1, dist=dist, sort_interval=4)
        cell = [np.floor((s[k] - full["prob_lo"][d]) / dx[d]).astype(int) for d, k in enumerate("xyz")]
        m = np.ones(len(s["x"]), dtype=bool)
        for d in range(3):
            m &= (cell[d] >= dec.box_lo[d]) & (cell[d] <= dec.box_hi[d])
        sim.add_species(s["name"], s["q"], s["m"], s["x"][m], s["y"][m], s["z"][m], s["w"][m], s["ux"][m], s["uy"][m], gid[m])
        sp = sim.species[0]
        who = sp.array("uz").to(torch.int64)                 # the engine sorted the particles when they were registered
        for d, k in enumerate("xyz"):                         # the "push"
            sp.array(k).add_(torch.from_numpy(shift[d]).to(sp.array(k).device)[who])
        assert sim.L.pic_engine_redistribute(sim.native, sim.stream) == 0, sim.L.pic_last_error()
        sim._sync_from_native()
        return dict(P=sim.species_numpy(0), box=(dec.box_lo, dec.box_hi))

    res = run_ranks(world, rank_fn)
    got_id = np.concatenate([r["P"]["uz"] for r in res])
    assert len(got_id) == len(gid) and np.array_equal(np.sort(got_id), gid)
    Q = orc.HostParticles(x=s["x"] + shift[0], y=s["y"] + shift[1], z=s["z"] + shift[2], w=s["w"], ux=s["ux"], uy=s["uy"], uz=gid)
    geom = abi.make_geom(full["n_cell"], full["prob_lo"], full["prob_hi"])
    orc.lib().orc_wrap_periodic(C.byref(Q.soa), C.byref(geom))
    moved = 0
    for r in res:
        P, (blo, bhi) = r["P"], r["box"]
        idx = P["uz"].astype(np.int64)
        for d, k in enumerate("xyz"):
            assert np.array_equal(P[k], getattr(Q, k)[idx]), k
            c = np.clip(np.floor((P[k] - full["prob_lo"][d]) / dx[d]).astype(int), 0, n - 1)
            assert np.all((c >= blo[d]) & (c <= bhi[d])), (k, "a particle is on a rank that does not own its cell")
        cell0 = [np.floor((s[k][idx] - full["prob_lo"][d]) / dx[d]).astype(int) for d, k in enumerate("xyz")]
        moved += int(np.sum(~np.all([(cell0[d] >= blo[d]) & (cell0[d] <= bhi[d]) for d in range(3)], axis=0)))
    assert moved > 100


@pytest.mark.parametrize("nb,periodic,ngalloc", [((2, 1, 1), (1, 1, 1), 3), ((2, 2, 2), (1, 1, 1), 3), ((1, 1, 2), (1, 1, 0), 3),
                                                 ((2, 2, 2), (1, 1, 1), 5), ((1, 1, 2), (1, 1, 0), 5)])
def test_halo_copy_and_add_match_oracle(orc, ranks, nb, periodic, ngalloc):
    """pic_halo_copy / pic_halo_add on random data over 8-cell bricks against the oracle's multi-box FillBoundary /
    SumBoundary: every staggering, ng below and at the allocated width, a non-periodic axis split into slabs; with 5
    guard cells, src_ng 4 and 5 -- SumBoundary's slabs from the two sides overlap on every axis."""
    import torch
    from warpx_b200.lib import lib
    Lp = lib()
    world = nb[0] * nb[1] * nb[2]
    n = tuple(8 * v for v in nb)
    nga = (ngalloc,) * 3
    geom = abi.make_geom(n, (0.0, 0.0, 0.0), tuple(float(v) for v in n), periodic=periodic)
    comps = HALO_COMPS
    decs = [parallel.Decomposition(n, nb, r) for r in range(world)]
    rng = np.random.default_rng(3)
    # valid points from one global array per component (points shared by neighbouring boxes and the periodic duplicates
    # hold equal values, as in every exchange of a run); guard cells start random
    start = [[None] * len(comps) for _ in decs]
    for k, c in enumerate(comps):
        stag = abi.YEE_STAG[c]
        G = rng.standard_normal(tuple(n[2 - ax] + stag[2 - ax] for ax in range(3)))
        for d in range(3):
            if periodic[d] and stag[d]:
                hi_, lo_ = [slice(None)] * 3, [slice(None)] * 3
                hi_[2 - d], lo_[2 - d] = n[d], 0
                G[tuple(hi_)] = G[tuple(lo_)]
        for r, dec in enumerate(decs):
            f = abi.make_fab(None, dec.box_lo, dec.box_hi, nga, stag)
            a = rng.standard_normal(f.shape)
            sl = tuple(slice(dec.box_lo[2 - ax], dec.box_hi[2 - ax] + 1 + stag[2 - ax]) for ax in range(3))
            a[f.valid_slices()] = G[sl]
            start[r][k] = a

    def run(op, ng, src_ng=None):
        def rank_fn(rank, dist):
            from warpx_b200.engine import release_comm, shared_comm
            comm = shared_comm(Lp, dist, torch, torch.device("cuda", torch.cuda.current_device()))
            d = decs[rank]
            eng = Lp.pic_engine_create(C.byref(geom), abi.int3(d.box_lo), abi.int3(d.box_hi), 1, 1, 0, 0, 1.0, 0.0, 4, 0,
                                       abi.int3((1, 1, 1)))
            if not all(periodic):
                names = ["periodic" if p else "pec" for p in periodic]
                assert Lp.pic_engine_set_boundaries(eng, C.byref(abi.make_boundaries(names, names))) == 0
            assert Lp.pic_engine_set_comm(eng, comm, abi.int3(nb)) == 0, Lp.pic_last_error()
            descs, dev = [], []
            for k, c in enumerate(comps):
                f = abi.make_fab(None, d.box_lo, d.box_hi, nga, abi.YEE_STAG[c])
                t = torch.from_numpy(start[rank][k]).cuda()
                f.p = t.data_ptr()
                descs.append(f)
                dev.append(t)
            arr = (abi.pic_fab * len(descs))(*descs)
            s = torch.cuda.current_stream().cuda_stream
            if op == "copy":
                rc = Lp.pic_halo_copy(eng, arr, len(descs), abi.int3(ng), s)
            else:
                rc = Lp.pic_halo_add(eng, arr, len(descs), abi.int3(src_ng), abi.int3(ng), s)
            assert rc == 0, Lp.pic_last_error()
            out = [t.cpu().numpy() for t in dev]
            dist.barrier()
            Lp.pic_engine_destroy(eng)
            release_comm(dist)
            return out
        return run_ranks(world, rank_fn)

    g = ngalloc
    if g == 3:
        cases = [("copy", (2, 1, 3), None), ("copy", (3, 3, 3), None), ("add", (3, 3, 3), (2, 2, 2) if all(periodic) else (2, 2, 3)),
                 ("add", (3, 3, 3), (3, 3, 3))]
    elif all(periodic):
        cases = [("copy", (2, 4, 5), None), ("copy", (5, 5, 5), None), ("add", (5, 5, 5), (2, 2, 2)),
                 ("add", (5, 5, 5), (4, 4, 4)), ("add", (5, 5, 5), (5, 4, 5))]
    else:
        # x and y span the domain (8 cells): the local sum folds at most 3 guard layers onto 8 cells (2 src_ng + 1 <= 8)
        cases = [("copy", (2, 4, 5), None), ("copy", (5, 5, 5), None), ("add", (5, 5, 5), (3, 3, 5)), ("add", (5, 5, 4), (3, 2, 4))]
    for op, ng, src_ng in cases:
        got = run(op, ng, src_ng)
        for k, c in enumerate(comps):
            boxes = [orc.HostFab(d.box_lo, d.box_hi, nga, abi.YEE_STAG[c], data=start[r][k].copy()) for r, d in enumerate(decs)]
            arr = orc.fab_array(boxes)
            if op == "copy":
                orc.lib().orc_fill_boundary(arr, world, abi.int3(ng), C.byref(geom))
            else:
                orc.lib().orc_sum_boundary(arr, world, abi.int3(src_ng), abi.int3(ng), C.byref(geom))
            for r in range(world):
                # AMReX touches the box grown by ng only; the axis sweeps also rewrite (never-read) cells beyond it
                sl = tuple(slice(nga[2 - ax] - ng[2 - ax], boxes[r].a.shape[ax] - (nga[2 - ax] - ng[2 - ax])) for ax in range(3))
                scale = np.max(np.abs(boxes[r].a[sl]))
                assert np.max(np.abs(got[r][k][sl] - boxes[r].a[sl])) <= 1e-14 * scale, (op, ng, src_ng, abi.COMP_NAMES[c], r)


@pytest.mark.parametrize("world", [2, 8])
def test_langmuir_64_bricks_match_warpx_golden_checksums(orc, ranks, golden, world):
    """Config 1 (64^3 Langmuir wave, 40 steps) on `world` bricks: WarpX's golden checksums at rtol 1e-9, particle
    count conserved through migration -- the first section of multi_gpu_check.py, on one GPU."""
    from warpx_b200.engine import Simulation
    ref = golden["test_3d_langmuir_multi"]
    n = 64
    full = workloads.langmuir_3d(n=n)
    OL = orc.lib()

    def rank_fn(rank, dist):
        dec = parallel.Decomposition((n, n, n), parallel.brick_grid(world), rank)
        sim = Simulation(full["n_cell"], full["prob_lo"], full["prob_hi"], nox=1, dist=dist, sort_interval=4)
        for s in full["species"]:
            cell = [np.floor((s[k] - full["prob_lo"][d]) / sim.dx[d]).astype(int) for d, k in enumerate("xyz")]
            m = np.ones(len(s["x"]), dtype=bool)
            for d in range(3):
                m &= (cell[d] >= dec.box_lo[d]) & (cell[d] <= dec.box_hi[d])
            sim.add_species(s["name"], s["q"], s["m"], *[s[k][m] for k in ("x", "y", "z", "w", "ux", "uy", "uz")])
        n0 = sim.total_particles()
        sim.Evolve(40)
        assert sim.total_particles() == n0 == 2 * n ** 3
        sums = []
        for c in range(9):
            d, a = sim.field_numpy(c)
            hf = orc.HostFab(sim.box_lo, sim.box_hi, d.ng, abi.YEE_STAG[c], data=a)
            sums.append(OL.orc_checksum_cell_centered(C.byref(hf.desc), abi.int3(sim.box_lo), abi.int3(sim.box_hi)))
        for isp in range(2):
            P = sim.species_numpy(isp)
            sums += [np.sum(np.abs(P["x"])), np.sum(np.abs(P["y"])), np.sum(np.abs(P["z"])),
                     np.sum(np.abs(P["ux"])) * workloads.M_E, np.sum(np.abs(P["uz"])) * workloads.M_E, np.sum(P["w"])]
        return np.array(sums)

    v = np.sum(run_ranks(world, rank_fn), axis=0)
    for c, name in enumerate(abi.COMP_NAMES):
        g = ref["lev=0"][name]
        assert abs(v[c] - g) <= 1e-9 * abs(g), (name, v[c], g)
    keys = ["particle_position_x", "particle_position_y", "particle_position_z", "particle_momentum_x",
            "particle_momentum_z", "particle_weight"]
    for isp, sname in enumerate(("electrons", "positrons")):
        for j, key in enumerate(keys):
            if key in ref[sname]:
                g = ref[sname][key]
                assert abs(v[9 + 6 * isp + j] - g) <= 1e-9 * abs(g), (sname, key, v[9 + 6 * isp + j], g)
