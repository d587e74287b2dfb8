"""Cases of the fluid tests, written once for a library and a torch device: tests/test_gpu_fluid.py runs them on the
GPU with the CUDA library, tests/test_fluid.py on the host build of the same sources (tests/host_harness)."""
import ctypes as C
import math

import numpy as np

import fluid_oracle as fo
from warpx_b200 import abi, workloads

N0 = 2.0e24
LX = 40.0e-6


def _inputs(kind, n_cell, u=3.0):
    """density(x, y, z), momentum(x, y, z) in units of c, field scale, all periodic over the domain.  u: momentum
    amplitude of the vacuum case (3 c makes one step's edge densities negative next to the vacuum)."""
    k = 2.0 * math.pi / LX
    if kind == "langmuir":
        wl = workloads.langmuir_fluid_3d(n=n_cell[0])
        f = wl["fluids"][0]
        return f["density"], f["momentum"], 1e12
    if kind == "vacuum":       # N = 0 nodes next to N > 0: zero edges and the positivity limiter
        def density(x, y, z):
            s = np.sin(k * x) + 0.5 * np.sin(k * y) + 0.25 * np.cos(k * z)
            return np.where(s > 0.2, N0 * (1.0 + s), 0.0)
        return density, lambda x, y, z: (u * np.sin(k * y), u * np.cos(k * z), u * np.sin(k * x + 0.3)), 1e12
    if kind == "drift":        # |u| ~ 10 c
        return (lambda x, y, z: N0 * (1.0 + 0.1 * np.sin(k * x) * np.cos(k * z)),
                lambda x, y, z: (6.0 + 0.5 * np.sin(k * z), -5.0 + 0.3 * np.cos(k * x), 6.0 * np.cos(k * y)), 1e13)
    raise ValueError(kind)


def make_state(kind, n_cell, box_lo, box_hi):
    """(descriptor, state [4 arrays]) on the box with its 2 guard nodes evaluated from the periodic profile."""
    desc = abi.make_fab(None, box_lo, box_hi, (2, 2, 2), (1, 1, 1))
    dx = [LX / n_cell[d] for d in range(3)]
    density, momentum, _ = _inputs(kind, n_cell)
    lo = [desc.lo[d] for d in range(3)]
    full = abi.make_fab(None, lo, [desc.hi[d] - 1 for d in range(3)], (0, 0, 0), (1, 1, 1))
    st = fo.initial_state(full, (-LX / 2,) * 3, dx, lo, density, momentum)
    return desc, st, dx


def random_fabs(comps, box_lo, box_hi, ng, scale, seed):
    rng = np.random.default_rng(seed)
    out = []
    for c in comps:
        d = abi.make_fab(None, box_lo, box_hi, ng, abi.YEE_STAG[c])
        out.append((d, rng.uniform(-scale, scale, d.shape)))
    return out


class Dev:
    """Arrays of one call on the library's device: torch tensors behind pic_fab descriptors."""

    def __init__(self, torch, device):
        self.t, self.device, self.keep = torch, device, []

    def fab(self, desc, a):
        x = self.t.from_numpy(np.array(a, dtype=np.float64)).to(self.device)       # a copy, on any device
        self.keep.append(x)
        d = abi.pic_fab.from_buffer_copy(desc)
        d.p = x.data_ptr()
        return d, x

    def fabs(self, pairs):
        got = [self.fab(d, a) for d, a in pairs]
        return (abi.pic_fab * len(got))(*[g[0] for g in got]), [g[1] for g in got]


def _stream(torch, device):
    return torch.cuda.current_stream().cuda_stream if device.type == "cuda" else None


def rel_linf(a, b):
    s = np.max(np.abs(b))
    return float(np.max(np.abs(a - b)) / s) if s > 0 else float(np.max(np.abs(a - b)))


def check_stages(L, torch, device, kind, n_cell, box_lo, box_hi, tol, seed=1):
    """Each stage on the library against the oracle on the same inputs; returns {stage: rel-L-inf}.  J and rho start
    from a random background; points outside the owned valid region keep its exact bits."""
    st = _stream(torch, device)
    desc, state, dx = make_state(kind, n_cell, box_lo, box_hi)
    _, _, fscale = _inputs(kind, n_cell)
    q, m, dt = -workloads.Q_E, workloads.M_E, 0.99 / (workloads.C * math.sqrt(sum(1.0 / v ** 2 for v in dx)))
    err = {}
    dev = Dev(torch, device)
    # gather + push
    E = random_fabs(range(3), box_lo, box_hi, (2, 2, 2), fscale, seed)
    B = random_fabs(range(3, 6), box_lo, box_hi, (2, 2, 2), fscale / workloads.C, seed + 1)
    U, Ut = dev.fabs([(desc, a) for a in state])
    Ea, _ = dev.fabs(E)
    Ba, _ = dev.fabs(B)
    assert L.pic_fluid_gather_push(U, Ea, Ba, q, m, dt, st) == 0
    ref = [a.copy() for a in state]
    fo.gather_push(ref, desc, E, B, q, m, dt)
    got = [x.cpu().numpy() for x in Ut]
    err["gather_push"] = max(rel_linf(got[c], ref[c]) for c in range(4))
    assert np.array_equal(got[0], ref[0])
    # advection (from the pushed state, guards as evaluated)
    Uo, Uot = dev.fabs([(desc, np.zeros(desc.shape)) for _ in range(4)])
    cnt = torch.zeros(2, dtype=torch.int64, device=device)
    assert L.pic_fluid_advect(U, Uo, abi.dbl3(dx), dt, cnt.data_ptr(), st) == 0
    counters = {}
    ref2 = fo.advect(ref, desc, dx, dt, counters)
    got2 = [x.cpu().numpy() for x in Uot]
    V = desc.valid_slices()
    err["advect"] = max(rel_linf(got2[c][V], ref2[c][V]) for c in range(4))
    assert cnt.cpu().tolist() == [counters["zero_edges"], counters["limited"]]
    # current and charge deposit from the advected state onto a random background
    J = random_fabs(range(6, 9), box_lo, box_hi, (3, 3, 3), 1e10, seed + 2)
    Ja, Jt = dev.fabs(J)
    assert L.pic_fluid_deposit_current(Uo, Ja, q, st) == 0
    Jref = [(d, a.copy()) for d, a in J]
    fo.deposit_current(ref2, desc, Jref, q)
    err["deposit_current"] = 0.0
    for c in range(3):
        g, r, bg = Jt[c].cpu().numpy(), Jref[c][1], J[c][1]
        err["deposit_current"] = max(err["deposit_current"], rel_linf(g - bg, r - bg))
        untouched = r == bg
        assert np.array_equal(g[untouched], bg[untouched])
    rd = abi.make_fab(None, box_lo, box_hi, (3, 3, 3), (1, 1, 1))
    rbg = np.random.default_rng(seed + 3).uniform(-1, 1, rd.shape)
    Ra, Rt = dev.fab(rd, rbg)
    assert L.pic_fluid_deposit_charge(C.byref(Uo[0]), C.byref(Ra), q, st) == 0
    rref = rbg.copy()
    fo.deposit_charge(ref2, desc, rd, rref, q)
    g = Rt.cpu().numpy()
    err["deposit_charge"] = rel_linf(g - rbg, rref - rbg)
    assert np.array_equal(g[rref == rbg], rbg[rref == rbg])
    for k, v in err.items():
        assert v <= tol, (kind, k, v)
    return err, counters


def check_reference_fixture(L, torch, device):
    """tests/golden/fluid_reference_stages.npz (tests/golden/make_fluid_reference.py: MusclHancockUtils.H and
    UpdateMomentumHigueraCary.H compiled verbatim): the library's advection and the numpy restatement give the stored
    bits on every case, the vacuum edge whose positivity limiter acts included.  Returns the kernel's path counters."""
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fluid_reference_stages.npz"))
    st = _stream(torch, device)
    seen = {}
    for name in ("vacuum", "drift", "vacuum_limited"):
        lohi = [int(v) for v in g[name + "/desc"]]
        desc = abi.make_fab(None, [v + 2 for v in lohi[:3]], [v - 3 for v in lohi[3:]], (2, 2, 2), (1, 1, 1))
        dxdt = g[name + "/dxdt"]
        state, want = list(g[name + "/in"]), g[name + "/out"]
        V = desc.valid_slices()
        ref = fo.advect(state, desc, list(dxdt[:3]), float(dxdt[3]))
        for c in range(4):
            assert np.array_equal(ref[c][V], want[c][V]), (name, "restatement", c)
        dev = Dev(torch, device)
        U, _ = dev.fabs([(desc, a) for a in state])
        Uo, Uot = dev.fabs([(desc, np.zeros(desc.shape)) for _ in range(4)])
        cnt = torch.zeros(2, dtype=torch.int64, device=device)
        assert L.pic_fluid_advect(U, Uo, abi.dbl3(dxdt[:3]), float(dxdt[3]), cnt.data_ptr(), st) == 0
        for c in range(4):
            assert np.array_equal(Uot[c].cpu().numpy()[V], want[c][V]), (name, "kernel", c)
        seen[name] = cnt.cpu().tolist()
    q, m, dt = (float(v) for v in g["hc/qmdt"])
    got = fo.push_hc(*g["hc/in"], q, m, dt)
    for c in range(3):
        assert np.array_equal(got[c], g["hc/out"][c]), ("higuera-cary", c)
    assert seen["vacuum_limited"][1] > 0 and seen["vacuum"][0] > 0, seen
    return seen
