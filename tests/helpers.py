"""Shared helpers of the parity tests."""
import numpy as np

from warpx_b200 import abi, workloads  # noqa: F401


def rel_linf(a, b):
    """max|a-b| / max|b| (fields with heavy cancellation are compared against their scale)."""
    s = np.max(np.abs(b))
    return float(np.max(np.abs(a - b)) / s) if s > 0 else float(np.max(np.abs(a - b)))


def random_fields(orc, box_lo, box_hi, ng, seed, comps=range(6), scale=None):
    """HostFab list Ex..jz with random values everywhere (guards included)."""
    rng = np.random.default_rng(seed)
    out = []
    for c in comps:
        f = orc.HostFab(box_lo, box_hi, ng, abi.YEE_STAG[c])
        s = 1.0 if scale is None else scale[c]
        f.a[...] = s * rng.standard_normal(f.a.shape)
        out.append(f)
    return out


def make_species_in_box(n_cell, prob_lo, prob_hi, ppc, u_th, seed, perturbation=0.0):
    wl = workloads.uniform_plasma_3d(n_cell=n_cell, ppc=ppc, u_th=u_th, seed=seed,
                                     lx=prob_hi[0] - prob_lo[0], perturbation=perturbation)
    return wl


def lower_corner(prob_lo, dx, box_lo, ng):
    lo = [box_lo[d] - ng[d] for d in range(3)]
    return [prob_lo[d] + dx[d] * lo[d] for d in range(3)], lo


class NumpyHaloOps:
    """CPU stand-in for the CUDA guard-cell kernels (same slab definitions as
    warpx_b200/csrc/halo.cu) so that parallel.HaloExchanger can be exercised over gloo."""

    def __init__(self, torch, n_cell):
        self.torch, self.n_cell = torch, n_cell

    def empty(self, n):
        return self.torch.empty(n, dtype=self.torch.float64)

    @staticmethod
    def _view(fab):
        return fab.host      # numpy array [k, j, i] attached to the descriptor by the test

    @staticmethod
    def _range(fab, dim, side, ng, mode, unpack):
        lc = fab.lo[dim] + fab.ng[dim]
        hc = fab.hi[dim] - fab.ng[dim] - fab.stag[dim]
        st = fab.stag[dim]
        if mode == 0:
            count = ng
            first = (hc + 1 - ng if side else lc + st) if not unpack else (hc + 1 + st if side else lc - ng)
        else:
            count = ng + st
            first = (hc + 1 if side else lc - ng) if not unpack else (hc + 1 - ng if side else lc)
        return first - fab.lo[dim], count

    def slab_count(self, fab, dim, ng, mode):
        n = 1
        for d in range(3):
            if d != dim:
                n *= fab.hi[d] - fab.lo[d] + 1
        return n * (ng if mode == 0 else ng + fab.stag[dim])

    def _slice(self, fab, dim, first, count):
        sl = [slice(None)] * 3
        sl[2 - dim] = slice(first, first + count)
        return tuple(sl)

    def pack(self, fab, dim, side, ng, mode, buf):
        first, count = self._range(fab, dim, side, ng, mode, False)
        a = self._view(fab)[self._slice(fab, dim, first, count)]
        buf.copy_(self.torch.from_numpy(np.ascontiguousarray(a).ravel()))

    def unpack(self, fab, dim, side, ng, mode, buf):
        first, count = self._range(fab, dim, side, ng, mode, True)
        sl = self._slice(fab, dim, first, count)
        a = self._view(fab)
        v = buf.numpy().reshape(a[sl].shape)
        if mode:
            a[sl] += v
        else:
            a[sl] = v

    def fill_local(self, fab, dim, ng):
        a = self._view(fab)
        N = self.n_cell[dim]
        vl, vh = fab.ng[dim], fab.hi[dim] - fab.lo[dim] - fab.ng[dim]
        ax = 2 - dim
        idx = np.arange(a.shape[ax])
        lo_g, hi_g = idx[vl - ng:vl], idx[vh + 1:vh + 1 + ng]
        a_sw = np.moveaxis(a, ax, 0)
        a_sw[lo_g] = a_sw[lo_g + N]
        a_sw[hi_g] = a_sw[hi_g - N]

    def sum_local(self, fab, dim, ng):
        a = np.moveaxis(self._view(fab), 2 - dim, 0)
        N = self.n_cell[dim]
        vl, vh = fab.ng[dim], fab.hi[dim] - fab.lo[dim] - fab.ng[dim]
        if fab.stag[dim]:
            s = a[vl] + a[vh]
            a[vl] = s
            a[vh] = s
        for g in range(1, ng + 1):
            a[vl - g + N] += a[vl - g]
            a[vh + g - N] += a[vh + g]


# ---------------------------------------------------------------------------------------------
# Outputs of the oracle's leaf arithmetic and stages on fixed, seeded inputs.  tests/golden/make_reference_leaves.py
# records them with the reference's own headers compiled in (oracle/_ref) as SHA-256 digests in
# tests/golden/reference_leaves.json; the tests recompute them with the restated leaves and compare bit for bit.
# ---------------------------------------------------------------------------------------------
def digest(a):
    """SHA-256 of the float64 bits of a (-0.0 counted as 0.0, as == does)."""
    import hashlib
    a = np.ascontiguousarray(np.asarray(a, dtype=np.float64) + 0.0, dtype="<f8")
    return hashlib.sha256(a.tobytes()).hexdigest()


def leaf_outputs(orc, L):
    """Shape factors (orders 0..4, plain and shifted), the three momentum pushers with the position update, the
    FDTD stencil coefficients and the largest stable dt of the library L."""
    import ctypes as C
    rng = np.random.default_rng(7)
    out = {}
    for order in range(0, 5):
        shp, shifted = [], []
        for x in rng.uniform(0.0, 40.0, 400):
            s = (C.c_double * 8)()
            i_new = L.orc_shape(order, x, s)
            shp.append([i_new] + list(s))
            xo = x + rng.uniform(-0.999, 0.999)
            s = (C.c_double * 8)()
            shifted.append([L.orc_shifted_shape(order, xo, i_new, s)] + list(s))
        out["shape%d" % order], out["shifted_shape%d" % order] = shp, shifted
    for pusher in (0, 1, 2):
        res = []
        for _ in range(300):
            u0 = rng.normal(0, 3e8, 3)
            eb = np.concatenate([rng.normal(0, 1e11, 3), rng.normal(0, 300.0, 3)])
            u = (C.c_double * 3)(*u0)
            L.orc_push_momentum(pusher, u, (C.c_double * 6)(*eb), -workloads.Q_E, workloads.M_E, 1.3e-16)
            x = (C.c_double * 3)(1e-6, 2e-6, 3e-6)
            L.orc_update_position(x, u, 1.3e-16)
            res.append(list(u) + list(x))
        out["pusher%d" % pusher] = res
    for algo in (0, 1):
        for k, dx in enumerate(([1e-6, 1e-6, 1e-6], [1e-6, 2e-6, 0.5e-6])):
            st = abi.pic_stencil()
            dxc = (C.c_double * 3)(*dx)
            L.orc_stencil_coefs(algo, dxc, C.byref(st))
            out["stencil%d_%d" % (algo, k)] = list(st.cx) + list(st.cy) + list(st.cz) + [L.orc_max_dt(algo, dxc)]
    return out


def stage_outputs(orc, L):
    """Whole stages of the library L on seeded inputs: FDTD EvolveB + EvolveE (Yee and CKC) on random fields, then
    gather + push (three pushers) and Esirkepov deposition at orders 1..3 (one thread)."""
    import ctypes as C
    n = 12
    box_lo, box_hi = (0, 0, 0), (n - 1,) * 3
    prob_lo, prob_hi = (-1e-5,) * 3, (1e-5,) * 3
    dx = [(prob_hi[d] - prob_lo[d]) / n for d in range(3)]
    threads = L.orc_num_threads()
    L.orc_set_num_threads(1)
    out = {}
    try:
        for algo in (0, 1):
            st = abi.pic_stencil()
            L.orc_stencil_coefs(algo, (C.c_double * 3)(*dx), C.byref(st))
            F = random_fields(orc, box_lo, box_hi, (2, 2, 2), 3, comps=range(9), scale=[1e9] * 3 + [3.0] * 3 + [1e12] * 3)
            E, Bf, J = orc.fab_array(F[0:3]), orc.fab_array(F[3:6]), orc.fab_array(F[6:9])
            L.orc_evolve_b(Bf, E, C.byref(st), 1e-15)
            L.orc_evolve_e(E, Bf, J, C.byref(st), 2e-15)
            for c, f in enumerate(F):
                out["fdtd%d_%s" % (algo, abi.COMP_NAMES[c])] = f.a.copy()
        sp = workloads.uniform_plasma_3d(n_cell=(n, n, n), ppc=(2, 1, 1), u_th=0.2, lx=2e-5)["species"][0]
        for nox in (1, 2, 3):
            ngEB = (4, 4, 4)
            xyzmin, lo = lower_corner(prob_lo, dx, box_lo, ngEB)
            dinv = [1.0 / v for v in dx]
            F = random_fields(orc, box_lo, box_hi, ngEB, 5, comps=range(9), scale=[1e10] * 3 + [30.0] * 3 + [0.0] * 3)
            P = orc.HostParticles(**{k: sp[k] for k in orc.HostParticles.NAMES})
            for pusher in (0, 1, 2):
                L.orc_gather_push(C.byref(P.soa), 0, P.np, orc.fab_array(F[0:3]), orc.fab_array(F[3:6]),
                                  abi.dbl3(dinv), abi.dbl3(xyzmin), abi.int3(lo), sp["q"], sp["m"], 2e-15,
                                  nox, 1, pusher, 1)
            L.orc_deposit_esirkepov(C.byref(P.soa), 0, P.np, orc.fab_array(F[6:9]), abi.dbl3(dinv),
                                    abi.dbl3(xyzmin), abi.int3(lo), sp["q"], 2e-15, -1e-15, nox)
            for name, a in (("x", P.x), ("ux", P.ux), ("uz", P.uz), ("jx", F[6].a), ("jy", F[7].a), ("jz", F[8].a)):
                out["particles%d_%s" % (nox, name)] = a.copy()
    finally:
        L.orc_set_num_threads(threads)
    return out


def order4_loop_fields(orc, kind):
    """Ex..jz after a 6-step order-4 loop of the oracle (kind: restated or reference leaves), on one thread."""
    wl = workloads.uniform_plasma_3d(n=12, ppc=(2, 1, 2), u_th=0.3, lx=3e-6, perturbation=0.02)
    s = wl["species"][0]
    L = orc.lib(kind)
    threads = L.orc_num_threads()
    L.orc_set_num_threads(1)
    try:
        sim = orc.OracleSim(wl["n_cell"], wl["prob_lo"], wl["prob_hi"], nox=4, kind=kind)
        assert sim.guards() == {"ng_EB": [4, 4, 4], "ng_J": [5, 5, 5], "ng_FG": [2, 2, 2], "ng_FS": [1, 1, 1]}
        sim.add_species(s["q"], s["m"], s["x"], s["y"], s["z"], s["w"], s["ux"], s["uy"], s["uz"])
        sim.evolve(6)
        return {abi.COMP_NAMES[c]: sim.fab(c)[1].copy() for c in range(9)}
    finally:
        L.orc_set_num_threads(threads)


def shape_factor_outputs(order, shape, shifted_shape):
    """shape(order, x, out) / shifted_shape(order, x_old, i_new, out) (the ctypes functions of a library) on the
    seeded positions of the device shape-factor test."""
    import ctypes as C
    rng = np.random.default_rng(60 + order)
    xs = np.concatenate([rng.uniform(0.0, 40.0, 4000), np.arange(0, 12) * 1.0, np.arange(0, 12) + 0.5])
    plain, shifted = [], []
    for x in xs:
        a = (C.c_double * 8)()
        i_new = shape(order, float(x), a)
        plain.append([i_new] + list(a))
        for dxo in (-0.7, -0.2, 0.0, 0.3, 0.9):
            x_old = float(x) + dxo
            if x_old < 0:
                continue
            s = (C.c_double * 8)()
            shifted.append([shifted_shape(order, x_old, i_new, s)] + list(s))
    return {"shape": plain, "shifted_shape": shifted}
