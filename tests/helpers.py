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


# ---------------------------------------------------------------------------------------------
# Gauss's law through the whole step.  Esirkepov deposition gives rho(x^{n+1}) - rho(x^n) = -dt div J to round-off,
# and EvolveE's downward differences give div E^{n+1} - div E^n = -(dt/ep0) div J (Yee and CKC alike), so
# G = div E - rho/ep0 is the same at every step on every node of a periodic box.
# ---------------------------------------------------------------------------------------------
def gauss_residual(E, rho, dx, n_cell):
    """G = div E - rho/ep0 on the N^3 unique nodes of a periodic box, as a numpy array or a torch tensor (whichever
    the inputs are).  E: the valid Ex, Ey, Ez arrays [k, j, i] of the whole box; rho: the valid nodal charge density
    (guard cells already summed in).  div E at node (i, j, k) is (Ex[i] - Ex[i-1])/dx + (same in y) + (same in z),
    taken periodically; the upper nodal duplicate is dropped."""
    xp = np if isinstance(rho, np.ndarray) else __import__("torch")
    u = tuple(slice(0, n_cell[2 - ax]) for ax in range(3))
    div = 0.0
    for d in range(3):
        e = E[d][u]
        div = div + (e - xp.roll(e, 1, 2 - d)) / dx[d]
    return div - rho[u] / workloads.EP0


def gauss_drift(G, G0, rho0):
    """max|G - G0| / max|rho0/ep0|: the change of G over the run, on the scale of the initial charge."""
    scale = float(abs(rho0).max()) / workloads.EP0
    return float(abs(G - G0).max()) / scale


def div_b_ratio(B, dx, n_cell):
    """max|div B| / (max|B|/dx) over the N^3 unique cells of a periodic box (B: valid Bx, By, Bz arrays [k, j, i])."""
    xp = np if isinstance(B[0], np.ndarray) else __import__("torch")
    u = tuple(slice(0, n_cell[2 - ax]) for ax in range(3))
    div, scale = 0.0, 0.0
    for d in range(3):
        b = B[d][u]
        div = div + (xp.roll(b, -1, 2 - d) - b) / dx[d]
        scale = max(scale, float(abs(b).max()) / dx[d])
    return float(abs(div).max()) / scale if scale > 0 else 0.0


def simulation_gauss(sim):
    """(G, rho) of a one-rank Simulation's current state as tensors on its device: rho from Simulation.rho_numpy
    (pic_deposit_charge, the filter when it is on, SumBoundary), div E with torch where the fields live."""
    t = sim.torch
    E = [sim.data[c][sim.fab[c].valid_slices()] for c in range(3)]
    d, rho = sim.rho_numpy()
    rho = t.from_numpy(rho[d.valid_slices()].copy()).to(sim.device)
    return gauss_residual(E, rho, sim.dx, sim.n_cell), rho


def oracle_rho(orc, n_cell, prob_lo, prob_hi, nox, parts, q, use_filter=False, filter_npass=(1, 1, 1)):
    """Valid nodal charge density [k, j, i] of the particles `parts` (dict x..uz) in the periodic box, computed by the
    oracle: orc_deposit_charge, then (with the filter) the bilinear filter over the grown box, then SumBoundary --
    the sequence of Simulation.rho_numpy."""
    import ctypes as C
    L = orc.lib()
    box_lo, box_hi = (0, 0, 0), tuple(v - 1 for v in n_cell)
    dx = [(prob_hi[d] - prob_lo[d]) / n_cell[d] for d in range(3)]
    ng = (nox + 2,) * 3
    rho = orc.HostFab(box_lo, box_hi, ng, (1, 1, 1))
    xyzmin, lo = lower_corner(prob_lo, dx, box_lo, ng)
    P = orc.HostParticles(**{k: parts[k] for k in orc.HostParticles.NAMES})
    assert L.orc_deposit_charge(C.byref(P.soa), C.byref(rho.desc), abi.dbl3([1.0 / v for v in dx]), abi.dbl3(xyzmin),
                                abi.int3(lo), q, nox) == 0
    geom = abi.make_geom(n_cell, prob_lo, prob_hi)
    if use_filter:
        out = orc.HostFab(box_lo, box_hi, [ng[d] + filter_npass[d] for d in range(3)], (1, 1, 1))
        L.orc_apply_filter(C.byref(rho.desc), C.byref(out.desc), abi.int3(filter_npass))
        rho = out
    L.orc_sum_boundary(C.byref(rho.desc), 1, abi.int3(rho.desc.ng), abi.int3(rho.desc.ng), C.byref(geom))
    return rho.valid()


def make_species_in_box(n_cell, prob_lo, prob_hi, ppc, u_th, seed, perturbation=0.0):
    wl = workloads.uniform_plasma_3d(n_cell=n_cell, ppc=ppc, u_th=u_th, seed=seed,
                                     lx=prob_hi[0] - prob_lo[0], perturbation=perturbation)
    return wl


def lower_corner(prob_lo, dx, box_lo, ng):
    lo = [box_lo[d] - ng[d] for d in range(3)]
    return [prob_lo[d] + dx[d] * lo[d] for d in range(3)], lo


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
