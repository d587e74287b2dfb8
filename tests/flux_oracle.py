"""TEST INFRASTRUCTURE -- float64 numpy restatement of one call of the flux injection (csrc/flux_injection.cu,
pic_add_flux_particles): PhysicalParticleContainer::AddPlasmaFlux with find_overlap_flux, InjectorPositionRandomPlane,
InjectorMomentumGaussianFlux, generateGaussianFluxDist, compute_scale_fac_area_plane and UpdatePosition over t_fract
(Source/Particles/..., Source/Initialization/...), with the project's random streams: Philox4x64-10 keyed by (seed, 0),
counter (j + 1, step, global plane cell, 2^63 | 2^61 | injector index << 32 | tag), tag 0 for a cell's count and
1 + p for particle p (two position uniforms, the normal momentum, the two transverse momenta, t_fract).

Vectorised over the particles; the transcendentals (log, exp, cos) are the C library's, called element by element
through Python's math module, so that a host build of the kernels agrees to the last bit.  Expressions keep the
kernel's evaluation order."""
import math

import numpy as np

from collision_oracle import Streams

C = 299792458.0
INV_C2 = 1.0 / (C * C)
PI = 3.14159265358979323846
FLUX_BIT = 1 << 29          # injector index field of the counter: (2^29 | index) << 32 = 2^61 | index << 32

_log = np.frompyfunc(math.log, 1, 1)
_exp = np.frompyfunc(math.exp, 1, 1)
_cos = np.frompyfunc(math.cos, 1, 1)


def log(x):
    return _log(np.asarray(x, dtype=np.float64)).astype(np.float64)


def exp(x):
    return _exp(np.asarray(x, dtype=np.float64)).astype(np.float64)


def cos(x):
    return _cos(np.asarray(x, dtype=np.float64)).astype(np.float64)


def random_normal(mean, stddev, rng, sel):
    """the project's amrex::RandomNormal: Box-Muller on two consecutive uniforms, the cosine branch"""
    u1 = rng.uniform(sel)
    u2 = rng.uniform(sel)
    return mean + stddev * (np.sqrt(-2.0 * log(u1)) * cos(2.0 * PI * u2))


def gaussian_flux(u_m, u_th, rng, sel):
    """generateGaussianFluxDist for the streams sel (index array): one u per stream"""
    sel = np.asarray(sel)
    u = np.zeros(len(sel))
    abs_u_m = abs(u_m)
    if u_th == 0.0:
        u[:] = u_m
    elif abs_u_m < 0.6 * u_th:
        umsign = math.copysign(1.0, u_m)
        approx_u_th = u_th / math.sqrt(1.0 - abs_u_m / u_th)
        reject_prefactor = (abs_u_m / u_th) / (2.0 * u_th * u_th)
        todo = np.arange(len(sel))
        while len(todo):
            with np.errstate(divide="ignore"):
                xrand = 1.0 - rng.uniform(sel[todo])
                v = approx_u_th * np.sqrt(2.0 * log(1.0 / xrand))
            u[todo] = v
            xrand = rng.uniform(sel[todo])
            with np.errstate(invalid="ignore"):
                accept = xrand < exp(-reject_prefactor * (v - umsign * u_th) * (v - umsign * u_th))
            todo = todo[~accept]
    else:
        approx_u_m = u_m + u_th * u_th / abs_u_m
        inv_um = 1.0 / abs_u_m
        todo = np.arange(len(sel))
        while len(todo):
            v = np.full(len(todo), -1.0)
            neg = np.arange(len(todo))
            while len(neg):
                v[neg] = random_normal(approx_u_m, u_th, rng, sel[todo[neg]])
                neg = neg[v[neg] < 0]
            u[todo] = v
            xrand = rng.uniform(sel[todo])
            accept = xrand < v * inv_um * exp(1.0 - v * inv_um)
            todo = todo[~accept]
    return u


def axes(axis):
    return (1, 2) if axis == 0 else ((0, 2) if axis == 1 else (0, 1))


def _cround(x):
    return int(math.copysign(math.floor(abs(x) + 0.5), x))


def plane_of_box(inj, geom, box_lo, box_hi):
    """find_overlap_flux with part_realbox = the problem domain: None, or (corner[3], n[3], shifted[3], tile_lo, tile_hi)
    with n = 1 along the normal; corner = prob_lo across the plane (the single box's overlap corner), the plane along it"""
    n_cell, plo, phi = geom
    dx = [(phi[d] - plo[d]) / n_cell[d] for d in range(3)]
    axis = inj["normal_axis"]
    corner, nov, shifted, tlo, thi = [0.0] * 3, [1] * 3, [0] * 3, [0.0] * 3, [0.0] * 3
    for d in range(3):
        tlo[d] = plo[d] + dx[d] * box_lo[d]
        thi[d] = plo[d] + dx[d] * (box_hi[d] + 1)
        if d == axis:
            pos = inj["surface_flux_pos"]
            if (pos < tlo[d] or pos >= thi[d]) if inj["direction"] > 0 else (pos <= tlo[d] or pos > thi[d]):
                return None
            corner[d] = pos
            continue
        if not tlo[d] <= phi[d] or not thi[d] >= plo[d]:
            return None
        ov_lo = plo[d] + max(math.floor((tlo[d] - plo[d]) / dx[d]), 0.0) * dx[d]
        ov_hi = phi[d] - max(math.floor((phi[d] - thi[d]) / dx[d]), 0.0) * dx[d]
        nov[d] = _cround((ov_hi - ov_lo) / dx[d])
        corner[d] = plo[d]          # positions from the domain's corner and global cell indices
        shifted[d] = _cround((ov_lo - plo[d]) / dx[d])
    t0, t1 = axes(axis)
    if nov[t0] <= 0 or nov[t1] <= 0:
        return None
    return corner, nov, shifted, tlo, thi


def inject(inj, geom, box_lo, box_hi, step, t, dt, first_id, injector_index=0):
    """One call for the box [box_lo, box_hi] of geom = (n_cell, prob_lo, prob_hi): (particles, ids_used), particles a
    dict of x, y, z, w, ux, uy, uz, id (int64) of the kept particles in creation order (cell-major, then p).
    inj: dict with the fields of pic_flux_injector."""
    n_cell, plo, phi = geom
    axis = inj["normal_axis"]
    t0, t1 = axes(axis)
    slots = int(math.floor(inj["num_ppc"])) + 1
    empty = {k: np.zeros(0) for k in ("x", "y", "z", "w", "ux", "uy", "uz")}
    empty["id"] = np.zeros(0, dtype=np.int64)
    tmin, tmax = inj["tmin"], inj["tmax"]
    if not ((tmin < 0 or t >= tmin) and (tmax < 0 or t < tmax)):
        return empty, 0
    ids_used = n_cell[t0] * n_cell[t1] * slots
    pl = plane_of_box(inj, geom, box_lo, box_hi)
    if pl is None:
        return empty, ids_used
    corner, nov, shifted, tlo, thi = pl
    dx = [(phi[d] - plo[d]) / n_cell[d] for d in range(3)]
    blo, bhi = inj["bound_lo"], inj["bound_hi"]
    c = np.arange(nov[t0] * nov[t1])
    i0, i1 = c % nov[t0], c // nov[t0]
    gcell = (shifted[t0] + i0) + n_cell[t0] * (shifted[t1] + i1)
    iv = [None] * 3
    iv[axis], iv[t0], iv[t1] = np.zeros_like(c), shifted[t0] + i0, shifted[t1] + i1
    overlaps = np.ones(len(c), dtype=bool)
    for d in range(3):
        lo = corner[d] + (iv[d] + 0.0) * dx[d]
        hi = corner[d] + (iv[d] + 1.0) * dx[d]
        overlaps &= (blo[d] <= hi) & (bhi[d] >= lo)
    cidx = FLUX_BIT | injector_index
    counts = np.zeros(len(c), dtype=np.int64)
    sel = np.nonzero(overlaps)[0]
    if len(sel):
        rng0 = Streams(inj["seed"], step, gcell[sel], cidx, np.zeros(len(sel), dtype=np.uint64))
        counts[sel] = np.minimum((inj["num_ppc"] + rng0.uniform(np.arange(len(sel)))).astype(np.int64), slots)
    cell = np.repeat(c, counts)
    p = np.arange(len(cell)) - np.repeat(np.cumsum(counts) - counts, counts)
    if len(cell) == 0:
        return empty, ids_used
    rng = Streams(inj["seed"], step, gcell[cell], cidx, (1 + p).astype(np.uint64))
    allp = np.arange(len(cell))
    ra, rb = rng.uniform(allp), rng.uniform(allp)
    r = [None] * 3
    r[axis], r[t0], r[t1] = np.zeros(len(cell)), ra, rb
    pos = [corner[d] + (iv[d][cell] + r[d]) * dx[d] for d in range(3)]
    un = gaussian_flux(inj["u_m"][axis], inj["u_th"][axis], rng, allp)
    if inj["direction"] < 0:
        un = -un
    u = [un if d == axis else random_normal(inj["u_m"][d], inj["u_th"][d], rng, allp) for d in range(3)]
    u = [v * C for v in u]
    ok = np.ones(len(cell), dtype=bool)
    for d in range(3):
        ok &= (tlo[d] <= pos[d]) & (pos[d] <= thi[d])
    for d in range(3):
        ok &= (pos[d] <= bhi[d]) & (pos[d] >= blo[d])
    if not inj["flux"] > 0:
        ok[:] = False
    keep = np.nonzero(ok)[0]
    t_fract = rng.uniform(keep) * dt
    uk = [v[keep] for v in u]
    inv_gamma = 1.0 / np.sqrt(1.0 + (uk[0] * uk[0] + uk[1] * uk[1] + uk[2] * uk[2]) * INV_C2)
    scale_fac = dx[0] * dx[1] * dx[2] / inj["num_ppc"]
    scale_fac /= dx[axis]
    out = {name: pos[d][keep] + uk[d] * inv_gamma * t_fract for d, name in enumerate(("x", "y", "z"))}
    out.update(ux=uk[0], uy=uk[1], uz=uk[2], w=np.full(len(keep), inj["flux"] * scale_fac * dt))
    out["id"] = (first_id + gcell[cell[keep]] * slots + p[keep]).astype(np.int64)
    return out, ids_used


def as_dict(f):
    """the fields of an abi.pic_flux_injector as the dict inject() takes"""
    return dict(num_ppc=f.num_ppc, surface_flux_pos=f.surface_flux_pos, normal_axis=f.normal_axis, direction=f.direction,
                flux=f.flux, tmin=f.tmin, tmax=f.tmax, bound_lo=list(f.bound_lo), bound_hi=list(f.bound_hi),
                u_m=list(f.u_m), u_th=list(f.u_th), seed=int(f.seed))


def sort_by_id(P):
    order = np.argsort(P["id"], kind="stable")
    return {k: v[order] for k, v in P.items()}


def concat(parts):
    return {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}


def deck(wl, steps=None):
    """The restatement of a flux deck (workloads.flux_injection_3d): every injector of every step on one box,
    at t = (s + 1) dt; the momenta and weights the analysis reads (maxwell_solver = none: nothing changes them)."""
    from warpx_b200 import abi
    geom = (wl["n_cell"], wl["prob_lo"], wl["prob_hi"])
    box_lo, box_hi = (0, 0, 0), tuple(v - 1 for v in wl["n_cell"])
    out = {}
    for k, s in enumerate(wl["species"]):
        inj = as_dict(abi.make_flux_injector(**s["flux"]))
        parts, next_id = [], 0
        for step in range(wl["max_step"] if steps is None else steps):
            P, used = inject(inj, geom, box_lo, box_hi, step, (step + 1) * wl["dt"], wl["dt"], next_id, k)
            parts.append(P)
            next_id += used
        out[s["name"]] = concat(parts)
    return out
