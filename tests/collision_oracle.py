"""TEST INFRASTRUCTURE -- numpy restatement of the pairwise Coulomb collision stage (csrc/collision.cu) and of a
collision deck's loop, vectorised over cells and pair chains.

It follows the reference's BinaryCollision::doCollisionsWithinTile with PairWiseCoulombCollisionFunc
(Source/Particles/Collision/BinaryCollision/...) and the project's determinism contract: inside a cell the particles
of each species are put in ascending id order, shuffled (Fisher-Yates) with the Philox4x64-10 stream of tag 0 / 1,
and chain c of independent pairs draws from the stream of tag 2 + c; stream block j has the counter
(j + 1, step, global cell, 2^63 | collision index << 32 | tag) and the key (seed, 0).  Sums run sequentially in canonical
order and every expression keeps the kernel's evaluation order, so the restatement agrees with the device to the
last bits up to the ulps of the transcendentals."""
import numpy as np

C = 299792458.0
INV_C2 = 1.0 / (C * C)
EP0 = 8.8541878128e-12
HBAR = 1.054571817e-34
PI = 3.14159265358979323846
DBL_MIN = np.finfo(np.float64).tiny
TWO_M53 = 1.0 / 9007199254740992.0
LAST_S12 = [None]          # the s12 of the pairs of the last perez_update (the fixture script sizes dt with it)

_M0, _M1 = 0xD2E7470EE14C6C93, 0xCA5A826395121157
_W0, _W1 = 0x9E3779B97F4A7C15, 0xBB67AE8584CAA73B
_MASK32 = np.uint64(0xFFFFFFFF)


def _mulhilo(a, b):
    """(high, low) 64-bit words of the 128-bit product of the constant a and the uint64 array b."""
    a_lo, a_hi = np.uint64(a & 0xFFFFFFFF), np.uint64(a >> 32)
    b_lo, b_hi = b & _MASK32, b >> np.uint64(32)
    p0, p1, p2, p3 = a_lo * b_lo, a_lo * b_hi, a_hi * b_lo, a_hi * b_hi
    mid = (p0 >> np.uint64(32)) + (p1 & _MASK32) + (p2 & _MASK32)
    hi = p3 + (p1 >> np.uint64(32)) + (p2 >> np.uint64(32)) + (mid >> np.uint64(32))
    return hi, np.uint64(a) * b


def philox4x64_10(seed, c0, c1, c2, c3):
    """Philox4x64-10 blocks of the counters (c0, c1, c2, c3) (uint64 arrays, broadcast) with the key (seed, 0):
    an array [..., 4] of uint64 words."""
    with np.errstate(over="ignore"):
        c0, c1, c2, c3 = (np.asarray(v, dtype=np.uint64) for v in np.broadcast_arrays(c0, c1, c2, c3))
        k0, k1 = np.uint64(seed), np.uint64(0)
        for r in range(10):
            if r > 0:
                k0 = np.uint64((int(k0) + _W0) & 0xFFFFFFFFFFFFFFFF)
                k1 = np.uint64((int(k1) + _W1) & 0xFFFFFFFFFFFFFFFF)
            hi0, lo0 = _mulhilo(_M0, c0)
            hi1, lo1 = _mulhilo(_M1, c2)
            c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        return np.stack([c0, c1, c2, c3], axis=-1)


class Streams:
    """Consecutive 64-bit words of a set of streams (one per entry of `tag`), each stream its own counter."""

    def __init__(self, seed, step, gcell, cidx, tag):
        self.seed = seed
        self.c1 = np.uint64(step)
        self.c2 = np.asarray(gcell, dtype=np.uint64)
        self.c3 = np.uint64(1 << 63) | (np.uint64(cidx) << np.uint64(32)) | np.asarray(tag, dtype=np.uint64)
        self.drawn = np.zeros(self.c2.shape, dtype=np.int64)

    def words(self, sel):
        """the next word of the streams sel (index array or mask)"""
        d = self.drawn[sel]
        blk = philox4x64_10(self.seed, (d // 4 + 1).astype(np.uint64), self.c1, self.c2[sel], self.c3[sel])
        self.drawn[sel] += 1
        return blk[np.arange(len(d)), d % 4]

    def uniform(self, sel):                   # amrex::Random: (0, 1]
        return ((self.words(sel) >> np.uint64(11)) + np.uint64(1)).astype(np.float64) * TWO_M53

    def random_int(self, sel, n):             # amrex::Random_int(n)
        return ((self.words(sel) >> np.uint64(11)).astype(np.float64) * TWO_M53 * n).astype(np.int64)


def _dmax(a, b):
    return np.where(a < b, b, a)


def _dmin(a, b):
    return np.where(b < a, b, a)


def perez_update(u1, u2, q1, m1, w1, q2, m2, w2, n12, sigma_max, L, bmax, dt, rng, sel):
    """UpdateMomentumPerezElastic for the pairs sel of the streams rng: u1, u2 = (ux, uy, uz) arrays of the pairs;
    returns the new (u1, u2)."""
    u1x, u1y, u1z = u1
    u2x, u2y, u2z = u2
    g1sq = (u1x * u1x + u1y * u1y + u1z * u1z) * INV_C2
    g2sq = (u2x * u2x + u2y * u2y + u2z * u2z) * INV_C2
    g1, g2 = np.sqrt(1.0 + g1sq), np.sqrt(1.0 + g2sq)
    dx, dy, dz = u1x - u2x, u1y - u2y, u1z - u2z
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        dm = np.sqrt((dx * dx + dy * dy + dz * dz) * INV_C2)
        sm = np.sqrt(g1sq) + np.sqrt(g2sq)
        go = ~((dm < DBL_MIN) | (dm / sm < 1.0e-10))
        p1x, p1y, p1z = u1x * m1, u1y * m1, u1z * m1
        p2x, p2y, p2z = u2x * m2, u2y * m2, u2z * m2
        mg = m1 * g1 + m2 * g2
        vx, vy, vz = (p1x + p2x) / mg, (p1y + p2y) / mg, (p1z + p2z) / mg
        v2 = vx * vx + vy * vy + vz * vz
        gc = 1.0 / np.sqrt(1.0 - v2 * INV_C2)
        vdv1 = (vx * u1x + vy * u1y + vz * u1z) / g1
        vdv2 = (vx * u2x + vy * u2y + vz * u2z) / g2
        lt = (gc * gc * vdv1 * INV_C2 / (1.0 + gc) - gc) * m1 * g1
        s1x, s1y, s1z = p1x + vx * lt, p1y + vy * lt, p1z + vz * lt
        s1m = np.sqrt(s1x * s1x + s1y * s1y + s1z * s1z)
        g1s = (1.0 - vdv1 * INV_C2) * gc * g1
        g2s = (1.0 - vdv2 * INV_C2) * gc * g2
        mu = g1s * m1 * g2s * m2 / (g1s * m1 + g2s * m2)
        vrel = s1m / mu
        den = 1.0 + s1m * s1m / (m1 * g1s * m2 * g2s) * INV_C2
        vrel_inv = vrel / den
        aq = abs(q1 * q2)
        b0 = aq / (2.0 * PI * EP0 * mu * vrel * vrel_inv)
        if L > 0.0:
            lnL = np.full_like(b0, L)
        else:
            bmin = _dmax(HBAR * 0.5 / s1m, 0.5 * b0)
            lnL = _dmax(np.full_like(b0, 2.0), 0.5 * np.log(1.0 + bmax * bmax / (bmin * bmin)))
        sig = _dmin(PI * b0 * b0 * lnL, sigma_max)
        s12 = np.where(s1m > DBL_MIN, sig * n12 * dt * vrel * g1s * g2s / (g1 * g2), 0.0)
        LAST_S12[0] = s12
        go &= s12 > DBL_MIN
        idx = np.flatnonzero(go)
        out1 = [a.copy() for a in u1]
        out2 = [a.copy() for a in u2]
        if idx.size == 0:
            return out1, out2
        s = s12[idx]
        streams = sel[idx]
        r = rng.uniform(streams)
        cx = np.empty_like(s)
        b1 = s <= 0.1
        cx[b1] = 1.0 + s[b1] * np.log(r[b1])
        redo = np.flatnonzero(b1 & ~(cx >= -1.0))
        while redo.size:
            r[redo] = rng.uniform(streams[redo])
            cx[redo] = 1.0 + s[redo] * np.log(r[redo])
            redo = redo[~(cx[redo] >= -1.0)]
        b2 = (s > 0.1) & (s <= 3.0)
        sb = s[b2]
        ai = 0.0056958 + 0.9560202 * sb - 0.508139 * sb * sb + 0.47913906 * sb * sb * sb - \
            0.12788975 * sb * sb * sb * sb + 0.02389567 * sb * sb * sb * sb * sb
        cx[b2] = ai * np.log(np.exp(-1.0 / ai) + 2.0 * r[b2] * np.sinh(1.0 / ai))
        b3 = (s > 3.0) & (s <= 6.0)
        A = 3.0 * np.exp(-s[b3])
        cx[b3] = 1.0 / A * np.log(np.exp(-A) + 2.0 * r[b3] * np.sinh(A))
        b4 = ~(b1 | b2 | b3)
        cx[b4] = 2.0 * r[b4] - 1.0
        sx = np.sqrt(1.0 - cx * cx)
        phi = rng.uniform(streams) * 2.0 * PI
        cp, sp = np.cos(phi), np.sin(phi)
        X, Y, Z, M = s1x[idx], s1y[idx], s1z[idx], s1m[idx]
        pp = np.sqrt(X * X + Y * Y)
        big = pp > DBL_MIN
        pz = np.sqrt(Y * Y + Z * Z)
        f1x = np.where(big, (X * Z / pp) * sx * cp + (Y * M / pp) * sx * sp + (X) * cx,
                       (-pz) * sx * cp + (0.0) * sx * sp + (X) * cx)
        f1y = np.where(big, (Y * Z / pp) * sx * cp + (-X * M / pp) * sx * sp + (Y) * cx,
                       (Y * X / pz) * sx * cp + (Z * M / pz) * sx * sp + (Y) * cx)
        f1z = np.where(big, (-pp) * sx * cp + (0.0) * sx * sp + (Z) * cx,
                       (Z * X / pz) * sx * cp + (-Y * M / pz) * sx * sp + (Z) * cx)
        f2x, f2y, f2z = -f1x, -f1y, -f1z
        Vx, Vy, Vz, G = vx[idx], vy[idx], vz[idx], gc[idx]
        vdf1 = Vx * f1x + Vy * f1y + Vz * f1z
        vdf2 = Vx * f2x + Vy * f2y + Vz * f2z
        fac = G * G * INV_C2 / (G + 1.0)
        fac1 = fac * vdf1 + m1 * g1s[idx] * G
        fac2 = fac * vdf2 + m2 * g2s[idx] * G
        q1v = (f1x + Vx * fac1, f1y + Vy * fac1, f1z + Vz * fac1)
        q2v = (f2x + Vx * fac2, f2y + Vy * fac2, f2z + Vz * fac2)
        W1, W2 = w1[idx], w2[idx]
        wmax = _dmax(W1, W2)
        k1 = W2 > rng.uniform(streams) * wmax
        k2 = W1 > rng.uniform(streams) * wmax
        for c in range(3):
            out1[c][idx[k1]] = q1v[c][k1] / m1
            out2[c][idx[k2]] = q2v[c][k2] / m2
    return out1, out2


def cells_of(sp, geom):
    """global cell index i + nx (j + ny k) of every particle, as the cell sort bins it (clamped to the box)"""
    n_cell, plo, phi, box_lo, box_hi = (geom[k] for k in ("n_cell", "prob_lo", "prob_hi", "box_lo", "box_hi"))
    g = np.zeros(len(sp["x"]), dtype=np.int64)
    mult = 1
    for d, name in enumerate("xyz"):
        dinv = 1.0 / ((phi[d] - plo[d]) / n_cell[d])
        c = np.floor((sp[name] - plo[d]) * dinv).astype(np.int64) - box_lo[d]
        c = np.clip(c, 0, box_hi[d] - box_lo[d]) + box_lo[d]
        g += c * mult
        mult *= n_cell[d]
    return g


def _sequential_sums(vals, start, n):
    """per segment [start, start + n): sum of vals in order, left to right"""
    acc = np.zeros(len(start))
    for k in range(int(n.max()) if len(n) else 0):
        m = n > k
        acc[m] += vals[start[m] + k]
    return acc


def _temperature(sp, start, n, m):
    vx, vy, vz, vs, wt = (np.zeros(len(start)) for _ in range(5))
    for k in range(int(n.max()) if len(n) else 0):
        a = n > k
        i = start[a] + k
        w, ux, uy, uz = sp["w"][i], sp["ux"][i], sp["uy"][i], sp["uz"][i]
        us = ux * ux + uy * uy + uz * uz
        gm = np.sqrt(1.0 + us * INV_C2)
        wt[a] += w
        vx[a] += w * ux / gm
        vy[a] += w * uy / gm
        vz[a] += w * uz / gm
        vs[a] += w * us / gm / gm
    with np.errstate(invalid="ignore", divide="ignore"):
        vx, vy, vz, vs = vx / wt, vy / wt, vz / wt, vs / wt
        return m / 3.0 * (vs - (vx * vx + vy * vy + vz * vz))


def _shuffle(perm, start, n, rng_seed, step, gcell, cidx, tag):
    rng = Streams(rng_seed, step, gcell, cidx, np.full(len(start), tag))
    for d in range(int(n.max()) - 1 if len(n) else 0):
        i = n - 1 - d
        act = np.flatnonzero(i >= 1)
        j = rng.random_int(act, (i[act] + 1).astype(np.float64))
        a, b = start[act] + i[act], start[act] + j
        pa = perm[a].copy()
        perm[a] = perm[b]
        perm[b] = pa


def _canonical(sp, geom):
    g = cells_of(sp, geom)
    order = np.lexsort((sp["id"], g))
    s = {k: np.asarray(sp[k])[order].copy() for k in ("x", "y", "z", "w", "ux", "uy", "uz", "id")}
    cells, start, n = np.unique(g[order], return_index=True, return_counts=True)
    return order, s, cells, start, n


def collide(sp1, sp2, coll, geom, dt, step, record=None):
    """One call of pic_collide_pairwise_coulomb: sp1 / sp2 = dicts of x y z w ux uy uz id arrays (sp2 ignored when
    coll["same_species"]); coll = dict(q1, m1, q2, m2, coulomb_log, seed, collision_index, same_species); geom =
    dict(n_cell, prob_lo, prob_hi, box_lo, box_hi).  Returns (ux, uy, uz) of each species in its storage order.
    record: a dict that receives the canonical pairs and shuffles (indices into the id-sorted cell order)."""
    same = bool(coll["same_species"])
    q1, m1, q2, m2 = coll["q1"], coll["m1"], coll["q2"], coll["m2"]
    if same:
        q2, m2 = q1, m1
    L, seed, cidx = float(coll["coulomb_log"]), int(coll["seed"]), int(coll["collision_index"])
    dxs = [(geom["prob_hi"][d] - geom["prob_lo"][d]) / geom["n_cell"][d] for d in range(3)]
    dV = dxs[0] * dxs[1] * dxs[2]
    o1, s1, c1, st1, n1 = _canonical(sp1, geom)
    if same:
        keep = n1 >= 2
        cells, st1, n1 = c1[keep], st1[keep], n1[keep]
        s2, st2, n2 = s1, st1, n1
    else:
        o2, s2, c2, st2, n2 = _canonical(sp2, geom)
        cells, i1, i2 = np.intersect1d(c1, c2, assume_unique=True, return_indices=True)
        st1, n1, st2, n2 = st1[i1], n1[i1], st2[i2], n2[i2]
    dn1 = _sequential_sums(s1["w"], st1, n1) / dV
    dn2 = dn1 if same else _sequential_sums(s2["w"], st2, n2) / dV
    T1 = T2 = np.zeros(len(cells))
    if L < 0.0:                              # temperatures only for CoulombLog < 0
        T1 = _temperature(s1, st1, n1, m1)
        T2 = T1 if same else _temperature(s2, st2, n2, m2)
    perm1 = np.arange(len(s1["x"]))
    _shuffle(perm1, st1, n1, seed, step, cells, cidx, 0)
    if same:
        perm2 = perm1
    else:
        perm2 = np.arange(len(s2["x"]))
        _shuffle(perm2, st2, n2, seed, step, cells, cidx, 1)
    with np.errstate(divide="ignore", invalid="ignore"):    # T <= 0 in a cell of one particle: NaN, as in the kernel
        lmdD = np.full(len(cells), -1.0) if L > 0.0 else \
            1.0 / np.sqrt(dn1 * q1 * q1 / (T1 * EP0) + dn2 * q2 * q2 / (T2 * EP0))
    maxn = _dmax(dn1, dn2)
    rmin = 1.0 / np.cbrt(4.0 * PI / 3.0 * maxn)
    bmax = _dmax(lmdD, rmin)
    sigma_max = 1.0 / (maxn * rmin)
    if same:
        half = n1 // 2
        base1, base2, NI1, NI2 = st1, st1 + half, half, n1 - half
    else:
        base1, base2, NI1, NI2 = st1, st2, n1, n2
    maxN, minN = np.maximum(NI1, NI2), np.minimum(NI1, NI2)
    chain_cell = np.repeat(np.arange(len(cells)), minN)
    first = np.cumsum(minN) - minN
    cc = np.arange(len(chain_cell)) - np.repeat(first, minN)
    rng = Streams(seed, step, cells[chain_cell], cidx, 2 + cc)
    U1 = [s1["ux"], s1["uy"], s1["uz"]]
    U2 = U1 if same else [s2["ux"], s2["uy"], s2["uz"]]
    pairs = []
    sstep = 0
    while True:
        k = cc + sstep * minN[chain_cell]
        act = np.flatnonzero(k < maxN[chain_cell])
        if act.size == 0:
            break
        cl = chain_cell[act]
        i1 = cc[act] + np.where(maxN[cl] == NI1[cl], sstep * minN[cl], 0)
        i2 = cc[act] + np.where(maxN[cl] == NI2[cl], sstep * minN[cl], 0)
        a, b = perm1[base1[cl] + i1], perm2[base2[cl] + i2]
        pairs.append((a, b))
        wa, wb = s1["w"][a], s2["w"][b]
        wpmax = _dmax(wa, wb)
        n12 = wpmax * (minN[cl] + maxN[cl] - 1).astype(np.float64) / dV if same else \
            wpmax * minN[cl].astype(np.float64) / dV
        new1, new2 = perez_update([u[a] for u in U1], [u[b] for u in U2], q1, m1, wa, q2, m2, wb, n12,
                                  sigma_max[cl], L, bmax[cl], dt, rng, act)
        for c in range(3):
            U1[c][a] = new1[c]
            U2[c][b] = new2[c]
        sstep += 1
    if record is not None:
        record.update(perm1=perm1, perm2=perm2, pairs=pairs, order1=o1, order2=None if same else o2)

    def back(s, order):
        out = []
        for name in ("ux", "uy", "uz"):
            v = np.empty_like(s[name])
            v[order] = s[name]
            out.append(v)
        return out
    return back(s1, o1), (None if same else back(s2, o2))


def deck_loop(species, collisions, geom, dt, steps, first_step=0):
    """A collision deck with algo.maxwell_solver = none and zero fields: per step the collisions due
    (int(floor(t / dt)) % ndt == 0, with dt * ndt), then x += u / gamma dt and the periodic wrap.  species: list of
    dicts (x y z w ux uy uz id q m), changed in place; collisions: list of dicts (species=(i, j), coulomb_log, ndt,
    seed) in registration order."""
    t = first_step * dt
    for step in range(first_step, first_step + steps):
        for ic, c in enumerate(collisions):
            if int(np.floor(t / dt)) % c["ndt"] != 0:
                continue
            i, j = c["species"]
            spec = dict(q1=species[i]["q"], m1=species[i]["m"], q2=species[j]["q"], m2=species[j]["m"],
                        coulomb_log=c["coulomb_log"], seed=c["seed"], collision_index=ic, same_species=int(i == j))
            r1, r2 = collide(species[i], species[j], spec, geom, dt * c["ndt"], step)
            for k, name in enumerate(("ux", "uy", "uz")):
                species[i][name] = r1[k]
                if r2 is not None:
                    species[j][name] = r2[k]
        for sp in species:
            ig = 1.0 / np.sqrt(1.0 + (sp["ux"] * sp["ux"] + sp["uy"] * sp["uy"] + sp["uz"] * sp["uz"]) * INV_C2)
            for d, (xn, un) in enumerate((("x", "ux"), ("y", "uy"), ("z", "uz"))):
                lo, hi = geom["prob_lo"][d], geom["prob_hi"][d]
                v = sp[xn] + sp[un] * ig * dt
                ln = hi - lo
                v = np.where(v > hi, v - ln, np.where(v < lo, v + ln, v))
                sp[xn] = np.clip(v, lo, hi)
        t += dt
    return species
