"""TEST INFRASTRUCTURE -- numpy restatement of the two-product nuclear fusion stage (csrc/fusion.cu): the event pass and
the product pass of one call, vectorised over cells and pair chains.

It follows the reference's BinaryCollision::doCollisionsWithinTile with NuclearFusionFunc, SingleNuclearFusionEvent,
BoschHaleFusionCrossSection and the products of ParticleCreationFunc / TwoProductFusionInitializeMomentum
(Source/Particles/Collision/BinaryCollision/...), and the project's determinism contract: a cell's live particles
(id != SPENT) of each species in ascending id order, shuffled with the streams of tag 0 / 1, chain c drawing from tag
2 + c (one uniform per pair with two live reactants), the products of the cell's j-th event drawing from the stream of
tag 2^62 | j; events numbered bin by bin (supercell-major bins), then by pair index.  Expressions keep the kernel's
evaluation order."""
import numpy as np

from collision_oracle import Streams, _shuffle, cells_of

C = 299792458.0
C_SQ = C * C
INV_CSQ = 1.0 / C_SQ
Q_E = 1.602176634e-19
ALPHA = 0.007297352573748943
PI = 3.14159265358979323846
DBL_MIN = np.finfo(np.float64).tiny
SPENT = np.int64(-1)                     # PIC_SPENT_ID as a signed 64-bit id
DT_NHE4, DD_PT, DD_NHE3 = 0, 1, 2
E_FUSION = {DT_NHE4: 17.5893e6 * Q_E, DD_PT: 4.032667e6 * Q_E, DD_NHE3: 3.268911e6 * Q_E}
BOSCH_HALE = {   # A1..A5, B1..B4
    DT_NHE4: (6.927e4, 7.454e8, 2.050e6, 5.2002e4, 0.0, 6.38e1, -9.95e-1, 6.981e-5, 1.728e-4),
    DD_PT: (5.5576e4, 2.1054e2, -3.2638e-2, 1.4987e-6, 1.8181e-10, 0.0, 0.0, 0.0, 0.0),
    DD_NHE3: (5.3701e4, 3.3027e2, -1.2706e-1, 2.9327e-5, -2.5151e-9, 0.0, 0.0, 0.0, 0.0),
}


def collision_parameters(u1, u2, m1, m2):
    """get_collision_parameters: (E_kin*, v_rel*, lab-to-CoM factor) of pairs, u = (ux, uy, uz) arrays"""
    u1x, u1y, u1z = u1
    u2x, u2y, u2z = u2
    g1 = np.sqrt(1.0 + (u1x * u1x + u1y * u1y + u1z * u1z) * INV_CSQ)
    g2 = np.sqrt(1.0 + (u2x * u2x + u2y * u2y + u2z * u2z) * INV_CSQ)
    sx, sy, sz = u1x * m1 + u2x * m2, u1y * m1 + u2y * m2, u1z * m1 + u2z * m2
    p_total_sq = sx * sx + sy * sy + sz * sz
    E_lab = (m1 * g1 + m2 * g2) * C_SQ
    E_star = np.sqrt(E_lab * E_lab - C_SQ * p_total_sq)
    E_kin = E_star - (m1 + m2) * C_SQ
    E_ratio = E_star / ((m1 + m2) * C_SQ)
    dm, er = m1 - m2, E_ratio - 1.0 / E_ratio
    p_star_sq = m1 * m2 * C_SQ * (E_ratio * E_ratio - 1.0) + dm * dm * C_SQ / 4.0 * (er * er)
    g1s = np.sqrt(1.0 + p_star_sq / (m1 * m1 * C_SQ))
    g2s = np.sqrt(1.0 + p_star_sq / (m2 * m2 * C_SQ))
    v_rel = np.sqrt(p_star_sq) * (1.0 / (m1 * g1s) + 1.0 / (m2 * g2s))
    return E_kin, v_rel, g1s * g2s / (g1 * g2)


def bosch_hale(E, ftype, m1, m2):
    """BoschHaleFusionCrossSection [m^2] of E* [J] (0 at E* = 0)"""
    joule_to_keV = 1.e-3 / Q_E
    E_keV = np.asarray(E) * joule_to_keV
    m_reduced = m1 / (1.0 + m1 / m2)
    B_G = PI * ALPHA * np.sqrt(2.0 * m_reduced * C * C * joule_to_keV)
    A1, A2, A3, A4, A5, B1, B2, B3, B4 = BOSCH_HALE[ftype]
    with np.errstate(divide="ignore", invalid="ignore"):
        S = (A1 + E_keV * (A2 + E_keV * (A3 + E_keV * (A4 + E_keV * A5)))) / \
            (1.0 + E_keV * (B1 + E_keV * (B2 + E_keV * (B3 + E_keV * B4))))
        sig = 1.e-31 * S / E_keV * np.exp(-B_G / np.sqrt(E_keV))
    return np.where(E_keV == 0.0, 0.0, sig)


def event_probability(u1, u2, m1, m2, w1, w2, dt, dV, mult, ratio, thr, target, ftype):
    """SingleNuclearFusionEvent up to the draw: (probability, reaction weight if it fuses)"""
    E, v, f = collision_parameters(u1, u2, m1, m2)
    w_min = np.where(w2 < w1, w2, w1)
    w_max = np.where(w1 < w2, w2, w1)
    sigma = bosch_hale(E, ftype, m1, m2)
    pe = ratio.astype(np.float64) * mult * f * w_max * sigma * v * dt / dV
    mult_eff = np.full_like(pe, mult)
    hi = pe > thr
    with np.errstate(divide="ignore"):
        cand = mult * target / pe
    mult_eff = np.where(hi, np.where(cand < 1.0, 1.0, cand), mult_eff)
    pe = np.where(hi, pe * (mult_eff / mult), pe)
    with np.errstate(over="ignore"):          # a negative fit (D-D at MeV) gives -inf, no event, as in the reference
        return -np.expm1(-pe), w_min / mult_eff


def product_momenta(u1, u2, m1, m2, mA, mB, E_fusion, r_theta, r_z):
    """TwoProductFusionComputeProductMomenta with RandomizeVelocity's two uniforms: (uA, uB)"""
    u1x, u1y, u1z = u1
    u2x, u2y, u2z = u2
    E_rest_in, E_rest_out = (m1 + m2) * C_SQ, (mA + mB) * C_SQ
    g1 = np.sqrt(1.0 + (u1x * u1x + u1y * u1y + u1z * u1z) * INV_CSQ)
    g2 = np.sqrt(1.0 + (u2x * u2x + u2y * u2y + u2z * u2z) * INV_CSQ)
    p1 = [u * m1 for u in u1]
    p2 = [u * m2 for u in u2]
    s = [p1[d] + p2[d] for d in range(3)]
    p_total_sq = s[0] * s[0] + s[1] * s[1] + s[2] * s[2]
    E_lab = (m1 * g1 + m2 * g2) * C_SQ
    ef = np.sqrt(E_lab * E_lab - C_SQ * p_total_sq) - E_rest_in + E_rest_out + E_fusion
    E_ratio = np.sqrt(ef * ef) / ((mA + mB) * C_SQ)
    dm, er = mA - mB, E_ratio - 1.0 / E_ratio
    p_star_sq = mA * mB * C_SQ * (E_ratio * E_ratio - 1.0) + dm * dm * C_SQ * 0.25 * (er * er)
    vp = np.sqrt(p_star_sq)
    theta = r_theta * 2.0 * PI
    z = 2.0 * r_z - 1.0
    xy = np.sqrt(1.0 - z * z)
    ps = [xy * np.cos(theta) * vp, xy * np.sin(theta) * vp, z * vp]
    mass_g = m1 * g1 + m2 * g2
    vc = [s[d] / mass_g for d in range(3)]
    vc_sq = vc[0] * vc[0] + vc[1] * vc[1] + vc[2] * vc[2]
    with np.errstate(divide="ignore", invalid="ignore"):
        gc = 1.0 / np.sqrt(1.0 - vc_sq * INV_CSQ)
        g_star = np.sqrt(1.0 + p_star_sq / (mA * mA * C_SQ))
        vcDps = vc[0] * ps[0] + vc[1] * ps[1] + vc[2] * ps[2]
        factor = (gc - 1.0) / vc_sq * vcDps + mA * g_star * gc
    moving = vc_sq > DBL_MIN
    q = [np.where(moving, ps[d] + vc[d] * factor, ps[d]) for d in range(3)]
    return [q[d] / mA for d in range(3)], [(s[d] - q[d]) / mB for d in range(3)]


def bins_of(gcell, geom, tile):
    """bin_of_cell (csrc/bins.cuh) of global cells: supercell-major, x fastest inside a supercell"""
    n = [geom["box_hi"][d] - geom["box_lo"][d] + 1 for d in range(3)]
    nt = [(n[d] + tile[d] - 1) // tile[d] for d in range(3)]
    nc = geom["n_cell"]
    c = [gcell % nc[0] - geom["box_lo"][0], (gcell // nc[0]) % nc[1] - geom["box_lo"][1],
         gcell // (nc[0] * nc[1]) - geom["box_lo"][2]]
    t = [c[d] // tile[d] for d in range(3)]
    lc = [c[d] - t[d] * tile[d] for d in range(3)]
    tt = t[0] + nt[0] * (t[1] + nt[1] * t[2])
    return tt * (tile[0] * tile[1] * tile[2]) + lc[0] + tile[0] * (lc[1] + tile[1] * lc[2])


def _live_canonical(sp, geom):
    """storage indices of the live particles in (cell, id) order, their cells, and per cell (cell, start, count)"""
    live = np.flatnonzero(np.asarray(sp["id"]) != SPENT)
    g = cells_of({k: np.asarray(sp[k])[live] for k in ("x", "y", "z")}, geom)
    o = np.lexsort((np.asarray(sp["id"])[live], g))
    idx = live[o]
    cells, start, n = np.unique(g[o], return_index=True, return_counts=True)
    return idx, cells, start, n


def fuse(sp1, sp2, coll, geom, dt, step, tile=(8, 8, 8)):
    """One pic_collide_nuclear_fusion + pic_fusion_create_products call.  sp1 / sp2: dicts of x y z w ux uy uz id arrays
    (storage order; sp2 ignored when coll["same_species"]); coll: dict(m1, m2, mA, mB, type, fusion_multiplier,
    fusion_probability_threshold, fusion_probability_target_value, seed, collision_index, same_species).
    Returns (sp1', sp2' or None, product A, product B): the reactants with their new w and ids in storage order, the
    products in creation order (ids from 0; add the species' next id)."""
    same = bool(coll["same_species"])
    m1 = coll["m1"]
    m2 = m1 if same else coll["m2"]
    seed, cidx, ftype = int(coll["seed"]), int(coll["collision_index"]), int(coll["type"])
    dxs = [(geom["prob_hi"][d] - geom["prob_lo"][d]) / geom["n_cell"][d] for d in range(3)]
    dV = dxs[0] * dxs[1] * dxs[2]
    out1 = {k: np.array(v, copy=True) for k, v in sp1.items()}
    out2 = out1 if same else {k: np.array(v, copy=True) for k, v in sp2.items()}
    idx1, c1, st1, n1 = _live_canonical(out1, geom)
    if same:
        keep = n1 >= 2
        cells, st1, n1 = c1[keep], st1[keep], n1[keep]
        idx2, st2, n2 = idx1, st1, n1
    else:
        idx2, c2, st2, n2 = _live_canonical(out2, geom)
        cells, i1, i2 = np.intersect1d(c1, c2, assume_unique=True, return_indices=True)
        st1, n1, st2, n2 = st1[i1], n1[i1], st2[i2], n2[i2]
    perm1 = np.arange(len(idx1))
    _shuffle(perm1, st1, n1, seed, step, cells, cidx, 0)
    if same:
        perm2 = perm1
        half = n1 // 2
        base1, base2, NI1, NI2 = st1, st1 + half, half, n1 - half
    else:
        perm2 = np.arange(len(idx2))
        _shuffle(perm2, st2, n2, seed, step, cells, cidx, 1)
        base1, base2, NI1, NI2 = st1, st2, n1, n2
    maxN, minN = np.maximum(NI1, NI2), np.minimum(NI1, NI2)
    ratio = (minN + maxN - 1) if same else minN
    chain_cell = np.repeat(np.arange(len(cells)), minN)
    first = np.cumsum(minN) - minN
    cc = np.arange(len(chain_cell)) - np.repeat(first, minN)
    rng = Streams(seed, step, cells[chain_cell], cidx, 2 + cc)
    w1, w2 = out1["w"], out2["w"]
    U1 = [out1[k] for k in ("ux", "uy", "uz")]
    U2 = [out2[k] for k in ("ux", "uy", "uz")]
    dead1 = np.zeros(len(w1), dtype=bool)
    dead2 = dead1 if same else np.zeros(len(w2), dtype=bool)
    ev_cell, ev_k, ev_a, ev_b, ev_wr = [], [], [], [], []
    sstep = 0
    while True:
        k = cc + sstep * minN[chain_cell]
        act = np.flatnonzero(k < maxN[chain_cell])
        if act.size == 0:
            break
        cl = chain_cell[act]
        i1 = cc[act] + np.where(maxN[cl] == NI1[cl], sstep * minN[cl], 0)
        i2 = cc[act] + np.where(maxN[cl] == NI2[cl], sstep * minN[cl], 0)
        a, b = idx1[perm1[base1[cl] + i1]], idx2[perm2[base2[cl] + i2]]
        go = ~dead1[a] & ~dead2[b]
        g = np.flatnonzero(go)
        if g.size:
            A, B = a[g], b[g]
            prob, wr = event_probability([u[A] for u in U1], [u[B] for u in U2], m1, m2, w1[A], w2[B], dt, dV,
                                         coll["fusion_multiplier"], ratio[cl[g]], coll["fusion_probability_threshold"],
                                         coll["fusion_probability_target_value"], ftype)
            r = rng.uniform(act[g])
            hit = r < prob
            A, B, wr = A[hit], B[hit], wr[hit]
            w1[A] = w1[A] + -wr
            dead1[A[w1[A] <= DBL_MIN]] = True
            w2[B] = w2[B] + -wr
            dead2[B[w2[B] <= DBL_MIN]] = True
            ev_cell.append(cl[g][hit]); ev_k.append(k[act][g][hit]); ev_a.append(A); ev_b.append(B); ev_wr.append(wr)
        sstep += 1
    out1["id"][dead1] = SPENT
    if not same:
        out2["id"][dead2] = SPENT
    cat = (lambda v, dt_: np.concatenate(v) if v else np.zeros(0, dtype=dt_))
    ecell, ek, ea, eb, ewr = (cat(ev_cell, np.int64), cat(ev_k, np.int64), cat(ev_a, np.int64), cat(ev_b, np.int64),
                              cat(ev_wr, np.float64))
    gcell = cells[ecell]
    order = np.lexsort((ek, bins_of(gcell, geom, tile)))
    gcell, ea, eb, ewr, ecell = gcell[order], ea[order], eb[order], ewr[order], ecell[order]
    # in-cell event index j
    j = np.zeros(len(order), dtype=np.int64)
    if len(order):
        newc = np.r_[True, ecell[1:] != ecell[:-1]]
        starts = np.flatnonzero(newc)
        j = np.arange(len(order)) - np.repeat(starts, np.diff(np.r_[starts, len(order)]))
    prng = Streams(seed, step, gcell, cidx, np.uint64(1 << 62) | j.astype(np.uint64))
    sel = np.arange(len(order))
    r_theta = prng.uniform(sel)
    r_z = prng.uniform(sel)
    uA, uB = product_momenta([u[ea] for u in U1], [u[eb] for u in U2], m1, m2, coll["mA"], coll["mB"],
                             E_FUSION[ftype], r_theta, r_z)
    prods = []
    for u in (uA, uB):
        p = {}
        for name, src in (("x", "x"), ("y", "y"), ("z", "z")):
            p[name] = np.stack([out1[src][ea], out2[src][eb]], axis=1).ravel()
        for d, name in enumerate(("ux", "uy", "uz")):
            p[name] = np.repeat(u[d], 2)
        p["w"] = np.repeat(ewr / 2.0, 2)
        p["id"] = np.arange(2 * len(order), dtype=np.int64)
        prods.append(p)
    return out1, (None if same else out2), prods[0], prods[1]
