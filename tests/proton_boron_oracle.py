"""TEST INFRASTRUCTURE -- numpy restatement of the proton-boron fusion stage (csrc/fusion.cu, PIC_FUSION_PB_3HE4): the
event pass with ProtonBoronFusionCrossSection.H and the product pass of ParticleCreationFunc.H:170-200 with
ProtonBoronFusionInitializeMomentum.H, vectorised over cells and pair chains.

The pairing, the streams, the spent marking and the event order are those of tests/fusion_oracle.py (the project's
determinism contract).  The products of the cell's j-th event draw four uniforms from the stream of tag 2^62 | j: theta
and z of the alpha + 8Be* emission, then theta and z of the 8Be* decay.  Event e writes alpha k (k = 0, 1, 2) at slots
6e + 2k (reactant 1's position) and 6e + 2k + 1 (reactant 2's).  Expressions keep the kernel's evaluation order."""
import numpy as np

import fusion_oracle as fo
from collision_oracle import Streams, _shuffle

C = fo.C
C_SQ = fo.C_SQ
Q_E = fo.Q_E
PI = fo.PI
DBL_MIN = fo.DBL_MIN
SPENT = fo.SPENT
M_U = 1.66053906660e-27
EP0 = 8.8541878128e-12
HBAR = 1.054571817e-34
PB_3HE4 = 3
MEV_TO_JOULE = Q_E * 1.e6
E_FUSION = 5.55610759 * MEV_TO_JOULE        # p + B11 -> alpha + 8Be*
E_DECAY = 3.12600414 * MEV_TO_JOULE         # 8Be* -> 2 alpha
M_ALPHA = M_U * 4.00260325413
M_BE = M_U * (8.0053095729 + 0.00325283863)
Q_TOTAL = E_FUSION + E_DECAY                # the kinetic energy the three alphas gain


def tentori(E_keV):
    """ProtonBoronFusionCrossSectionTentori [barn] of E* in keV (0 at E* = 0)"""
    E_keV = np.asarray(E_keV, dtype=np.float64)
    E_MeV = E_keV * 1.e-3
    joule_to_MeV = 1.e-6 / Q_E
    m_boron, m_hydrogen = 11.00930536 * M_U, 1.00782503223 * M_U
    m_reduced = m_boron / (1.0 + m_boron / m_hydrogen)
    a = Q_E * Q_E * 5.0 / (2.0 * EP0 * HBAR)
    gamow = m_reduced / 2.0 * a * a * joule_to_MeV
    low = 197.0 + 0.269 * E_keV + 2.54e-4 * (E_keV * E_keV) + 1.82e4 / ((E_keV - 148.0) * (E_keV - 148.0) + 2.35 * 2.35)
    En = (E_keV - 400.0) * 1.e-2
    En2 = En * En
    mid = 346.0 + 150.0 * En + -59.9 * En2 + -0.460 * (En * (En2 * En2))
    high = (1.98e6 / ((E_keV - 640.9) * (E_keV - 640.9) + 85.5 * 85.5) +
            3.89e6 / ((E_keV - 1211.0) * (E_keV - 1211.0) + 414.0 * 414.0) +
            1.36e6 / ((E_keV - 2340.0) * (E_keV - 2340.0) + 221.0 * 221.0) +
            3.71e6 / ((E_keV - 3294.0) * (E_keV - 3294.0) + 351.0 * 351.0) + 0.381)
    S = np.where(E_keV < 400.0, low, np.where(E_keV < 668.0, mid, high))
    with np.errstate(divide="ignore", invalid="ignore"):
        sig = S / E_MeV * np.exp(-np.sqrt(gamow / E_MeV))
    return np.where(E_keV == 0.0, 0.0, sig)


def cross_section(E):
    """ProtonBoronFusionCrossSection [m^2] of E* [J]: Tentori up to 9.76 MeV, Buck's power law above"""
    E_keV = np.asarray(E, dtype=np.float64) * (1.e-3 / Q_E)
    with np.errstate(divide="ignore", invalid="ignore"):
        buck = 0.01277998 * np.power(E_keV / 9760.0, -2.661840717596765)
    return np.where(E_keV <= 9760.0, tentori(E_keV), buck) * 1.e-28


def event_probability(u1, u2, m1, m2, w1, w2, dt, dV, mult, ratio, thr, target):
    """SingleNuclearFusionEvent up to the draw: (probability, reaction weight if it fuses)"""
    E, v, f = fo.collision_parameters(u1, u2, m1, m2)
    w_min = np.where(w2 < w1, w2, w1)
    w_max = np.where(w1 < w2, w2, w1)
    pe = ratio.astype(np.float64) * mult * f * w_max * cross_section(E) * v * dt / dV
    hi = pe > thr
    with np.errstate(divide="ignore"):
        cand = mult * target / pe
    mult_eff = np.where(hi, np.where(cand < 1.0, 1.0, cand), mult)
    pe = np.where(hi, pe * (mult_eff / mult), pe)
    return -np.expm1(-pe), w_min / mult_eff


def alpha_momenta(u1, u2, m1, m2, r):
    """ProtonBoronFusionInitializeMomentum with the four uniforms r[0..3]: [u of alpha 0, 1, 2], each (ux, uy, uz)"""
    u0, uBe = fo.product_momenta(u1, u2, m1, m2, M_ALPHA, M_BE, E_FUSION, r[0], r[1])
    pBe = [M_BE * u for u in uBe]
    gamma_s = 1.0 + 0.5 * E_DECAY / (M_ALPHA * C_SQ)
    p_s = M_ALPHA * C * np.sqrt(gamma_s * gamma_s - 1.0)
    theta = r[2] * 2.0 * PI
    z = 2.0 * r[3] - 1.0
    xy = np.sqrt(1.0 - z * z)
    ps = [xy * np.cos(theta) * p_s, xy * np.sin(theta) * p_s, z * p_s]
    p_Be_sq = pBe[0] * pBe[0] + pBe[1] * pBe[1] + pBe[2] * pBe[2]
    g_Be = np.sqrt(1.0 + p_Be_sq / ((M_BE * M_BE) * C_SQ))
    mg = M_BE * g_Be
    v = [p / mg for p in pBe]
    v_sq = v[0] * v[0] + v[1] * v[1] + v[2] * v[2]
    with np.errstate(divide="ignore", invalid="ignore"):
        factor = (g_Be - 1.0) / v_sq * (v[0] * ps[0] + v[1] * ps[1] + v[2] * ps[2]) + M_ALPHA * gamma_s * g_Be
    moving = v_sq > DBL_MIN
    p2 = [np.where(moving, ps[d] + v[d] * factor, ps[d]) for d in range(3)]
    return [u0, [p / M_ALPHA for p in p2], [(pBe[d] - p2[d]) / M_ALPHA for d in range(3)]]


def fuse(sp1, sp2, coll, geom, dt, step, tile=(8, 8, 8)):
    """One pic_collide_nuclear_fusion + pic_fusion_create_products call of type PB_3HE4 (sp1 and sp2 are the proton and
    the boron species, in either order).  Returns (sp1', sp2', alphas): the reactants with their new w and ids in storage
    order, the alphas in creation order (ids from 0; add the species' next id)."""
    m1, m2 = coll["m1"], coll["m2"]
    seed, cidx = int(coll["seed"]), int(coll["collision_index"])
    dxs = [(geom["prob_hi"][d] - geom["prob_lo"][d]) / geom["n_cell"][d] for d in range(3)]
    dV = dxs[0] * dxs[1] * dxs[2]
    out1 = {k: np.array(v, copy=True) for k, v in sp1.items()}
    out2 = {k: np.array(v, copy=True) for k, v in sp2.items()}
    idx1, c1, st1, n1 = fo._live_canonical(out1, geom)
    idx2, c2, st2, n2 = fo._live_canonical(out2, geom)
    cells, i1, i2 = np.intersect1d(c1, c2, assume_unique=True, return_indices=True)
    st1, NI1, st2, NI2 = st1[i1], n1[i1], st2[i2], n2[i2]
    perm1, perm2 = np.arange(len(idx1)), np.arange(len(idx2))
    _shuffle(perm1, st1, NI1, seed, step, cells, cidx, 0)
    _shuffle(perm2, st2, NI2, seed, step, cells, cidx, 1)
    maxN, minN = np.maximum(NI1, NI2), np.minimum(NI1, NI2)
    chain_cell = np.repeat(np.arange(len(cells)), minN)
    cc = np.arange(len(chain_cell)) - np.repeat(np.cumsum(minN) - minN, minN)
    rng = Streams(seed, step, cells[chain_cell], cidx, 2 + cc)
    w1, w2 = out1["w"], out2["w"]
    U1 = [out1[k] for k in ("ux", "uy", "uz")]
    U2 = [out2[k] for k in ("ux", "uy", "uz")]
    dead1, dead2 = np.zeros(len(w1), dtype=bool), np.zeros(len(w2), dtype=bool)
    ev = []
    sstep = 0
    while True:
        k = cc + sstep * minN[chain_cell]
        act = np.flatnonzero(k < maxN[chain_cell])
        if act.size == 0:
            break
        cl = chain_cell[act]
        j1 = cc[act] + np.where(maxN[cl] == NI1[cl], sstep * minN[cl], 0)
        j2 = cc[act] + np.where(maxN[cl] == NI2[cl], sstep * minN[cl], 0)
        a, b = idx1[perm1[st1[cl] + j1]], idx2[perm2[st2[cl] + j2]]
        g = np.flatnonzero(~dead1[a] & ~dead2[b])
        if g.size:
            A, B = a[g], b[g]
            prob, wr = event_probability([u[A] for u in U1], [u[B] for u in U2], m1, m2, w1[A], w2[B], dt, dV,
                                         coll["fusion_multiplier"], minN[cl[g]], coll["fusion_probability_threshold"],
                                         coll["fusion_probability_target_value"])
            hit = rng.uniform(act[g]) < prob
            A, B, wr = A[hit], B[hit], wr[hit]
            w1[A] = w1[A] + -wr
            dead1[A[w1[A] <= DBL_MIN]] = True
            w2[B] = w2[B] + -wr
            dead2[B[w2[B] <= DBL_MIN]] = True
            ev.append((cl[g][hit], k[act][g][hit], A, B, wr))
        sstep += 1
    out1["id"][dead1] = SPENT
    out2["id"][dead2] = SPENT
    ecell, ek, ea, eb = (np.concatenate([e[i] for e in ev]) if ev else np.zeros(0, dtype=np.int64) for i in range(4))
    ewr = np.concatenate([e[4] for e in ev]) if ev else np.zeros(0)
    gcell = cells[ecell]
    order = np.lexsort((ek, fo.bins_of(gcell, geom, tile)))
    gcell, ea, eb, ewr, ecell = gcell[order], ea[order], eb[order], ewr[order], ecell[order]
    j = np.zeros(len(order), dtype=np.int64)
    if len(order):
        starts = np.flatnonzero(np.r_[True, ecell[1:] != ecell[:-1]])
        j = np.arange(len(order)) - np.repeat(starts, np.diff(np.r_[starts, len(order)]))
    prng = Streams(seed, step, gcell, cidx, np.uint64(1 << 62) | j.astype(np.uint64))
    sel = np.arange(len(order))
    r = [prng.uniform(sel) for _ in range(4)]
    ua = alpha_momenta([u[ea] for u in U1], [u[eb] for u in U2], m1, m2, r)
    n = len(order)
    alphas = {}
    for name in ("x", "y", "z"):
        pair = np.stack([out1[name][ea], out2[name][eb]], axis=1)          # [event, side]
        alphas[name] = np.repeat(pair[:, None, :], 3, axis=1).ravel()
    for d, name in enumerate(("ux", "uy", "uz")):
        per = np.stack([ua[al][d] for al in range(3)], axis=1)              # [event, alpha]
        alphas[name] = np.repeat(per, 2, axis=1).ravel()
    alphas["w"] = np.repeat(ewr / 2.0, 6)
    alphas["id"] = np.arange(6 * n, dtype=np.int64)
    return out1, out2, alphas
