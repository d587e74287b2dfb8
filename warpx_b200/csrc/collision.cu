// Binary Coulomb collisions (collisions.collision_names, <name>.type = pairwisecoulomb) over the rank's box.
//
// Restates, for one tile = the rank's box (paths relative to Source/Particles/Collision/ of ECP-WarpX/WarpX):
//   the cell walk             <- BinaryCollision::doCollisionsWithinTile     BinaryCollision/BinaryCollision.H:234-750
//   (binary_collision.cuh)       (intra-species :287-490, inter-species :491-750), ShuffleFisherYates.H
//   PairwiseCoulomb           <- PairWiseCoulombCollisionFunc with ElasticCollisionPerez  Coulomb/ElasticCollisionPerez.H:57-148
//   PairwiseCoulomb::species  <- the density loops :395-403, :626-642 and ComputeTemperature (Coulomb/ComputeTemperature.H)
//   perez_update              <- UpdateMomentumPerezElastic                  Coulomb/UpdateMomentumPerezElastic.H
//
// Determinism: the result is a function of (the particles of each cell by id, seed, collision index, step, global
// cell) and nothing else -- not of the storage order, the thread mapping or the decomposition:
//   * canonical order: a cell's particles of each species are first put in ascending id order (the cell sort leaves
//     them in whatever order its warp-aggregated atomics produced), then shuffled;
//   * random streams: Philox4x64-10 (philox.cuh) keyed by (seed, 0), counter (j + 1, step, global cell index
//     i + nx (j + ny k), 2^63 | collision index << 32 | tag) for block j of a stream.  Tag 0 and 1 shuffle species 1
//     and 2; tag 2 + c is independent pair chain c, consumed 4 words per block in order.  Bit 63 of the last word keeps
//     these streams apart from the counters (j + 1, 0, 0, 0) that initial conditions draw from under the same seed;
//   * conversions: amrex::Random = ((w >> 11) + 1) 2^-53 in (0, 1] (curand_uniform_double's range, which AMReX uses
//     on GPUs), Random_int(n) = floor(((w >> 11) 2^-53) n);
//   * sums (density, temperature) run sequentially in canonical order; the file is compiled without FMA contraction.
//
// One pass of the cell walk of binary_collision.cuh over the binned particles, which takes every particle of a cell
// and writes ux, uy, uz back to where it read them.  x, y, z, w, ids, cell_start and src are never written.
#include "binary_collision.cuh"

namespace pic {

namespace coll {

// The Perez (2012) momentum update of one pair, with the computed Coulomb logarithm when L <= 0 and the weighted
// rejection of unequal weights; expression order as in UpdateMomentumPerezElastic.H.
__host__ __device__ __forceinline__ void perez_update(double& u1x, double& u1y, double& u1z, double& u2x, double& u2y,
                                                      double& u2z, double q1, double m1, double w1, double q2, double m2,
                                                      double w2, double n12, double sigma_max, double L, double bmax,
                                                      double dt, Stream& rng) {
    const double g1sq = (u1x * u1x + u1y * u1y + u1z * u1z) * INV_C2;
    const double g2sq = (u2x * u2x + u2y * u2y + u2z * u2z) * INV_C2;
    const double g1 = sqrt(1.0 + g1sq), g2 = sqrt(1.0 + g2sq);
    const double dx = u1x - u2x, dy = u1y - u2y, dz = u1z - u2z;
    const double dm = sqrt((dx * dx + dy * dy + dz * dz) * INV_C2);
    const double sm = sqrt(g1sq) + sqrt(g2sq);
    if (dm < DBL_MIN_ || dm / sm < 1.0e-10) return;            // identical momenta: no collision

    const double p1x = u1x * m1, p1y = u1y * m1, p1z = u1z * m1;
    const double p2x = u2x * m2, p2y = u2y * m2, p2z = u2z * m2;
    // centre-of-momentum velocity and Lorentz factor
    const double mg = m1 * g1 + m2 * g2;
    const double vx = (p1x + p2x) / mg, vy = (p1y + p2y) / mg, vz = (p1z + p2z) / mg;
    const double v2 = vx * vx + vy * vy + vz * vz;
    const double gc = 1.0 / sqrt(1.0 - v2 * INV_C2);
    const double vdv1 = (vx * u1x + vy * u1y + vz * u1z) / g1;
    const double vdv2 = (vx * u2x + vy * u2y + vz * u2z) / g2;
    // p1 in the centre-of-momentum frame, (gc - 1)/v^2 written as gc^2/(c^2 (1 + gc))
    const double lt = (gc * gc * vdv1 * INV_C2 / (1.0 + gc) - gc) * m1 * g1;
    const double s1x = p1x + vx * lt, s1y = p1y + vy * lt, s1z = p1z + vz * lt;
    const double s1m = sqrt(s1x * s1x + s1y * s1y + s1z * s1z);
    const double g1s = (1.0 - vdv1 * INV_C2) * gc * g1;
    const double g2s = (1.0 - vdv2 * INV_C2) * gc * g2;
    const double mu = g1s * m1 * g2s * m2 / (g1s * m1 + g2s * m2);
    const double vrel = s1m / mu;
    const double den = 1.0 + s1m * s1m / (m1 * g1s * m2 * g2s) * INV_C2;
    const double vrel_inv = vrel / den;

    double s12 = 0.0;
    if (s1m > DBL_MIN_) {
        const double aq = q1 * q2 < 0 ? -(q1 * q2) : q1 * q2;
        const double b0 = aq / (2.0 * PI * EP0 * mu * vrel * vrel_inv);
        double lnL;
        if (L > 0.0) lnL = L;
        else {
            const double bmin_qm = HBAR * 0.5 / s1m;
            const double bmin = dmax(bmin_qm, 0.5 * b0);
            lnL = dmax(2.0, 0.5 * log(1.0 + bmax * bmax / (bmin * bmin)));
        }
        const double sig = dmin(PI * b0 * b0 * lnL, sigma_max);
        s12 = sig * n12 * dt * vrel * g1s * g2s / (g1 * g2);
    }
    if (!(s12 > DBL_MIN_)) return;

    double r = rng.uniform();
    double cx;                                                  // cos of the scattering angle
    if (s12 <= 0.1) {
        while (true) {
            cx = 1.0 + s12 * log(r);
            if (cx >= -1.0) break;                              // r so small that cos < -1: draw again
            r = rng.uniform();
        }
    } else if (s12 > 0.1 && s12 <= 3.0) {
        const double ai = 0.0056958 + 0.9560202 * s12 - 0.508139 * s12 * s12 + 0.47913906 * s12 * s12 * s12 -
                          0.12788975 * s12 * s12 * s12 * s12 + 0.02389567 * s12 * s12 * s12 * s12 * s12;
        cx = ai * log(exp(-1.0 / ai) + 2.0 * r * sinh(1.0 / ai));
    } else if (s12 > 3.0 && s12 <= 6.0) {
        const double A = 3.0 * exp(-s12);
        cx = 1.0 / A * log(exp(-A) + 2.0 * r * sinh(A));
    } else {
        cx = 2.0 * r - 1.0;
    }
    const double sx = sqrt(1.0 - cx * cx);
    const double phi = rng.uniform() * 2.0 * PI;
    double cp, sp;
#ifdef __CUDA_ARCH__
    sincos(phi, &sp, &cp);
#else
    sp = sin(phi); cp = cos(phi);
#endif
    double f1x, f1y, f1z;
    double pp = sqrt(s1x * s1x + s1y * s1y);
    if (pp > DBL_MIN_) {
        f1x = (s1x * s1z / pp) * sx * cp + (s1y * s1m / pp) * sx * sp + (s1x) * cx;
        f1y = (s1y * s1z / pp) * sx * cp + (-s1x * s1m / pp) * sx * sp + (s1y) * cx;
        f1z = (-pp) * sx * cp + (0.0) * sx * sp + (s1z) * cx;
    } else {                                                    // p1* along z: rotate the axes x -> y -> z -> x
        pp = sqrt(s1y * s1y + s1z * s1z);
        f1y = (s1y * s1x / pp) * sx * cp + (s1z * s1m / pp) * sx * sp + (s1y) * cx;
        f1z = (s1z * s1x / pp) * sx * cp + (-s1y * s1m / pp) * sx * sp + (s1z) * cx;
        f1x = (-pp) * sx * cp + (0.0) * sx * sp + (s1x) * cx;
    }
    const double f2x = -f1x, f2y = -f1y, f2z = -f1z;
    // back to the lab frame
    const double vdf1 = vx * f1x + vy * f1y + vz * f1z;
    const double vdf2 = vx * f2x + vy * f2y + vz * f2z;
    const double fac = gc * gc * INV_C2 / (gc + 1.0);
    const double fac1 = fac * vdf1 + m1 * g1s * gc;
    const double fac2 = fac * vdf2 + m2 * g2s * gc;
    const double q1x = f1x + vx * fac1, q1y = f1y + vy * fac1, q1z = f1z + vz * fac1;
    const double q2x = f2x + vx * fac2, q2y = f2y + vy * fac2, q2z = f2z + vz * fac2;
    // each side keeps its new momentum with probability (its partner's weight) / (the larger weight)
    const double wmax = dmax(w1, w2);
    r = rng.uniform();
    if (w2 > r * wmax) { u1x = q1x / m1; u1y = q1y / m1; u1z = q1z / m1; }
    r = rng.uniform();
    if (w1 > r * wmax) { u2x = q2x / m2; u2y = q2y / m2; u2z = q2z / m2; }
}

// The cell walk's functor (binary_collision.cuh) for PairWiseCoulombCollisionFunc.
struct PairwiseCoulomb {
    struct Args : PairArgs {
        double q1, q2, L;
    };
    static constexpr bool skip_spent = false;
    struct Scalars { double n[2], T[2]; };   // density and temperature of each species

    // n = sum w / dV and (for a computed Coulomb log) the temperature, sequentially over the n particles in canonical
    // order
    template <class V>
    __device__ static void species(const Args& a, const V& v, int sp, const int* I, int n, Scalars& x) {
        double wt = 0.0;
        for (int i = 0; i < n; ++i) wt += v.w(sp, I[i]);
        x.n[sp - 1] = wt / a.dV;
        x.T[sp - 1] = 0.0;
        if (a.L < 0.0) {             // m_computeSpeciesTemperatures: CoulombLog < 0 (PairWiseCoulombCollisionFunc.H)
            double vx = 0.0, vy = 0.0, vz = 0.0, vs = 0.0, wtot = 0.0;
            for (int i = 0; i < n; ++i) {
                const int k = I[i];
                const double w = v.w(sp, k), ux = v.ux(sp, k), uy = v.uy(sp, k), uz = v.uz(sp, k);
                const double us = ux * ux + uy * uy + uz * uz;
                const double gm = sqrt(1.0 + us * INV_C2);
                wtot += w;
                vx += w * ux / gm;
                vy += w * uy / gm;
                vz += w * uz / gm;
                vs += w * us / gm / gm;
            }
            vx = vx / wtot; vy = vy / wtot; vz = vz / wtot; vs = vs / wtot;
            x.T[sp - 1] = (sp == 1 ? a.m1 : a.m2) / 3.0 * (vs - (vx * vx + vy * vy + vz * vz));
        }
    }

    double bmax, sigma_max, q2, m2, pairs;

    // the cell's screening from its densities and temperatures (ElasticCollisionPerez.H:57-148)
    __device__ PairwiseCoulomb(const Args& a, long, const Scalars& x, int minN, int maxN) {
        const double dn1 = x.n[0], T1 = x.T[0];
        const double dn2 = a.same ? dn1 : x.n[1], T2 = a.same ? T1 : x.T[1];
        double lmdD = -1.0;
        if (a.L <= 0.0) lmdD = 1.0 / sqrt(dn1 * a.q1 * a.q1 / (T1 * EP0) + dn2 * a.q2 * a.q2 / (T2 * EP0));
        const double maxn = dmax(dn1, dn2);
        const double rmin = 1.0 / cbrt(4.0 * PI / 3.0 * maxn);
        bmax = dmax(lmdD, rmin);
        sigma_max = 1.0 / (maxn * rmin);
        q2 = a.same ? a.q1 : a.q2;
        m2 = a.same ? a.m1 : a.m2;
        pairs = (double)(a.same ? minN + maxN - 1 : minN);
    }

    template <class V>
    __device__ void pair(const Args& a, const V& v, int e1, int e2, int, Stream& rng) const {
        const double wpmax = dmax(v.w(1, e1), v.w(2, e2));
        const double n12 = wpmax * pairs / a.dV;
        perez_update(v.ux(1, e1), v.uy(1, e1), v.uz(1, e1), v.ux(2, e2), v.uy(2, e2), v.uz(2, e2), a.q1, a.m1,
                     v.w(1, e1), q2, m2, v.w(2, e2), n12, sigma_max, a.L, bmax, a.dt, rng);
    }

    template <int G> __device__ void end_cell(const Args&, long, int, Scalars&) const { group_sync<G>(); }

    template <class V>
    __device__ static void store(const Args& a, const V& v, int sp, int e) {
        const SoaView& P = sp == 1 ? a.P1 : a.P2;
        const int p = v.storage(sp, e);
        P.ux[p] = v.ux(sp, e); P.uy[p] = v.uy(sp, e); P.uz[p] = v.uz(sp, e);
    }
};

}  // namespace coll
}  // namespace pic

using namespace pic;

extern "C" int pic_collide_pairwise_coulomb(const pic_coulomb_collision* c, const pic_soa* p1, const pic_bins* b1,
                                            const int* src1, const pic_soa* p2, const pic_bins* b2, const int* src2,
                                            const pic_geom* g, double dt, long step, int* scratch1, int* scratch2,
                                            int* status, void* stream) {
    const char* what = "pic_collide_pairwise_coulomb";
    coll::PairwiseCoulomb::Args a;
    if (int rc = coll::pair_args(what, c, p1, b1, src1, p2, b2, src2, g, dt, step, scratch1, scratch2, status, a))
        return rc;
    PIC_REQUIRE(c->m1 > 0.0 && (c->same_species || c->m2 > 0.0), "%s: masses must be positive", what);
    a.q1 = c->q1; a.q2 = c->q2; a.L = c->coulomb_log;
    if (p1->np == 0 || (!c->same_species && p2->np == 0)) return 0;
    return coll::launch<coll::PairwiseCoulomb>(what, a, (cudaStream_t)stream);
}
