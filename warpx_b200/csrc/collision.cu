// Binary Coulomb collisions (collisions.collision_names, <name>.type = pairwisecoulomb) over the rank's box.
//
// Restates, for one tile = the rank's box (paths relative to Source/Particles/Collision/ of ECP-WarpX/WarpX):
//   collide_cell            <- BinaryCollision::doCollisionsWithinTile     BinaryCollision/BinaryCollision.H:234-750
//                              (intra-species :287-490, inter-species :491-750) with PairWiseCoulombCollisionFunc
//   cell_density_temperature <- the density loops :395-403, :626-642 and ComputeTemperature (Coulomb/ComputeTemperature.H)
//   shuffle                 <- ShuffleFisherYates                          BinaryCollision/ShuffleFisherYates.H
//   chain                   <- ElasticCollisionPerez                       Coulomb/ElasticCollisionPerez.H:57-148
//   perez_update            <- UpdateMomentumPerezElastic                  Coulomb/UpdateMomentumPerezElastic.H
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
// One pass over the binned particles: a warp takes a cell of at most SMALL_CAP particles, a 256-thread block a cell of
// at most LARGE_CAP.  Each group loads its cell through the pending permutation src (when there is one), ranks the
// particles by id in shared memory, shuffles there, walks the independent pair chains on the shared copy and writes
// ux, uy, uz back to where it read them.  A cell beyond LARGE_CAP takes a block that keeps only the cell's canonical
// order in global memory -- the caller's per-slot int scratch at the cell's own slots, so cells never share it -- and
// reads and writes the particles there; same arithmetic, same draws, same result.  x, y, z, w, ids, cell_start and
// src are never written.
#include "binary_collision.cuh"

namespace pic {

namespace coll {

constexpr int SMALL_CAP = 64;          // particles of a cell (both species) a warp handles
constexpr int SMALL_WARPS = 4;         // warps per block of the small-cell kernel
constexpr int LARGE_CAP = 2048;        // particles of a cell a block handles
constexpr int LARGE_THREADS = 256;
constexpr int LARGE_SCAN = 32;         // bins a block of the large-cell kernel looks at per round

struct Args {
    SoaView P1, P2;
    const uint64_t* id1; const uint64_t* id2;
    const int* src1; const int* src2;   // slot -> storage index, or null
    int* scr1; int* scr2;               // one int per slot (cells beyond LARGE_CAP), or null
    BinsView b1, b2;
    int gn[2];                          // global cells along x, y (stream counter)
    double q1, m1, q2, m2, L, dt, dV;
    uint64_t seed, cidx;
    uint64_t step;
    int same;
    int* status;
};

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

// Shared memory of one group for `cap` particles: w ux uy uz (canonical order), ids (load order), 4 cell scalars,
// storage index (load order), storage index (canonical order), shuffled positions.
__host__ __device__ constexpr size_t group_bytes(int cap) { return (size_t)cap * (4 * 8 + 8 + 3 * 4) + 4 * 8; }

struct Group {
    double *w, *ux, *uy, *uz, *scal;
    uint64_t* key;
    int *lp, *pp, *sh;
    __device__ Group(char* base, int cap) {
        double* d = reinterpret_cast<double*>(base);
        w = d; ux = d + cap; uy = d + 2 * cap; uz = d + 3 * cap;
        key = reinterpret_cast<uint64_t*>(d + 4 * cap);
        scal = reinterpret_cast<double*>(key + cap);
        lp = reinterpret_cast<int*>(scal + 4); pp = lp + cap; sh = pp + cap;
    }
};

// particles of the cell's species 1 (and 2) the collision takes part in; 0 when nothing collides there
__device__ __forceinline__ int cell_load(const Args& a, long bin, long* cs1, int* n1, long* cs2, int* n2) {
    *cs1 = a.b1.cell_start[bin];
    *n1 = a.b1.cell_start[bin + 1] - (int)*cs1;
    if (a.same) { *cs2 = *cs1; *n2 = 0; return *n1 >= 2 ? *n1 : 0; }
    *cs2 = a.b2.cell_start[bin];
    *n2 = a.b2.cell_start[bin + 1] - (int)*cs2;
    return (*n1 >= 1 && *n2 >= 1) ? *n1 + *n2 : 0;
}

// n = sum w / dV and (for a computed Coulomb log) the temperature, sequentially over the n particles in canonical
// order -- element i is w[idx[i]] (w[i] when idx is null) -- then the Fisher-Yates shuffle of sh[0, n) with the stream
// of `tag` (sh may be idx itself: the sums are done before it changes)
__device__ void cell_density_temperature_shuffle(const Args& g, const double* w, const double* ux, const double* uy,
                                                 const double* uz, const int* idx, int* sh, int n, double m,
                                                 uint64_t gcell, int tag, double* n_out, double* T_out) {
    double wt = 0.0;
    for (int i = 0; i < n; ++i) wt += w[idx ? idx[i] : i];
    *n_out = wt / g.dV;
    *T_out = 0.0;
    if (g.L < 0.0) {                 // m_computeSpeciesTemperatures: CoulombLog < 0 (PairWiseCoulombCollisionFunc.H)
        double vx = 0.0, vy = 0.0, vz = 0.0, vs = 0.0, wtot = 0.0;
        for (int i = 0; i < n; ++i) {
            const int k = idx ? idx[i] : i;
            const double us = ux[k] * ux[k] + uy[k] * uy[k] + uz[k] * uz[k];
            const double gm = sqrt(1.0 + us * INV_C2);
            wtot += w[k];
            vx += w[k] * ux[k] / gm;
            vy += w[k] * uy[k] / gm;
            vz += w[k] * uz[k] / gm;
            vs += w[k] * us / gm / gm;
        }
        vx = vx / wtot; vy = vy / wtot; vz = vz / wtot; vs = vs / wtot;
        *T_out = m / 3.0 * (vs - (vx * vx + vy * vy + vz * vz));
    }
    Stream rng(g.seed, g.step, gcell, (g.cidx << 32) | (uint64_t)tag);
    for (int i = n - 1; i >= 1; --i) {
        const int j = rng.random_int(i + 1);
        const int t = sh[i]; sh[i] = sh[j]; sh[j] = t;
    }
}

// The independent pair chains of one cell (ElasticCollisionPerez.H:57-148), chain c by thread c, c + G, ...: the
// cell's screening from its densities and temperatures, then pairs (I1[i1], I2[i2]) of the index sets -- halves of the
// shuffled cell, or the two shuffled species -- into the arrays of species 1 (w1, u1) and 2 (w2, u2).
template <int G>
__device__ void chains(const Args& a, int t, uint64_t gcell, double dn1, double dn2, double T1, double T2,
                       const int* I1, const int* I2, int NI1, int NI2, const double* w1, double* u1x, double* u1y,
                       double* u1z, const double* w2, double* u2x, double* u2y, double* u2z) {
    double lmdD = -1.0;
    if (a.L <= 0.0) lmdD = 1.0 / sqrt(dn1 * a.q1 * a.q1 / (T1 * EP0) + dn2 * a.q2 * a.q2 / (T2 * EP0));
    const double maxn = dmax(dn1, dn2);
    const double rmin = 1.0 / cbrt(4.0 * PI / 3.0 * maxn);
    const double bmax = dmax(lmdD, rmin);
    const double sigma_max = 1.0 / (maxn * rmin);
    const int maxN = NI1 > NI2 ? NI1 : NI2, minN = NI1 < NI2 ? NI1 : NI2;
    const double q2 = a.same ? a.q1 : a.q2, m2 = a.same ? a.m1 : a.m2;
    for (int c = t; c < minN; c += G) {
        Stream rng(a.seed, a.step, gcell, (a.cidx << 32) | (uint64_t)(2 + c));
        int i1 = c, i2 = c;
        for (int k = c; k < maxN; k += minN) {
            const int e1 = I1[i1], e2 = I2[i2];
            const double wpmax = dmax(w1[e1], w2[e2]);
            const double n12 = a.same ? wpmax * (double)(minN + maxN - 1) / a.dV : wpmax * (double)minN / a.dV;
            perez_update(u1x[e1], u1y[e1], u1z[e1], u2x[e2], u2y[e2], u2z[e2], a.q1, a.m1, w1[e1], q2, m2, w2[e2], n12,
                         sigma_max, a.L, bmax, a.dt, rng);
            if (maxN == NI1) i1 += minN;
            if (maxN == NI2) i2 += minN;
        }
    }
}

// One cell with n (= n1 + n2, or n1 for intra-species collisions) particles, 0 < n <= cap, by a group of G threads.
template <int G>
__device__ void collide_cell(const Args& a, long bin, int t, char* smem, int cap, long cs1, int n1, long cs2, int n2) {
    Group s(smem, cap);
    const int n = n1 + n2;
    // load the ids through the permutation
    for (int e = t; e < n; e += G) {
        const int p = storage_index(a, e, n1, cs1, cs2);
        s.key[e] = (e >= n1 ? a.id2 : a.id1)[p];
        s.lp[e] = p;
    }
    group_sync<G>();
    // canonical order: rank by id inside each species (ties, which unique ids never produce, by load position)
    for (int e = t; e < n; e += G) {
        const int lo = e < n1 ? 0 : n1, hi = e < n1 ? n1 : n;
        const uint64_t k = s.key[e];
        int r = lo;
        for (int f = lo; f < hi; ++f) { const uint64_t kf = s.key[f]; r += (kf < k) || (kf == k && f < e); }
        const int p = s.lp[e];
        const SoaView& P = e < n1 ? a.P1 : a.P2;
        s.pp[r] = p;
        s.w[r] = P.w[p]; s.ux[r] = P.ux[p]; s.uy[r] = P.uy[p]; s.uz[r] = P.uz[p];
        s.sh[e] = e;
    }
    group_sync<G>();
    const uint64_t gcell = global_cell(a, bin);
    constexpr int second = G == 32 ? 1 : 32;      // the thread of species 2 (another warp in a block)
    if (t == 0)
        cell_density_temperature_shuffle(a, s.w, s.ux, s.uy, s.uz, nullptr, s.sh, n1, a.m1, gcell, 0, &s.scal[0], &s.scal[1]);
    if (t == second && !a.same)
        cell_density_temperature_shuffle(a, s.w + n1, s.ux + n1, s.uy + n1, s.uz + n1, nullptr, s.sh + n1, n2, a.m2, gcell,
                                         1, &s.scal[2], &s.scal[3]);
    group_sync<G>();
    const double dn1 = s.scal[0], T1 = s.scal[1];
    const double dn2 = a.same ? dn1 : s.scal[2], T2 = a.same ? T1 : s.scal[3];
    const int half = n1 / 2;
    chains<G>(a, t, gcell, dn1, dn2, T1, T2, s.sh, a.same ? s.sh + half : s.sh + n1, a.same ? half : n1,
              a.same ? n1 - half : n2, s.w, s.ux, s.uy, s.uz, s.w, s.ux, s.uy, s.uz);
    group_sync<G>();
    for (int e = t; e < n; e += G) {
        const SoaView& P = e < n1 ? a.P1 : a.P2;
        const int p = s.pp[e];
        P.ux[p] = s.ux[e]; P.uy[p] = s.uy[e]; P.uz[p] = s.uz[e];
    }
    group_sync<G>();
}

// A cell beyond LARGE_CAP by a block, on the particles in place: the canonical order of each species goes to the
// caller's scratch at the cell's own slots (storage indices), the shuffle permutes it there, the chains read and write
// the particle arrays through it.  Same sums, draws and pair updates as collide_cell.
__device__ void collide_cell_global(const Args& a, long bin, int t, double* scal, long cs1, int n1, long cs2, int n2) {
    constexpr int G = LARGE_THREADS;
    const int n = n1 + n2;
    int* I1 = a.scr1 + cs1;
    int* I2 = a.same ? nullptr : a.scr2 + cs2;
    for (int e = t; e < n; e += G) {
        const bool two = e >= n1;
        const int lo = two ? n1 : 0, hi = two ? n : n1;
        const uint64_t* id = two ? a.id2 : a.id1;
        const int p = storage_index(a, e, n1, cs1, cs2);
        const uint64_t k = id[p];
        int r = 0;
        for (int f = lo; f < hi; ++f) {
            const uint64_t kf = id[storage_index(a, f, n1, cs1, cs2)];
            r += (kf < k) || (kf == k && f < e);
        }
        (two ? I2 : I1)[r] = p;
    }
    __syncthreads();
    const uint64_t gcell = global_cell(a, bin);
    if (t == 0)
        cell_density_temperature_shuffle(a, a.P1.w, a.P1.ux, a.P1.uy, a.P1.uz, I1, I1, n1, a.m1, gcell, 0, &scal[0], &scal[1]);
    if (t == 32 && !a.same)
        cell_density_temperature_shuffle(a, a.P2.w, a.P2.ux, a.P2.uy, a.P2.uz, I2, I2, n2, a.m2, gcell, 1, &scal[2], &scal[3]);
    __syncthreads();
    const double dn1 = scal[0], T1 = scal[1];
    const double dn2 = a.same ? dn1 : scal[2], T2 = a.same ? T1 : scal[3];
    const int half = n1 / 2;
    chains<G>(a, t, gcell, dn1, dn2, T1, T2, I1, a.same ? I1 + half : I2, a.same ? half : n1, a.same ? n1 - half : n2,
              a.P1.w, a.P1.ux, a.P1.uy, a.P1.uz, a.P2.w, a.P2.ux, a.P2.uy, a.P2.uz);
    __syncthreads();
}

// a warp per cell of at most SMALL_CAP particles
__global__ void __launch_bounds__(SMALL_WARPS * 32) collide_small_kernel(Args a, long nbins) {
    PIC_STATIC_SMEM(double, smem, SMALL_WARPS * group_bytes(SMALL_CAP) / 8);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    char* mine = reinterpret_cast<char*>(smem) + warp * group_bytes(SMALL_CAP);
    const long stride = (long)gridDim.x * SMALL_WARPS;
    for (long bin = (long)blockIdx.x * SMALL_WARPS + warp; bin < nbins; bin += stride) {
        long cs1, cs2; int n1, n2;
        const int n = cell_load(a, bin, &cs1, &n1, &cs2, &n2);
        if (n == 0 || n > SMALL_CAP) continue;
        collide_cell<32>(a, bin, lane, mine, SMALL_CAP, cs1, n1, cs2, n2);
    }
}

// a block per cell of more than SMALL_CAP particles: each block lists the large cells among its LARGE_SCAN bins
__global__ void __launch_bounds__(LARGE_THREADS) collide_large_kernel(Args a, long nbins) {
    PIC_DYNAMIC_SMEM(double, smem);
    PIC_STATIC_SMEM(int, list, LARGE_SCAN + 1);
    PIC_STATIC_SMEM(double, scal, 4);
    const int t = threadIdx.x;
    for (long base = (long)blockIdx.x * LARGE_SCAN; base < nbins; base += (long)gridDim.x * LARGE_SCAN) {
        if (t == 0) list[LARGE_SCAN] = 0;
        __syncthreads();
        const long bin = base + t;
        if (t < LARGE_SCAN && bin < nbins) {
            long cs1, cs2; int n1, n2;
            if (cell_load(a, bin, &cs1, &n1, &cs2, &n2) > SMALL_CAP) list[atomicAdd(&list[LARGE_SCAN], 1)] = t;   // shared memory only
        }
        __syncthreads();
        const int nl = list[LARGE_SCAN];
        for (int k = 0; k < nl; ++k) {
            const long b = base + list[k];
            long cs1, cs2; int n1, n2;
            const int n = cell_load(a, b, &cs1, &n1, &cs2, &n2);
            if (n <= LARGE_CAP) collide_cell<LARGE_THREADS>(a, b, t, reinterpret_cast<char*>(smem), LARGE_CAP, cs1, n1, cs2, n2);
            else if (a.scr1 && (a.same || a.scr2)) collide_cell_global(a, b, t, scal, cs1, n1, cs2, n2);
            else if (t == 0) *a.status = 1;
        }
        __syncthreads();
    }
}


}  // namespace coll
}  // namespace pic

using namespace pic;

extern "C" int pic_collide_pairwise_coulomb(const pic_coulomb_collision* c, const pic_soa* p1, const pic_bins* b1,
                                            const int* src1, const pic_soa* p2, const pic_bins* b2, const int* src2,
                                            const pic_geom* g, double dt, long step, int* scratch1, int* scratch2,
                                            int* status, void* stream) {
    PIC_REQUIRE(c && p1 && b1 && g && status, "pic_collide_pairwise_coulomb: null argument");
    PIC_REQUIRE(b1->cell_start && b1->np_binned == p1->np, "pic_collide_pairwise_coulomb: species 1 needs current bins");
    PIC_REQUIRE(p1->idcpu && p1->w, "pic_collide_pairwise_coulomb: species 1 needs ids and weights");
    PIC_REQUIRE(c->m1 > 0.0 && (c->same_species || c->m2 > 0.0), "pic_collide_pairwise_coulomb: masses must be positive");
    PIC_REQUIRE(step >= 0, "pic_collide_pairwise_coulomb: negative step");
    if (!c->same_species) {
        PIC_REQUIRE(p2 && b2 && b2->cell_start && b2->np_binned == p2->np && p2->idcpu && p2->w,
                    "pic_collide_pairwise_coulomb: species 2 needs current bins, ids and weights");
        for (int d = 0; d < 3; ++d)
            PIC_REQUIRE(b1->box_lo[d] == b2->box_lo[d] && b1->box_hi[d] == b2->box_hi[d] && b1->tile[d] == b2->tile[d],
                        "pic_collide_pairwise_coulomb: the two species' bins must describe the same box and tiles");
    }
    coll::Args a;
    a.P1 = make_soa(*p1, 0); a.id1 = p1->idcpu; a.src1 = src1; a.b1 = make_bins(*b1);
    if (c->same_species) { a.P2 = a.P1; a.id2 = a.id1; a.src2 = a.src1; a.b2 = a.b1; }
    else { a.P2 = make_soa(*p2, 0); a.id2 = p2->idcpu; a.src2 = src2; a.b2 = make_bins(*b2); }
    a.gn[0] = g->n_cell[0]; a.gn[1] = g->n_cell[1];
    double dx[3];
    for (int d = 0; d < 3; ++d) dx[d] = (g->prob_hi[d] - g->prob_lo[d]) / g->n_cell[d];
    a.dV = dx[0] * dx[1] * dx[2];
    a.q1 = c->q1; a.m1 = c->m1; a.q2 = c->q2; a.m2 = c->m2; a.L = c->coulomb_log; a.dt = dt;
    a.seed = c->seed; a.cidx = (uint64_t)(uint32_t)c->collision_index; a.step = (uint64_t)step; a.same = c->same_species;
    a.scr1 = scratch1; a.scr2 = c->same_species ? nullptr : scratch2;
    a.status = status;
    const long nbins = bins_count(a.b1);
    if (p1->np == 0 || (!c->same_species && p2->np == 0)) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    const long small_blocks = (nbins + coll::SMALL_WARPS - 1) / coll::SMALL_WARPS;
    coll::collide_small_kernel<<<(unsigned)(small_blocks < 2147483647L ? small_blocks : 2147483647L),
                                 coll::SMALL_WARPS * 32, 0, s>>>(a, nbins);
    count_launch();
    static const size_t large_smem = coll::group_bytes(coll::LARGE_CAP);
    static bool attr = [] {
        return cudaFuncSetAttribute(coll::collide_large_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)large_smem) == cudaSuccess;
    }();
    PIC_REQUIRE(attr, "pic_collide_pairwise_coulomb: cannot reserve %zu bytes of shared memory", large_smem);
    const long large_rounds = (nbins + coll::LARGE_SCAN - 1) / coll::LARGE_SCAN;
    const long large_blocks = large_rounds < 16L * NUM_SMS ? large_rounds : 16L * NUM_SMS;
    coll::collide_large_kernel<<<(unsigned)large_blocks, coll::LARGE_THREADS, large_smem, s>>>(a, nbins);
    count_launch();
    return check_launch("pic_collide_pairwise_coulomb") ? 0 : 1;
}
