// The cell walk of the binary collisions (collision.cu: pairwise Coulomb, fusion.cu: nuclear fusion), written once as
// templates over a per-collision functor F, as the reference's BinaryCollision<Functor> is; with the reference's
// constants, the per-cell Philox random stream of their determinism contract (collision.cu) and the amrex::min / max
// they restate.  Each .cu instantiates the templates with its own functor, so the walk is compiled with that file's
// flags (-fmad=false).
//
// Per cell of the two species' bins (species 2 is species 1 for an intra-species collision, a.same):
//   * canonical order: the cell's particles of each species, loaded through the pending permutation src (when there
//     is one), ranked by id; with F::skip_spent the particles whose id is PIC_SPENT_ID are left out;
//   * per species, F::species (one thread, before the shuffle) and the Fisher-Yates shuffle with stream tag 0 / 1;
//   * F's constructor (the cell's set-up), then the independent pair chains: chain c on thread c, c + G, ... with
//     stream tag 2 + c, pairs (I1[i1], I2[i2]) of the halves of the shuffled species 1 (intra-species) or of the two
//     shuffled species, each through F::pair;
//   * F::end_cell (per-bin results), then, for a cell copied to shared memory, F::store of each particle.
// A warp takes a cell of at most SMALL_CAP particles, a block of LARGE_THREADS a cell of at most LARGE_CAP, both on a
// copy of the cell in shared memory.  A larger cell takes a block that keeps only the cell's canonical order, as
// storage indices, in the caller's per-slot int scratch at the cell's own slots (so cells never share it), and works
// on the particles in place: the same sums, draws and pair updates, so the same result.  Without that scratch it sets
// *status = 1.
//
// The functor F provides:
//   Args                 its argument block, derived from PairArgs;
//   skip_spent           whether particles with the id PIC_SPENT_ID are left out of the canonical order;
//   Scalars              per-cell values of a group in shared memory, zeroed at the start of each cell (with skip_spent:
//                        live[2], the live particles of each species);
//   species(a, v, sp, I, n, x)           before the shuffle of species sp (1, 2), its n particles v[I[0, n)];
//   F(a, bin, x, minN, maxN)             the cell's set-up after the shuffles;
//   pair(a, v, e1, e2, k, rng)           pair k of the cell, particles e1 of species 1 and e2 of species 2;
//   end_cell<G>(a, bin, t, x)            after this thread's pairs; ends with a barrier of the group;
//   store(a, v, sp, e)                   writes particle e of the shared copy back to the particle arrays.
// v is a particle accessor: SharedCell (e is the position in the shared copy) or InPlace (e is the storage index).
#ifndef PIC_BINARY_COLLISION_CUH_
#define PIC_BINARY_COLLISION_CUH_
#include "pic_common.cuh"
#include "bins.cuh"
#include "philox.cuh"

namespace pic {
namespace coll {

constexpr double PI = 3.14159265358979323846;      // MathConst::pi, Source/ablastr/constant.H
constexpr double HBAR = 1.054571817e-34;            // PhysConst::hbar
constexpr double DBL_MIN_ = 2.2250738585072014e-308;  // std::numeric_limits<double>::min()
constexpr double TWO_M53 = 1.0 / 9007199254740992.0;

constexpr int SMALL_CAP = 64;          // particles of a cell (both species) a warp handles
constexpr int SMALL_WARPS = 4;         // warps per block of the small-cell kernel
constexpr int LARGE_CAP = 2048;        // particles of a cell a block handles in shared memory
constexpr int LARGE_THREADS = 256;
constexpr int LARGE_SCAN = 32;         // bins a block of the large-cell kernel looks at per round

// one random stream: consecutive 64-bit words of the blocks j = 0, 1, ... of counter (j + 1, c1, c2, c3)
struct Stream {
    uint64_t seed, c1, c2, c3, block;
    uint64_t w0, w1, w2, w3;
    int left;
    __host__ __device__ __forceinline__ Stream(uint64_t s, uint64_t a, uint64_t b, uint64_t c)
        : seed(s), c1(a), c2(b), c3(c | (1ull << 63)), block(0), w0(0), w1(0), w2(0), w3(0), left(0) {}
    __host__ __device__ __forceinline__ uint64_t next() {
        if (left == 0) {
            uint64_t o[4];
            philox4x64_10_counter(seed, block + 1, c1, c2, c3, o);
            w0 = o[0]; w1 = o[1]; w2 = o[2]; w3 = o[3];
            ++block; left = 4;
        }
        const uint64_t r = w0;
        w0 = w1; w1 = w2; w2 = w3;
        --left;
        return r;
    }
    __host__ __device__ __forceinline__ double uniform() { return (double)((next() >> 11) + 1) * TWO_M53; }
    __host__ __device__ __forceinline__ int random_int(int n) { return (int)(((double)(next() >> 11) * TWO_M53) * n); }
};

__host__ __device__ __forceinline__ double dmax(double a, double b) { return (a < b) ? b : a; }   // std::max
__host__ __device__ __forceinline__ double dmin(double a, double b) { return (b < a) ? b : a; }   // std::min

// What the arguments of every binary collision start with.
struct PairArgs {
    SoaView P1, P2;                     // P2, id2, src2, b2 are species 1's for an intra-species collision
    uint64_t* id1; uint64_t* id2;
    const int* src1; const int* src2;   // slot -> storage index, or null
    int* scr1; int* scr2;               // one int per slot (cells beyond LARGE_CAP), or null
    BinsView b1, b2;
    int gn[2];                          // global cells along x, y (stream counter)
    double m1, m2, dt, dV;
    uint64_t seed, cidx, step;
    int same;
    int* status;
};

// The refusals every binary collision makes about its two species.
inline int check_species(const char* what, bool same, const pic_soa* p1, const pic_bins* b1, const pic_soa* p2,
                         const pic_bins* b2) {
    PIC_REQUIRE(b1->cell_start && b1->np_binned == p1->np, "%s: species 1 needs current bins", what);
    PIC_REQUIRE(p1->idcpu && p1->w, "%s: species 1 needs ids and weights", what);
    if (!same) {
        PIC_REQUIRE(p2 && b2 && b2->cell_start && b2->np_binned == p2->np && p2->idcpu && p2->w,
                    "%s: species 2 needs current bins, ids and weights", what);
        for (int d = 0; d < 3; ++d)
            PIC_REQUIRE(b1->box_lo[d] == b2->box_lo[d] && b1->box_hi[d] == b2->box_hi[d] && b1->tile[d] == b2->tile[d],
                        "%s: the two species' bins must describe the same box and tiles", what);
    }
    return 0;
}

// The refusals every binary collision pass makes, then a's PairArgs from them and the collision c (its m1, m2, seed,
// collision_index, same_species); 0 or the failure.
template <class Spec>
int pair_args(const char* what, const Spec* c, const pic_soa* p1, const pic_bins* b1, const int* src1,
              const pic_soa* p2, const pic_bins* b2, const int* src2, const pic_geom* g, double dt, long step,
              int* scratch1, int* scratch2, int* status, PairArgs& a) {
    PIC_REQUIRE(c && p1 && b1 && g && status, "%s: null argument", what);
    if (int rc = check_species(what, c->same_species, p1, b1, p2, b2)) return rc;
    PIC_REQUIRE(step >= 0, "%s: negative step", what);
    a.P1 = make_soa(*p1, 0); a.id1 = p1->idcpu; a.src1 = src1; a.b1 = make_bins(*b1);
    if (c->same_species) { a.P2 = a.P1; a.id2 = a.id1; a.src2 = a.src1; a.b2 = a.b1; }
    else { a.P2 = make_soa(*p2, 0); a.id2 = p2->idcpu; a.src2 = src2; a.b2 = make_bins(*b2); }
    a.gn[0] = g->n_cell[0]; a.gn[1] = g->n_cell[1];
    double dx[3];
    for (int d = 0; d < 3; ++d) dx[d] = (g->prob_hi[d] - g->prob_lo[d]) / g->n_cell[d];
    a.dV = dx[0] * dx[1] * dx[2];
    a.m1 = c->m1; a.m2 = c->m2; a.dt = dt;
    a.seed = c->seed; a.cidx = (uint64_t)(uint32_t)c->collision_index; a.step = (uint64_t)step; a.same = c->same_species;
    a.scr1 = scratch1; a.scr2 = c->same_species ? nullptr : scratch2;
    a.status = status;
    return 0;
}

template <int G> __device__ __forceinline__ void group_sync() {
    if constexpr (G == 32) __syncwarp(); else __syncthreads();
}

// global cell index of the stream counter
template <class Args>
__device__ __forceinline__ uint64_t global_cell(const Args& a, long bin) {
    int tc[3], lc[3];
    const long tv = (long)a.b1.tile[0] * a.b1.tile[1] * a.b1.tile[2];
    tile_coords(a.b1, (int)(bin / tv), tc);
    const int l = (int)(bin % tv);
    lc[0] = l % a.b1.tile[0]; lc[1] = (l / a.b1.tile[0]) % a.b1.tile[1]; lc[2] = l / (a.b1.tile[0] * a.b1.tile[1]);
    return (uint64_t)(tc[0] * a.b1.tile[0] + lc[0] + a.b1.box_lo[0]) +
        (uint64_t)a.gn[0] * ((uint64_t)(tc[1] * a.b1.tile[1] + lc[1] + a.b1.box_lo[1]) +
                             (uint64_t)a.gn[1] * (uint64_t)(tc[2] * a.b1.tile[2] + lc[2] + a.b1.box_lo[2]));
}

// storage index of slot e of the cell (species 1 at [0, n1), species 2 after)
__device__ __forceinline__ int storage_index(const PairArgs& a, int e, int n1, long cs1, long cs2) {
    const bool two = e >= n1;
    const long slot = two ? cs2 + (e - n1) : cs1 + e;
    const int* src = two ? a.src2 : a.src1;
    return src ? src[slot] : (int)slot;
}

// particles of the cell's species 1 (and 2), spent ones included; 0 when fewer than a pair's worth are stored
__device__ __forceinline__ int cell_load(const PairArgs& a, long bin, long* cs1, int* n1, long* cs2, int* n2) {
    *cs1 = a.b1.cell_start[bin];
    *n1 = a.b1.cell_start[bin + 1] - (int)*cs1;
    if (a.same) { *cs2 = *cs1; *n2 = 0; return *n1 >= 2 ? *n1 : 0; }
    *cs2 = a.b2.cell_start[bin];
    *n2 = a.b2.cell_start[bin + 1] - (int)*cs2;
    return (*n1 >= 1 && *n2 >= 1) ? *n1 + *n2 : 0;
}

// Shared memory of one group for `cap` particles: w ux uy uz (canonical order), ids (load order), storage index (load
// order), storage index (canonical order), index sets, F::Scalars, spent flags (canonical order, with F::skip_spent);
// a multiple of 8 bytes, so that the groups of a block stay aligned.
template <class F> __host__ __device__ constexpr size_t group_bytes(int cap) {
    return ((size_t)cap * (4 * 8 + 8 + 3 * 4 + (F::skip_spent ? 1 : 0)) + sizeof(typename F::Scalars) + 7) & ~(size_t)7;
}

template <class F> struct Group {
    double *w, *ux, *uy, *uz;
    uint64_t* key;
    int *lp, *pp, *sh;
    typename F::Scalars* x;
    unsigned char* dead;
    __device__ Group(char* base, int cap) {
        double* d = reinterpret_cast<double*>(base);
        w = d; ux = d + cap; uy = d + 2 * cap; uz = d + 3 * cap;
        key = reinterpret_cast<uint64_t*>(d + 4 * cap);
        lp = reinterpret_cast<int*>(key + cap); pp = lp + cap; sh = pp + cap;
        x = reinterpret_cast<typename F::Scalars*>(sh + cap);
        dead = reinterpret_cast<unsigned char*>(x + 1);
    }
};

// the particles of a cell's copy in shared memory: element e is its canonical position (both species in one array)
template <class F> struct SharedCell {
    Group<F> s;
    __device__ __forceinline__ double& w(int, int e) const { return s.w[e]; }
    __device__ __forceinline__ double& ux(int, int e) const { return s.ux[e]; }
    __device__ __forceinline__ double& uy(int, int e) const { return s.uy[e]; }
    __device__ __forceinline__ double& uz(int, int e) const { return s.uz[e]; }
    __device__ __forceinline__ bool spent(int, int e) const { return s.dead[e]; }
    __device__ __forceinline__ void spend(int, int e) const { s.dead[e] = 1; }
    __device__ __forceinline__ int storage(int, int e) const { return s.pp[e]; }
};

// the particles of a species sp (1, 2) in place: element e is the storage index
struct InPlace {
    const PairArgs& a;
    __device__ __forceinline__ const SoaView& P(int sp) const { return sp == 1 ? a.P1 : a.P2; }
    __device__ __forceinline__ uint64_t* id(int sp) const { return sp == 1 ? a.id1 : a.id2; }
    __device__ __forceinline__ double& w(int sp, int e) const { return P(sp).w[e]; }
    __device__ __forceinline__ double& ux(int sp, int e) const { return P(sp).ux[e]; }
    __device__ __forceinline__ double& uy(int sp, int e) const { return P(sp).uy[e]; }
    __device__ __forceinline__ double& uz(int sp, int e) const { return P(sp).uz[e]; }
    __device__ __forceinline__ bool spent(int sp, int e) const { return id(sp)[e] == PIC_SPENT_ID; }
    __device__ __forceinline__ void spend(int sp, int e) const { id(sp)[e] = PIC_SPENT_ID; }
    __device__ __forceinline__ int storage(int, int e) const { return e; }
};

__device__ __forceinline__ void shuffle(const PairArgs& a, int* sh, int n, uint64_t gcell, int tag) {
    Stream rng(a.seed, a.step, gcell, (a.cidx << 32) | (uint64_t)tag);
    for (int i = n - 1; i >= 1; --i) {
        const int j = rng.random_int(i + 1);
        const int t = sh[i]; sh[i] = sh[j]; sh[j] = t;
    }
}

// The cell once its canonical order stands: I1 / I2 hold the L1 / L2 particles of species 1 / 2 as elements of v.
// Returns false, before any barrier, when the cell has fewer than a pair's worth of them.
template <class F, int G, class V>
__device__ bool walk(const typename F::Args& a, long bin, int t, const V& v, typename F::Scalars& x, int* I1, int* I2,
                     int L1, int L2) {
    if (a.same ? L1 < 2 : (L1 < 1 || L2 < 1)) return false;   // uniform over the group
    const uint64_t gcell = global_cell(a, bin);
    constexpr int second = G == 32 ? 1 : 32;      // the thread of species 2 (another warp in a block)
    if (t == 0) { F::species(a, v, 1, I1, L1, x); shuffle(a, I1, L1, gcell, 0); }
    if (t == second && !a.same) { F::species(a, v, 2, I2, L2, x); shuffle(a, I2, L2, gcell, 1); }
    group_sync<G>();
    const int half = L1 / 2;
    const int NI1 = a.same ? half : L1, NI2 = a.same ? L1 - half : L2;
    const int* J2 = a.same ? I1 + half : I2;
    const int maxN = NI1 > NI2 ? NI1 : NI2, minN = NI1 < NI2 ? NI1 : NI2;
    F f(a, bin, x, minN, maxN);
    for (int c = t; c < minN; c += G) {
        Stream rng(a.seed, a.step, gcell, (a.cidx << 32) | (uint64_t)(2 + c));
        int i1 = c, i2 = c;
        for (int k = c; k < maxN; k += minN) {
            f.pair(a, v, I1[i1], J2[i2], k, rng);
            if (maxN == NI1) i1 += minN;
            if (maxN == NI2) i2 += minN;
        }
    }
    f.template end_cell<G>(a, bin, t, x);
    return true;
}

// One cell with n (= n1 + n2, or n1 for intra-species collisions) particles, 0 < n <= cap, by a group of G threads on
// a copy in shared memory.
template <class F, int G>
__device__ void cell_shared(const typename F::Args& a, long bin, int t, char* smem, int cap, long cs1, int n1, long cs2,
                            int n2) {
    Group<F> s(smem, cap);
    const int n = n1 + n2;
    if (t == 0) *s.x = typename F::Scalars{};
    for (int e = t; e < n; e += G) {
        const int p = storage_index(a, e, n1, cs1, cs2);
        s.key[e] = (e >= n1 ? a.id2 : a.id1)[p];
        s.lp[e] = p;
    }
    group_sync<G>();
    // canonical order: rank by id inside each species (ties, which unique ids never produce, by load position)
    for (int e = t; e < n; e += G) {
        const bool two = e >= n1;
        const int lo = two ? n1 : 0, hi = two ? n : n1;
        const uint64_t k = s.key[e];
        if constexpr (F::skip_spent) {
            if (k == PIC_SPENT_ID) continue;                  // the largest id: spent ones rank last
            atomicAdd(&s.x->live[two], 1);                    // shared memory only
        }
        int r = lo;
        for (int f = lo; f < hi; ++f) { const uint64_t kf = s.key[f]; r += (kf < k) || (kf == k && f < e); }
        const int p = s.lp[e];
        const SoaView& P = two ? a.P2 : a.P1;
        s.pp[r] = p;
        s.w[r] = P.w[p]; s.ux[r] = P.ux[p]; s.uy[r] = P.uy[p]; s.uz[r] = P.uz[p];
        if constexpr (F::skip_spent) s.dead[r] = 0;
        s.sh[r] = r;
    }
    group_sync<G>();
    int L1 = n1, L2 = n2;
    if constexpr (F::skip_spent) {
        L1 = s.x->live[0]; L2 = s.x->live[1];
        group_sync<G>();                                      // read by all before the next cell resets them
    }
    if (!walk<F, G>(a, bin, t, SharedCell<F>{s}, *s.x, s.sh, s.sh + n1, L1, L2)) return;
    for (int e = t; e < n1 + L2; e += G)
        if (e < L1 || e >= n1) F::store(a, SharedCell<F>{s}, e >= n1 ? 2 : 1, e);
    group_sync<G>();
}

// A cell beyond LARGE_CAP by a block, on the particles in place: the canonical order of each species goes to the
// caller's scratch at the cell's own slots (storage indices), the shuffle permutes it there.  A particle is spent when
// its id says so; a particle is in one pair chain only, so no chain reads an id that another one writes.
template <class F>
__device__ void cell_in_place(const typename F::Args& a, long bin, int t, typename F::Scalars& x, long cs1, int n1,
                              long cs2, int n2) {
    constexpr int G = LARGE_THREADS;
    const int n = n1 + n2;
    int* I1 = a.scr1 + cs1;
    int* I2 = a.same ? nullptr : a.scr2 + cs2;
    if (t == 0) x = typename F::Scalars{};
    __syncthreads();
    for (int e = t; e < n; e += G) {
        const bool two = e >= n1;
        const int lo = two ? n1 : 0, hi = two ? n : n1;
        const uint64_t* id = two ? a.id2 : a.id1;
        const int p = storage_index(a, e, n1, cs1, cs2);
        const uint64_t k = id[p];
        if constexpr (F::skip_spent) {
            if (k == PIC_SPENT_ID) continue;
            atomicAdd(&x.live[two], 1);
        }
        int r = 0;
        for (int f = lo; f < hi; ++f) {
            const uint64_t kf = id[storage_index(a, f, n1, cs1, cs2)];
            r += (kf < k) || (kf == k && f < e);
        }
        (two ? I2 : I1)[r] = p;
    }
    __syncthreads();
    int L1 = n1, L2 = n2;
    if constexpr (F::skip_spent) {
        L1 = x.live[0]; L2 = x.live[1];
        __syncthreads();
    }
    if (walk<F, G>(a, bin, t, InPlace{a}, x, I1, I2, L1, L2)) __syncthreads();
}

// a warp per cell of at most SMALL_CAP particles
template <class F>
__global__ void __launch_bounds__(SMALL_WARPS * 32) small_kernel(const typename F::Args a, long nbins) {
    PIC_STATIC_SMEM(double, smem, SMALL_WARPS * group_bytes<F>(SMALL_CAP) / 8);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    char* mine = reinterpret_cast<char*>(smem) + warp * group_bytes<F>(SMALL_CAP);
    const long stride = (long)gridDim.x * SMALL_WARPS;
    for (long bin = (long)blockIdx.x * SMALL_WARPS + warp; bin < nbins; bin += stride) {
        long cs1, cs2; int n1, n2;
        const int n = cell_load(a, bin, &cs1, &n1, &cs2, &n2);
        if (n == 0 || n > SMALL_CAP) continue;
        cell_shared<F, 32>(a, bin, lane, mine, SMALL_CAP, cs1, n1, cs2, n2);
    }
}

// a block per cell of more than SMALL_CAP particles: each block lists the large cells among its LARGE_SCAN bins
template <class F>
__global__ void __launch_bounds__(LARGE_THREADS) large_kernel(const typename F::Args a, long nbins) {
    PIC_DYNAMIC_SMEM(double, smem);
    PIC_STATIC_SMEM(int, list, LARGE_SCAN + 1);
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
            if (n <= LARGE_CAP)
                cell_shared<F, LARGE_THREADS>(a, b, t, reinterpret_cast<char*>(smem), LARGE_CAP, cs1, n1, cs2, n2);
            else if (a.scr1 && (a.same || a.scr2))
                cell_in_place<F>(a, b, t, *Group<F>(reinterpret_cast<char*>(smem), LARGE_CAP).x, cs1, n1, cs2, n2);
            else if (t == 0) *a.status = 1;
        }
        __syncthreads();
    }
}

// Both kernels of F over the bins of a.b1; the large-cell kernel's shared memory is reserved once per functor.  Static:
// the flag stays the library's own (the local static of a template with external linkage is one object per process).
template <class F>
static int launch(const char* what, const typename F::Args& a, cudaStream_t s) {
    const long nbins = bins_count(a.b1);
    const long small_blocks = (nbins + SMALL_WARPS - 1) / SMALL_WARPS;
    small_kernel<F><<<(unsigned)(small_blocks < 2147483647L ? small_blocks : 2147483647L), SMALL_WARPS * 32, 0, s>>>(a, nbins);
    count_launch();
    static const size_t large_smem = group_bytes<F>(LARGE_CAP);
    static bool attr = [] {
        return cudaFuncSetAttribute(large_kernel<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)large_smem) ==
               cudaSuccess;
    }();
    PIC_REQUIRE(attr, "%s: cannot reserve %zu bytes of shared memory", what, large_smem);
    const long large_rounds = (nbins + LARGE_SCAN - 1) / LARGE_SCAN;
    const long large_blocks = large_rounds < 16L * NUM_SMS ? large_rounds : 16L * NUM_SMS;
    large_kernel<F><<<(unsigned)large_blocks, LARGE_THREADS, large_smem, s>>>(a, nbins);
    count_launch();
    return check_launch(what) ? 0 : 1;
}

}  // namespace coll
}  // namespace pic
#endif
