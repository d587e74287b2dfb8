// Supercell gather + push for cell-sorted particles (the timed path of PushPX / PushP).
//
// One CTA per supercell (pic_bins.tile).  The six field components are staged ONCE into a
// shared-memory block covering the supercell plus the gather halo (2 points each side: node
// weights reach c-1..c+2, cell weights c-2..c+2 for order 3), then every particle of the supercell
// gathers its 252 (order 3, Galerkin) grid values from shared memory.  Cell-sorted particles of
// the same cell are adjacent lanes reading the same addresses -> shared-memory broadcasts.
// Particles that drifted out of their supercell since the last sort are NOT gathered inline (one
// such lane would drag its whole warp through ~250 dependent global loads -- measured +40% kernel
// time per step since the last sort): they are appended to a list and a second, order-agnostic
// kernel pushes them with one thread each.  Any particle order is correct.
// PERM (pic_gather_push_permuted): the push that follows a cell sort carries out the sort's move.  Slot ip of the
// binned order is loaded from perm.in at perm.src[ip] and stored, pushed, to P[ip]; nothing else changes.
//
// gather_push_pair_kernel (pic_set_gather_mode(PIC_GATHER_PAIRS); order 3 or 1, Galerkin, Yee): the gather
// is bound by the shared-memory data return (252 LDS.64 per particle = 15.75 clk per particle per SM,
// against ~8 clk of fp64 work).  With the node weights at order N = 3 (1) and the cell weights at the
// Galerkin order N - 1 = 2 (0) every stencil of a particle starts at `cell - 1` (`cell`) -- the SAME
// points for all particles of a cell.  So a lane takes TWO particles of one cell and feeds both from
// one set of loads: 126 LDS.64 per particle.  Particles that are not in the cell of their bin (moved
// since the sort) go to the stray lists as before.
#include "pic_common.cuh"
#include "gather_common.cuh"
#include "bins.cuh"
#include <algorithm>
#include <vector>

namespace pic {

constexpr int GT_HALO = 2;
constexpr int GT_THREADS = 256;
constexpr int GT_LOCAL_STRAYS = 1022;   // per-CTA list of particles that changed row inside the supercell

// Shared-memory block of the six components.  BD* > 0: compile-time extents (the 8x8x8 supercell:
// every stencil offset becomes an immediate of the LDS); BD0 == 0: run-time extents.
template <int BD0, int BD1, int BD2>
struct SmemFields {
    const double* blk;     // [6][BD2][BD1][BD0]
    int o0, o1, o2;        // global index of block element (0,0,0)
    int rb0, rb01, rbvol;  // run-time extents (generic instance only)
    struct Acc {
        const double* b; int s1, s2;
        __device__ __forceinline__ double operator()(int ix, int iy, int iz) const {
            if constexpr (BD0 > 0) return b[ix + BD0 * iy + BD0 * BD1 * iz];
            else return b[ix + s1 * iy + s2 * iz];
        }
    };
    __device__ __forceinline__ Acc at(int c, int i0, int j0, int k0) const {
        if constexpr (BD0 > 0)
            return Acc{blk + c * (BD0 * BD1 * BD2) + (i0 - o0) + BD0 * ((j0 - o1) + BD1 * (k0 - o2)), 0, 0};
        else
            return Acc{blk + c * rbvol + (i0 - o0) + rb0 * ((j0 - o1) + rb01 / rb0 * (k0 - o2)), rb0, rb01};
    }
};

#ifdef PIC_SIMT_HOST      // tests/host_harness only: the SIMT emulator copies synchronously
__device__ __forceinline__ void prefetch_l1(const void*) {}
__device__ __forceinline__ void cp_async8(double* smem_dst, const double* gsrc) { *smem_dst = *gsrc; }
__device__ __forceinline__ void cp_async_commit() {}
__device__ __forceinline__ void cp_async_wait_all() {}
#else
__device__ __forceinline__ void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" :: "l"(p)); }
__device__ __forceinline__ void cp_async8(double* smem_dst, const double* gsrc) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" :: "r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
#endif

struct StrayList { int* idx; int* count; int cap; };

template <int N, int G, bool YEE, int TX, int TY, int TZ, bool PERM = false>
__global__ void __launch_bounds__(GT_THREADS, 2)
gather_push_tile_kernel(SoaView P, BinsView bins, GlobalFields gf, GatherGeom gg, double qdt2m,
                        double dt, int pusher, int push_position, EscapeView esc, StrayList stray, PermSrc perm) {
    PIC_DYNAMIC_SMEM(double, smem);
    constexpr bool FIXED = TX > 0;
    const int BD0 = FIXED ? TX + 2 * GT_HALO : bins.tile[0] + 2 * GT_HALO;
    const int BD1 = FIXED ? TY + 2 * GT_HALO : bins.tile[1] + 2 * GT_HALO;
    const int BD2 = FIXED ? TZ + 2 * GT_HALO : bins.tile[2] + 2 * GT_HALO;
    const int bvol = BD0 * BD1 * BD2;
    const int t = blockIdx.x;
    int tc[3];
    tile_coords(bins, t, tc);
    const long tvol = (long)bins.tile[0] * bins.tile[1] * bins.tile[2];
    const int p_begin = min(bins.cell_start[(long)t * tvol], bins.np_limit);
    const int p_end = min(bins.cell_start[(long)(t + 1) * tvol], bins.np_limit);
    if (p_begin >= p_end) return;
    const int t0 = bins.box_lo[0] + tc[0] * bins.tile[0];
    const int t1 = bins.box_lo[1] + tc[1] * bins.tile[1];
    const int t2 = bins.box_lo[2] + tc[2] * bins.tile[2];
    SmemFields<FIXED ? TX + 2 * GT_HALO : 0, FIXED ? TY + 2 * GT_HALO : 0, FIXED ? TZ + 2 * GT_HALO : 0> sf;
    sf.blk = smem; sf.o0 = t0 - GT_HALO; sf.o1 = t1 - GT_HALO; sf.o2 = t2 - GT_HALO;
    sf.rb0 = BD0; sf.rb01 = BD0 * BD1; sf.rbvol = bvol;

    // ---- stage the six sub-blocks with asynchronous 8-byte copies (LDGSTS): all ~40 copies of a
    //      thread are in flight at once, no register staging ----
    // one THREAD per row of BD0 contiguous doubles: the component / row / bounds / address arithmetic is paid once
    // per row instead of once per element (the element-wise loop was 15 % of the kernel's instructions)
    for (int row = threadIdx.x; row < 6 * BD1 * BD2; row += GT_THREADS) {
        const int c = row / (BD1 * BD2), r2 = row - c * (BD1 * BD2);
        const int lk = r2 / BD1, lj = r2 - lk * BD1;
        const FabView& F = gf.v[c];
        const int gj = sf.o1 + lj, gk = sf.o2 + lk;
        const bool jk_in = gj >= F.lo1 && gj < F.lo1 + F.n1 && gk >= F.lo2 && gk < F.lo2 + F.n2;
        double* dst = smem + c * bvol + BD0 * (lj + BD1 * lk);
        const double* src = F.p + F.off(sf.o0, gj, gk);           // dereferenced only where the point exists
        const int i_first = F.lo0 - sf.o0, i_end = F.lo0 + F.n0 - sf.o0;   // li range inside the allocation
#pragma unroll
        for (int li = 0; li < (FIXED ? TX + 2 * GT_HALO : 64); ++li) {
            if (li >= BD0) break;
            if (jk_in && li >= i_first && li < i_end) cp_async8(dst + li, src + li);
            else dst[li] = 0.0;
        }
    }
    cp_async_commit();

    // the push touches neither weight nor id: they move here, coalesced, while the field copies are in flight
    // (four particles per thread and round: the index -> value -> store chains of a round overlap)
    if constexpr (PERM) {
        const bool ids = perm.id_in && perm.id_out;
        for (int i0 = p_begin + threadIdx.x; i0 < p_end; i0 += 4 * GT_THREADS) {
            int j[4]; double wv[4]; uint64_t iv[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) j[u] = i0 + u * GT_THREADS < p_end ? perm.src[i0 + u * GT_THREADS] : -1;
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                wv[u] = j[u] >= 0 ? perm.in.w[j[u]] : 0.0;
                iv[u] = j[u] >= 0 && ids ? perm.id_in[j[u]] : 0;
            }
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (j[u] >= 0) { P.w[i0 + u * GT_THREADS] = wv[u]; if (ids) perm.id_out[i0 + u * GT_THREADS] = iv[u]; }
        }
    }
    const SoaView& L = PERM ? perm.in : P;                     // where slot i is loaded from, and at which index
    auto at = [&](int i) -> int { if constexpr (PERM) return perm.src[i]; else return i; };
    // a particle handed to a list is pushed in place later: with PERM its record has to be in P by then
    auto hand_on = [&](int i, double xp, double yp, double zp, double ux, double uy, double uz) {
        if constexpr (PERM) { P.x[i] = xp; P.y[i] = yp; P.z[i] = zp; P.ux[i] = ux; P.uy[i] = uy; P.uz[i] = uz; }
    };

    // software prefetch: the next particle of this thread is requested before the current one is
    // gathered, so the HBM latency overlaps ~700 instructions of shared-memory gather + push
    double nx = 0, ny = 0, nz = 0, nux = 0, nuy = 0, nuz = 0;
    int ip = p_begin + threadIdx.x;
    if (ip < p_end) { const int j = at(ip); nx = L.x[j]; ny = L.y[j]; nz = L.z[j]; nux = L.ux[j]; nuy = L.uy[j]; nuz = L.uz[j]; }
    cp_async_wait_all();
    __syncthreads();

    // Lanes of a warp hold consecutive cell-sorted particles, i.e. particles of ONE (y,z) row of
    // cells (or two at a row end): their stencil reads hit the same few shared-memory rows and
    // cost about one wavefront each.  A particle that changed row since the sort makes every LDS of
    // its warp conflict; such particles (isolated row among their neighbours) are deferred to a
    // CTA-local list and gathered after the main sweep, so the regular warps stay conflict-free.
    PIC_STATIC_SMEM(int, s_stray, GT_LOCAL_STRAYS);
    PIC_STATIC_SMEM(int, s_nstray_, 1);
    int& s_nstray = s_nstray_[0];
    if (threadIdx.x == 0) s_nstray = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    auto finish = [&](int ipp, double xp, double yp, double zp, double ux, double uy, double uz, bool in_tile) {
        double F[6];
        if (in_tile) gather_fields<N, G, YEE>(sf, gg, xp, yp, zp, F);
        else gather_fields<N, G, YEE>(gf, gg, xp, yp, zp, F);      // global list full: inline, slow but correct
        push_particle(xp, yp, zp, ux, uy, uz, F, qdt2m, dt, pusher, push_position);
        P.ux[ipp] = ux; P.uy[ipp] = uy; P.uz[ipp] = uz;
        if (push_position) { P.x[ipp] = xp; P.y[ipp] = yp; P.z[ipp] = zp; esc.note(ipp, xp, yp, zp); }
    };
    auto cell_in_tile = [&](double xp, double yp, double zp, int& row) -> bool {
        // cell of the particle (global index) from the same coordinates the gather uses
        const int ci = gg.lo[0] + (int)((xp - gg.xyzmin[0]) * gg.dinv[0]);
        const int cj = gg.lo[1] + (int)((yp - gg.xyzmin[1]) * gg.dinv[1]);
        const int ck = gg.lo[2] + (int)((zp - gg.xyzmin[2]) * gg.dinv[2]);
        row = cj * 65536 + ck;
        return ci >= t0 && ci < t0 + bins.tile[0] && cj >= t1 && cj < t1 + bins.tile[1] &&
               ck >= t2 && ck < t2 + bins.tile[2];
    };

    for (; ip - lane < p_end; ip += GT_THREADS) {          // warp-uniform trip count
        const bool valid = ip < p_end;
        double xp = nx, yp = ny, zp = nz, ux = nux, uy = nuy, uz = nuz;
        const int in = ip + GT_THREADS;
        if (in < p_end) { const int j = at(in); nx = L.x[j]; ny = L.y[j]; nz = L.z[j]; nux = L.ux[j]; nuy = L.uy[j]; nuz = L.uz[j]; }
        int row = -1 - lane;
        const bool in_tile = valid && cell_in_tile(xp, yp, zp, row);
        const int row_prev = __shfl_up_sync(0xffffffffu, row, 1), row_next = __shfl_down_sync(0xffffffffu, row, 1);
        const bool isolated = !(lane > 0 && row == row_prev) && !(lane < 31 && row == row_next);
        bool now = valid;
        if (valid && !in_tile) {                  // left the supercell since the sort: second kernel
            const int n = atomicAdd(stray.count, 1);
            if (n < stray.cap) { hand_on(ip, xp, yp, zp, ux, uy, uz); stray.idx[n] = ip; now = false; }
        } else if (valid && isolated) {           // changed row inside the supercell: after the sweep
            const int n = atomicAdd(&s_nstray, 1);
            if (n < GT_LOCAL_STRAYS) { hand_on(ip, xp, yp, zp, ux, uy, uz); s_stray[n] = ip; now = false; }
        }
        __syncwarp();                             // one convergent pass through the 700-instruction body
        if (now) finish(ip, xp, yp, zp, ux, uy, uz, in_tile);
    }
    __syncthreads();
    const int nloc = min(s_nstray, GT_LOCAL_STRAYS);
    for (int t2l = threadIdx.x; t2l < nloc; t2l += GT_THREADS) {
        const int ipp = s_stray[t2l];
        finish(ipp, P.x[ipp], P.y[ipp], P.z[ipp], P.ux[ipp], P.uy[ipp], P.uz[ipp], true);
    }
}


// ---- two particles of one cell per lane ---------------------------------------------------------
// Shared memory: [6][BD2][BD1][BD0] doubles of fields | pair_start[tvol + 1] | s_stray[GT_LOCAL_STRAYS] | s_nstray.
// pair_start[c] = number of lane-pairs in the cells before c of this supercell (ceil(n_c / 2) each).
// MINB = 2: 128 registers (116 B of spill traffic at order 3), 16 warps per SM like the default kernel;
// MINB = 1: 254 registers, no spills, 8 warps per SM; 192 threads with MINB = 2: 168 registers, no spills, 12 warps.
constexpr int GP_THREADS = 256;

template <int N, int G, bool YEE, int TX, int TY, int TZ, int MINB, int NT = GP_THREADS>
__global__ void __launch_bounds__(NT, MINB)
gather_push_pair_kernel(SoaView P, BinsView bins, GlobalFields gf, GatherGeom gg, double qdt2m,
                        double dt, int pusher, int push_position, EscapeView esc, StrayList stray) {
    PIC_DYNAMIC_SMEM(double, smem);
    constexpr bool FIXED = TX > 0;
    const int BD0 = FIXED ? TX + 2 * GT_HALO : bins.tile[0] + 2 * GT_HALO;
    const int BD1 = FIXED ? TY + 2 * GT_HALO : bins.tile[1] + 2 * GT_HALO;
    const int BD2 = FIXED ? TZ + 2 * GT_HALO : bins.tile[2] + 2 * GT_HALO;
    const int bvol = BD0 * BD1 * BD2;
    const int t = blockIdx.x;
    int tc[3];
    tile_coords(bins, t, tc);
    const int tvol = bins.tile[0] * bins.tile[1] * bins.tile[2];
    const int* __restrict__ cs = bins.cell_start + (long)t * tvol;
    const int p_begin = min(cs[0], bins.np_limit);
    const int p_end = min(cs[tvol], bins.np_limit);
    if (p_begin >= p_end) return;
    const int t0 = bins.box_lo[0] + tc[0] * bins.tile[0];
    const int t1 = bins.box_lo[1] + tc[1] * bins.tile[1];
    const int t2 = bins.box_lo[2] + tc[2] * bins.tile[2];
    SmemFields<FIXED ? TX + 2 * GT_HALO : 0, FIXED ? TY + 2 * GT_HALO : 0, FIXED ? TZ + 2 * GT_HALO : 0> sf;
    sf.blk = smem; sf.o0 = t0 - GT_HALO; sf.o1 = t1 - GT_HALO; sf.o2 = t2 - GT_HALO;
    sf.rb0 = BD0; sf.rb01 = BD0 * BD1; sf.rbvol = bvol;
    int* pair_start = reinterpret_cast<int*>(smem + 6 * bvol);
    int* s_stray = pair_start + tvol + 1;
    int& s_nstray = s_stray[GT_LOCAL_STRAYS];

    // one THREAD per row of BD0 contiguous doubles: the component / row / bounds / address arithmetic is paid once
    // per row instead of once per element (the element-wise loop was 15 % of the kernel's instructions)
    for (int row = threadIdx.x; row < 6 * BD1 * BD2; row += NT) {
        const int c = row / (BD1 * BD2), r2 = row - c * (BD1 * BD2);
        const int lk = r2 / BD1, lj = r2 - lk * BD1;
        const FabView& F = gf.v[c];
        const int gj = sf.o1 + lj, gk = sf.o2 + lk;
        const bool jk_in = gj >= F.lo1 && gj < F.lo1 + F.n1 && gk >= F.lo2 && gk < F.lo2 + F.n2;
        double* dst = smem + c * bvol + BD0 * (lj + BD1 * lk);
        const double* src = F.p + F.off(sf.o0, gj, gk);           // dereferenced only where the point exists
        const int i_first = F.lo0 - sf.o0, i_end = F.lo0 + F.n0 - sf.o0;   // li range inside the allocation
#pragma unroll
        for (int li = 0; li < (FIXED ? TX + 2 * GT_HALO : 64); ++li) {
            if (li >= BD0) break;
            if (jk_in && li >= i_first && li < i_end) cp_async8(dst + li, src + li);
            else dst[li] = 0.0;
        }
    }
    cp_async_commit();

    // pairs per cell, then an exclusive scan by warp 0 (each lane sums a chunk, shuffle scan across lanes)
    for (int c = threadIdx.x; c < tvol; c += NT) {
        const int n_c = min(cs[c + 1], bins.np_limit) - min(cs[c], bins.np_limit);
        pair_start[c + 1] = (n_c + 1) >> 1;
    }
    if (threadIdx.x == 0) { pair_start[0] = 0; s_nstray = 0; }
    __syncthreads();
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        const int chunk = (tvol + 31) / 32;
        const int c0 = lane * chunk, c1 = min(c0 + chunk, tvol);
        int sum = 0;
        for (int c = c0; c < c1; ++c) sum += pair_start[c + 1];
        int incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        int run = incl - sum;                       // pairs before this lane's chunk
        for (int c = c0; c < c1; ++c) { run += pair_start[c + 1]; pair_start[c + 1] = run; }
    }
    cp_async_wait_all();
    __syncthreads();
    const int npairs = pair_start[tvol];

    auto in_cell = [&](double xp, double yp, double zp, int ci, int cj, int ck, bool& in_tile) -> bool {
        const int pi = gg.lo[0] + (int)((xp - gg.xyzmin[0]) * gg.dinv[0]);
        const int pj = gg.lo[1] + (int)((yp - gg.xyzmin[1]) * gg.dinv[1]);
        const int pk = gg.lo[2] + (int)((zp - gg.xyzmin[2]) * gg.dinv[2]);
        in_tile = pi >= t0 && pi < t0 + bins.tile[0] && pj >= t1 && pj < t1 + bins.tile[1] &&
                  pk >= t2 && pk < t2 + bins.tile[2];
        return pi == ci && pj == cj && pk == ck;
    };
    auto defer = [&](int ipp, bool in_tile) -> bool {          // true: listed (handled later), false: lists full
        if (in_tile) {
            const int n = atomicAdd(&s_nstray, 1);
            if (n < GT_LOCAL_STRAYS) { s_stray[n] = ipp; return true; }
            return false;
        }
        const int n = atomicAdd(stray.count, 1);
        if (n < stray.cap) { stray.idx[n] = ipp; return true; }
        return false;
    };
    auto single = [&](int ipp, bool in_tile) {                 // one particle, alone (rare paths)
        double xp = P.x[ipp], yp = P.y[ipp], zp = P.z[ipp], ux = P.ux[ipp], uy = P.uy[ipp], uz = P.uz[ipp];
        double F[6];
        if (in_tile) gather_fields<N, G, YEE>(sf, gg, xp, yp, zp, F);
        else gather_fields<N, G, YEE>(gf, gg, xp, yp, zp, F);
        push_particle(xp, yp, zp, ux, uy, uz, F, qdt2m, dt, pusher, push_position);
        P.ux[ipp] = ux; P.uy[ipp] = uy; P.uz[ipp] = uz;
        if (push_position) { P.x[ipp] = xp; P.y[ipp] = yp; P.z[ipp] = zp; esc.note(ipp, xp, yp, zp); }
    };

    for (int p = threadIdx.x; p < npairs; p += NT) {
        // cell of pair p: the last c with pair_start[c] <= p
        int lo = 0, hi = tvol;                       // invariant: pair_start[lo] <= p < pair_start[hi]
        while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (pair_start[mid] <= p) lo = mid; else hi = mid; }
        const int c = lo;
        const int cbeg = min(cs[c], bins.np_limit), cend = min(cs[c + 1], bins.np_limit);
        const int ia = cbeg + 2 * (p - pair_start[c]);
        int ib = ia + 1 < cend ? ia + 1 : -1;
        const int li = c % bins.tile[0], lj = (c / bins.tile[0]) % bins.tile[1], lk = c / (bins.tile[0] * bins.tile[1]);
        const int ci = t0 + li, cj = t1 + lj, ck = t2 + lk;
        double xa = P.x[ia], ya = P.y[ia], za = P.z[ia];
        // the momenta are needed only after ~1500 instructions of gather: request the lines now (no registers held)
        prefetch_l1(P.ux + ia); prefetch_l1(P.uy + ia); prefetch_l1(P.uz + ia);
        bool a_tile, b_tile = false;
        bool a_ok = in_cell(xa, ya, za, ci, cj, ck, a_tile);
        double xb = xa, yb = ya, zb = za;
        bool b_ok = false;
        if (ib >= 0) { xb = P.x[ib]; yb = P.y[ib]; zb = P.z[ib]; b_ok = in_cell(xb, yb, zb, ci, cj, ck, b_tile); }
        // a particle that left the cell of its bin is listed; when the lists are full it is pushed here, alone
        // (todo: at most two per pair, one shared copy of the single-particle body below)
        int todo[2] = {-1, -1};
        bool todo_tile[2] = {false, false};
        if (!a_ok && !defer(ia, a_tile)) { todo[0] = ia; todo_tile[0] = a_tile; }
        if (ib >= 0 && !b_ok && !defer(ib, b_tile)) { todo[1] = ib; todo_tile[1] = b_tile; }
        if (a_ok || b_ok) {
        if (!a_ok) { xa = xb; ya = yb; za = zb; }                   // one survivor: it rides in both slots
        if (!b_ok) { xb = xa; yb = ya; zb = za; }
        const int ja = a_ok ? ia : ib, jb = b_ok ? ib : ia;
        DirWeights<N, G> ax, ay, az, bx, by, bz;
        ax.compute((xa - gg.xyzmin[0]) * gg.dinv[0]); ay.compute((ya - gg.xyzmin[1]) * gg.dinv[1]); az.compute((za - gg.xyzmin[2]) * gg.dinv[2]);
        bx.compute((xb - gg.xyzmin[0]) * gg.dinv[0]); by.compute((yb - gg.xyzmin[1]) * gg.dinv[1]); bz.compute((zb - gg.xyzmin[2]) * gg.dinv[2]);
        bool both = ja != jb;
        if (both && !same_stencils<N, G, YEE>(gg, ax, ay, az, bx, by, bz)) {
            // same cell but different stencil origins (orders / centerings other than the tuned ones): B goes alone
            if (!defer(jb, true)) { todo[1] = jb; todo_tile[1] = true; }
            bx = ax; by = ay; bz = az; xb = xa; yb = ya; zb = za;
            both = false;
        }
        double FA[6], FB[6];
        gather_fields_pair<N, G, YEE>(sf, gg, ax, ay, az, bx, by, bz, FA, FB);
        {
            double ux = P.ux[ja], uy = P.uy[ja], uz = P.uz[ja];
            push_particle(xa, ya, za, ux, uy, uz, FA, qdt2m, dt, pusher, push_position);
            P.ux[ja] = ux; P.uy[ja] = uy; P.uz[ja] = uz;
            if (push_position) { P.x[ja] = xa; P.y[ja] = ya; P.z[ja] = za; esc.note(ja, xa, ya, za); }
        }
        if (both) {
            double ux = P.ux[jb], uy = P.uy[jb], uz = P.uz[jb];
            push_particle(xb, yb, zb, ux, uy, uz, FB, qdt2m, dt, pusher, push_position);
            P.ux[jb] = ux; P.uy[jb] = uy; P.uz[jb] = uz;
            if (push_position) { P.x[jb] = xb; P.y[jb] = yb; P.z[jb] = zb; esc.note(jb, xb, yb, zb); }
        }
        }
#pragma unroll 1
        for (int k = 0; k < 2; ++k)
            if (todo[k] >= 0) single(todo[k], todo_tile[k]);
    }
    __syncthreads();
    const int nloc = min(s_nstray, GT_LOCAL_STRAYS);
    for (int t2l = threadIdx.x; t2l < nloc; t2l += NT) single(s_stray[t2l], true);
}

// the listed strays, one thread each, fields through the read-only global path
template <int N, int G, bool YEE>
__global__ void __launch_bounds__(128)
gather_push_listed_kernel(SoaView P, StrayList stray, GlobalFields fld, GatherGeom gg, double qdt2m, double dt,
                          int pusher, int push_position, EscapeView esc) {
    const int n = min(*stray.count, stray.cap);
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
        const int ip = stray.idx[t];
        double xp = P.x[ip], yp = P.y[ip], zp = P.z[ip];
        double F[6];
        gather_fields<N, G, YEE>(fld, gg, xp, yp, zp, F);
        double ux = P.ux[ip], uy = P.uy[ip], uz = P.uz[ip];
        push_particle(xp, yp, zp, ux, uy, uz, F, qdt2m, dt, pusher, push_position);
        P.ux[ip] = ux; P.uy[ip] = uy; P.uz[ip] = uz;
        if (push_position) { P.x[ip] = xp; P.y[ip] = yp; P.z[ip] = zp; esc.note(ip, xp, yp, zp); }
    }
}

// pic_set_gather_mode: PIC_GATHER_TILE (0, default), PIC_GATHER_PAIRS (1) / PIC_GATHER_PAIRS_WIDE (2): two particles
// of a cell per lane, used for the orders / gathers whose stencils coincide inside a cell, i.e. order 3 or 1 with
// the Galerkin gather on the Yee grid
int g_gather_mode = 0;

template <int N, int G>
static int launch(SoaView P, const BinsView& bv, const GlobalFields& gf, const GatherGeom& gg,
                  bool yee, double qdt2m, double dt, int pusher, int push_position, const EscapeView& esc,
                  const PermSrc& perm, cudaStream_t s) {
    const long bvol = (long)(bv.tile[0] + 2 * GT_HALO) * (bv.tile[1] + 2 * GT_HALO) * (bv.tile[2] + 2 * GT_HALO);
    const long tvol = (long)bv.tile[0] * bv.tile[1] * bv.tile[2];
    const bool permute = perm.src != nullptr;
    const bool pairs = !permute && g_gather_mode != 0 && yee && G == 1 && (N == 3 || N == 1);
    const bool wide = g_gather_mode == 2, mid = g_gather_mode == 3;
    const size_t smem = (size_t)6 * bvol * sizeof(double) + (pairs ? sizeof(int) * (size_t)(tvol + 1 + GT_LOCAL_STRAYS + 1) : 0);
    const size_t static_smem = pairs ? 0 : sizeof(int) * (GT_LOCAL_STRAYS + 2);       // s_stray + s_nstray
    if (smem + static_smem > 227 * 1024) return fail("pic_gather_push: supercell too large for shared memory (%zu B)", smem);
    const int ntiles = bv.nt[0] * bv.nt[1] * bv.nt[2];
    const bool t888 = bv.tile[0] == 8 && bv.tile[1] == 8 && bv.tile[2] == 8;
    // stray list (stream-ordered scratch): a few per mille of the particles per step since the sort
    StrayList stray;
    stray.cap = (int)(bv.np_limit / 8 + 1024);
#define PIC_KARGS P, bv, gf, gg, qdt2m, dt, pusher, push_position, esc, stray
#define PIC_PERM , perm          /* the supercell kernel's extra argument */
    // the default kernel: 8x8x8 supercells on the Yee grid are the tuned instance (immediate LDS offsets)
#define PIC_LAUNCH_TILE \
    else if (permute && yee && t888) PIC_LAUNCH_K(gather_push_tile_kernel, GT_THREADS, PIC_PERM, true, 8, 8, 8, true); \
    else if (permute && yee) PIC_LAUNCH_K(gather_push_tile_kernel, GT_THREADS, PIC_PERM, true, 0, 0, 0, true); \
    else if (permute) PIC_LAUNCH_K(gather_push_tile_kernel, GT_THREADS, PIC_PERM, false, 0, 0, 0, true); \
    else if (yee && t888) PIC_LAUNCH_K(gather_push_tile_kernel, GT_THREADS, PIC_PERM, true, 8, 8, 8); \
    else if (yee) PIC_LAUNCH_K(gather_push_tile_kernel, GT_THREADS, PIC_PERM, true, 0, 0, 0); \
    else PIC_LAUNCH_K(gather_push_tile_kernel, GT_THREADS, PIC_PERM, false, 0, 0, 0);
#ifndef PIC_SIMT_HOST
    int* scratch = nullptr;
    if (cudaMallocAsync((void**)&scratch, sizeof(int) * (size_t)(stray.cap + 1), s) != cudaSuccess)
        return fail("pic_gather_push: cannot allocate %ld B of scratch", (long)(sizeof(int) * (stray.cap + 1)));
    stray.count = scratch; stray.idx = scratch + 1;
    cudaMemsetAsync(stray.count, 0, sizeof(int), s);
#define PIC_LAUNCH_K(KERNEL, THREADS, EXTRA, ...) do { \
        auto k = KERNEL<N, G, __VA_ARGS__>; \
        if (cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024 - static_smem - 1024)) != cudaSuccess) \
            return fail("pic_gather_push: cannot raise the dynamic shared memory limit"); \
        k<<<ntiles, THREADS, smem, s>>>(PIC_KARGS EXTRA); } while (0)
    if (pairs) {
        if constexpr (G == 1 && (N == 3 || N == 1)) {
            if (t888 && wide) PIC_LAUNCH_K(gather_push_pair_kernel, GP_THREADS, , true, 8, 8, 8, 1);
            else if (t888 && mid) PIC_LAUNCH_K(gather_push_pair_kernel, 192, , true, 8, 8, 8, 2, 192);
            else if (t888) PIC_LAUNCH_K(gather_push_pair_kernel, GP_THREADS, , true, 8, 8, 8, 2);
            else PIC_LAUNCH_K(gather_push_pair_kernel, GP_THREADS, , true, 0, 0, 0, 2);
        }
    }
    PIC_LAUNCH_TILE
#undef PIC_LAUNCH_K
    if (yee) gather_push_listed_kernel<N, G, true><<<NUM_SMS * 8, 128, 0, s>>>(P, stray, gf, gg, qdt2m, dt, pusher, push_position, esc);
    else gather_push_listed_kernel<N, G, false><<<NUM_SMS * 8, 128, 0, s>>>(P, stray, gf, gg, qdt2m, dt, pusher, push_position, esc);
    count_launch(2);
    cudaFreeAsync(scratch, s);
    return check_launch("pic_gather_push(tile)") ? 0 : 1;
#else       // tests/host_harness: the same kernels under the SIMT emulator (simt_host.h)
    (void)s; (void)t888;
    std::vector<int> scratch((size_t)stray.cap + 1, 0);
    stray.count = scratch.data(); stray.idx = scratch.data() + 1;
#define PIC_LAUNCH_K(KERNEL, THREADS, EXTRA, ...) \
        ::simt::launch(dim3(ntiles), dim3(THREADS), smem + 64, [&] { KERNEL<N, G, __VA_ARGS__>(PIC_KARGS EXTRA); })
    if (pairs) {
        if constexpr (G == 1 && (N == 3 || N == 1)) {
            if (t888 && wide) PIC_LAUNCH_K(gather_push_pair_kernel, GP_THREADS, , true, 8, 8, 8, 1);
            else if (t888 && mid) PIC_LAUNCH_K(gather_push_pair_kernel, 192, , true, 8, 8, 8, 2, 192);
            else if (t888) PIC_LAUNCH_K(gather_push_pair_kernel, GP_THREADS, , true, 8, 8, 8, 2);
            else PIC_LAUNCH_K(gather_push_pair_kernel, GP_THREADS, , true, 0, 0, 0, 2);
        }
    }
    PIC_LAUNCH_TILE
#undef PIC_LAUNCH_K
    if (yee) ::simt::launch(dim3(4), dim3(128), 64, [&] { gather_push_listed_kernel<N, G, true>(P, stray, gf, gg, qdt2m, dt, pusher, push_position, esc); });
    else ::simt::launch(dim3(4), dim3(128), 64, [&] { gather_push_listed_kernel<N, G, false>(P, stray, gf, gg, qdt2m, dt, pusher, push_position, esc); });
    return 0;
#endif
#undef PIC_LAUNCH_TILE
#undef PIC_PERM
#undef PIC_KARGS
}

int gather_push_tile_launch(const pic_soa* p, long offset, long np, const pic_fab E[3],
                            const pic_fab B[3], const GatherGeom& gg, double qdt2m, double dt,
                            int nox, int galerkin, int pusher, int push_position,
                            const pic_bins* bins, const EscapeView& esc, const PermSrc& perm, cudaStream_t s) {
    PIC_REQUIRE(offset == 0 && np == p->np, "pic_gather_push: bins describe the whole tile (offset 0, np = all)");
    BinsView bv = make_bins(*bins);
    bv.np_limit = (int)std::min<long>(bins->np_binned, np);   // the tile may have shrunk since the sort
    GlobalFields gf;
    for (int c = 0; c < 3; ++c) { gf.v[c] = make_view(E[c]); gf.v[3 + c] = make_view(B[c]); }
    SoaView P = make_soa(*p, 0);
    const bool yee = is_yee(E, B);
#define PIC_GT(N, G) return launch<N, G>(P, bv, gf, gg, yee, qdt2m, dt, pusher, push_position, esc, perm, s)
    if (nox == 1 && galerkin) PIC_GT(1, 1);
    if (nox == 1) PIC_GT(1, 0);
    if (nox == 2 && galerkin) PIC_GT(2, 1);
    if (nox == 2) PIC_GT(2, 0);
    if (nox == 3 && galerkin) PIC_GT(3, 1);
    PIC_GT(3, 0);
#undef PIC_GT
}

// the ordinary push: in place, no permutation
int gather_push_tile_launch(const pic_soa* p, long offset, long np, const pic_fab E[3],
                            const pic_fab B[3], const GatherGeom& gg, double qdt2m, double dt,
                            int nox, int galerkin, int pusher, int push_position,
                            const pic_bins* bins, const EscapeView& esc, cudaStream_t s) {
    return gather_push_tile_launch(p, offset, np, E, B, gg, qdt2m, dt, nox, galerkin, pusher, push_position, bins, esc,
                                   PermSrc{}, s);
}

}  // namespace pic
