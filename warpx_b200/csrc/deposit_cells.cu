// Esirkepov deposition for cell-sorted particles, one LANE PER CELL (pic_set_deposit_mode(PIC_DEPOSIT_CELLS);
// replaces doEsirkepovDepositionShapeN, Source/Particles/Deposition/CurrentDeposition.H:642-907).
//
// For a particle whose old and new position lie in one cell ("quiet", > 95 % of a thermal plasma) the stencil
// is anchored at that cell: ALL quiet particles of a cell add into the same (N+1)^2 x N nodes per component,
//     Jx[i][j][k] += cx[i] * (Sy_new[j] Az[k] + Sy_old[j] Bz[k]),   cx = prefix sums of wq/(dt dy dz)(Sx_old - Sx_new),
//     Az = Sz_new/3 + Sz_old/6,  Bz = Sz_old/3 + Sz_new/6            (cyclically for Jy, Jz).
// deposit_runs.cu gives every stencil LINE a lane and walks the particles: each lane re-reads the particle's
// record from shared memory (17 doubles for 15 FMA) and the kernel is bound by the shared-memory return path
// (profiles/r1k_ncu_full_256cube.txt: L1 92 %, fp64 32 %).  Here a lane owns a CELL and one component: its
// (N+1)^2 x N partial sums (48 at order 3) stay in registers while it walks the particles of its cell, and a
// particle costs it 19 doubles of shared-memory reads for 80 FMA -- the fp64 pipe becomes the bound.
//
// One CTA per supercell (8 x 8 x 8 cells), four warps with fixed roles (rotated by block so that the heavier
// role does not always land on the same SM sub-partition):
//   producer   lane = cell; slice s = the s-th particle of every cell of a group of 32 cells (4 rows along
//              x): positions, shape factors, prefix sums -> one record per lane in shared memory (double
//              buffered), and a header telling the consumers what the buffer holds;
//   consumer c (c = x, y, z)   same lane = cell mapping; reads the record of its lane and accumulates component c.
// After the last slice of a group a consumer adds its sums into the CTA's shared-memory J block of its
// component with plain read-modify-writes: it is the only writer of that block, and inside one instruction the
// lanes (distinct cells, same stencil offset) touch distinct nodes.  At the end the block goes to J with one
// fp64 red.global per touched node (7 per cell instead of the 40 of deposit_runs.cu, 540 per particle in
// the reference).
//
// Particles that are not quiet in the cell of their bin -- they crossed a cell face during this step, or moved
// since the last sort -- are split into sub-particles of the quiet form: a particle that changes cell along a
// direction is exactly the sum of two quiet-form stencils anchored at consecutive cells (window slots 0..N with
// prefix entries 0..N-1, and slot N+1 with prefix entry N: the same products as the full stencil, term by
// term).  The sub-particle anchored at the lane's own cell rides in the regular slice; the others are queued in
// shared memory and deposited after the groups in EXTRA ROUNDS: a lane takes one queued sub-particle of any cell
// (distinct cells within a round, __match_any_sync), the consumers accumulate it like a slice and add it at the
// record's own anchor.  Only particles with a sub-particle outside the supercell go to the list of
// deposit_general_kernel (deposit_runs.cu): about one in eight of the movers.
// Orders 1 and 3 (the stencil of every particle of a cell starts at the same node; not so at order 2).
#include "pic_common.cuh"
#include "deposit_common.cuh"
#include "bins.cuh"
#ifdef PIC_SIMT_HOST
#include <vector>
#endif

namespace pic {

constexpr unsigned DC_FULL = 0xffffffffu;

template <int N> struct CellsCfg {
    static_assert(N == 1 || N == 3, "one lane per cell: orders 1 and 3");
    static constexpr int T = 8;                   // supercell edge (pic_bins tile)
    static constexpr int QS = N + 1;              // stencil nodes per direction
    static constexpr int QP = N;                  // live prefix entries
    static constexpr int O0 = -((N - 1) / 2);     // first stencil node relative to the cell
    static constexpr int PX = 12, PY = T + QS - 1, PZ = T + QS - 1;   // J block: pitch 12 keeps rows r, r+2 in disjoint banks
    static constexpr int TS = PX * PY * PZ;       // doubles per component
    static constexpr int NCP = (QP + 1) / 2;      // double2 elements of one component's prefix sums
    // record (double2 per lane): (Sx_new,Sx_old)[QS], (Sy_new,Sy_old)[QS], (Ay,By)[QS], (Az,Bz)[QS], cds x/y/z [NCP] each,
    // then one element of integers {active, offset of the anchor cell in the J block} (extra rounds only)
    static constexpr int F_SX = 0, F_SY = QS, F_ABY = 2 * QS, F_ABZ = 3 * QS, F_CDS = 4 * QS, F_META = 4 * QS + 3 * NCP;
    static constexpr int NF = F_META + 1;
    static constexpr int QCAP = 768;              // queued sub-particles per supercell (8 bytes each)
    static constexpr size_t smem_bytes = sizeof(double2) * 2 * NF * 32 + sizeof(double) * 3 * TS + sizeof(int2) * QCAP + 64;
};

// what the consumers do with a record buffer (written by the producer before the barrier)
struct CellsHeader { int kind, retire, g, pad; };
constexpr int DC_END = 0, DC_SLICE = 1, DC_EXTRA = 2;

// ---- what a producer warp does with one particle ---------------------------------------------------------------
template <int N> struct CellsPart {
    double wn[3][N + 1], wo[3][N + 1], wq;
    int t[3];       // anchor of the low sub-particle, in cells of the supercell
    int sh[3];      // i_old - i_new
    bool inside;    // every sub-particle is anchored at a cell of this supercell
};

template <int N> struct CellsProducer {
    using T = CellsCfg<N>;
    static constexpr int QS = T::QS, QP = T::QP, NCP = T::NCP;
    SoaView P; DepositGeom dg;
    int amin[3];            // anchor (leftmost index of a quiet particle's stencil, CurrentDeposition.H:759) of the supercell's cell 0
    int* list; int* list_count;
    int lane;

    __device__ __forceinline__ void load(long ip, double* v7) const {
        v7[0] = P.x[ip]; v7[1] = P.y[ip]; v7[2] = P.z[ip]; v7[3] = P.w[ip]; v7[4] = P.ux[ip]; v7[5] = P.uy[ip]; v7[6] = P.uz[ip];
    }
    __device__ __forceinline__ void compute(const double* v7, CellsPart<N>& q) const {      // v7 = x y z w ux uy uz
        const ParticleGeom pg = particle_geom(v7[0], v7[1], v7[2], v7[3], v7[4], v7[5], v7[6], dg);
        q.wq = pg.wq;
        bool in = true;
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const int inew = dr_dir<N>(pg.pos_new[d], pg.pos_old[d], q.wn[d], q.wo[d], q.sh[d]);
            q.t[d] = inew + (q.sh[d] < 0 ? q.sh[d] : 0) - amin[d];
            in = in && q.sh[d] >= -1 && q.sh[d] <= 1 && q.t[d] >= 0 && q.t[d] + (q.sh[d] ? 1 : 0) < T::T;
        }
        q.inside = in;
    }
    // quiet in the cell (lc) of the lane: the hot path
    __device__ __forceinline__ bool simple(const CellsPart<N>& q, const int lc[3]) const {
        return q.inside && (q.sh[0] | q.sh[1] | q.sh[2]) == 0 && q.t[0] == lc[0] && q.t[1] == lc[1] && q.t[2] == lc[2];
    }
    // The record of sub-particle v (v[d] = 0 low, 1 high) of q.  Window slot s (0..N+1) of direction d holds
    //   wn5[s] = wn[s - (sh < 0)],  wo5[s] = wo[s - (sh > 0)]   (0 outside 0..N),
    // c5[i] = prefix sum of wq/(dt dA) (wo5 - wn5) up to slot i; low: slots 0..N, c5[0..N-1]; high: slot N+1, c5[N].
    __device__ __forceinline__ void emit(const CellsPart<N>& q, const int v[3], double2* r, int active, int base) const {
        double2 s2[3][QS];
        double cds[3][2 * NCP];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const bool nsh = q.sh[d] < 0, osh = q.sh[d] > 0, hi = v[d] != 0;
            const double wqd = q.wq * dg.invdtd[d];
            double run = 0.0;
#pragma unroll
            for (int s = 0; s <= N; ++s) {
                const double n5 = nsh ? (s >= 1 ? q.wn[d][s >= 1 ? s - 1 : 0] : 0.0) : q.wn[d][s];
                const double o5 = osh ? (s >= 1 ? q.wo[d][s >= 1 ? s - 1 : 0] : 0.0) : q.wo[d][s];
                run += wqd * (o5 - n5);
                if (s < QP) cds[d][s] = hi ? 0.0 : run;
                s2[d][s] = hi ? make_double2(0.0, 0.0) : make_double2(n5, o5);
            }
            if (2 * NCP > QP) cds[d][2 * NCP - 1] = 0.0;
            if (hi) {     // slot N+1 and prefix entry N, at the local positions N and N-1 of the next cell
                s2[d][N] = make_double2(nsh ? q.wn[d][N] : 0.0, osh ? q.wo[d][N] : 0.0);
                cds[d][QP - 1] = run;            // c5[N]
            }
        }
#pragma unroll
        for (int s = 0; s < QS; ++s) {
            r[(T::F_SX + s) * 32] = s2[0][s];
            r[(T::F_SY + s) * 32] = s2[1][s];
            r[(T::F_ABY + s) * 32] = make_double2((1.0 / 3.0) * s2[1][s].x + (1.0 / 6.0) * s2[1][s].y,
                                                  (1.0 / 3.0) * s2[1][s].y + (1.0 / 6.0) * s2[1][s].x);
            r[(T::F_ABZ + s) * 32] = make_double2((1.0 / 3.0) * s2[2][s].x + (1.0 / 6.0) * s2[2][s].y,
                                                  (1.0 / 3.0) * s2[2][s].y + (1.0 / 6.0) * s2[2][s].x);
        }
#pragma unroll
        for (int d = 0; d < 3; ++d)
#pragma unroll
            for (int m = 0; m < NCP; ++m) r[(T::F_CDS + d * NCP + m) * 32] = make_double2(cds[d][2 * m], cds[d][2 * m + 1]);
        *reinterpret_cast<int2*>(&r[T::F_META * 32]) = make_int2(active, base);
    }
    // the record of a particle that is quiet in the lane's own cell (no shifts): no selects
    __device__ __forceinline__ void emit_simple(const CellsPart<N>& q, double2* r) const {
#pragma unroll
        for (int s = 0; s < QS; ++s) {
            r[(T::F_SX + s) * 32] = make_double2(q.wn[0][s], q.wo[0][s]);
            r[(T::F_SY + s) * 32] = make_double2(q.wn[1][s], q.wo[1][s]);
            r[(T::F_ABY + s) * 32] = make_double2((1.0 / 3.0) * q.wn[1][s] + (1.0 / 6.0) * q.wo[1][s],
                                                  (1.0 / 3.0) * q.wo[1][s] + (1.0 / 6.0) * q.wn[1][s]);
            r[(T::F_ABZ + s) * 32] = make_double2((1.0 / 3.0) * q.wn[2][s] + (1.0 / 6.0) * q.wo[2][s],
                                                  (1.0 / 3.0) * q.wo[2][s] + (1.0 / 6.0) * q.wn[2][s]);
        }
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const double wqd = q.wq * dg.invdtd[d];
            double cds[2 * NCP];
            cds[2 * NCP - 1] = 0.0;
            double run = 0.0;
#pragma unroll
            for (int i = 0; i < QP; ++i) {
                run += wqd * (q.wo[d][i] - q.wn[d][i]);
                cds[i] = run;
            }
#pragma unroll
            for (int m = 0; m < NCP; ++m) r[(T::F_CDS + d * NCP + m) * 32] = make_double2(cds[2 * m], cds[2 * m + 1]);
        }
    }
    __device__ __forceinline__ void emit_nothing(double2* r) const {    // zero prefix sums: the weights left in the record are finite
#pragma unroll
        for (int m = 0; m < 3 * NCP; ++m) r[(T::F_CDS + m) * 32] = make_double2(0.0, 0.0);
        *reinterpret_cast<int2*>(&r[T::F_META * 32]) = make_int2(0, 0);
    }
    // A particle that is not simple: every sub-particle into the queue (returns false: no room / outside -> the list)
    __device__ __forceinline__ bool enqueue(const CellsPart<N>& q, long ip, int2* queue, int* q_count, int qcap = T::QCAP) const {
        if (!q.inside) return false;
        const int nq = (q.sh[0] ? 2 : 1) * (q.sh[1] ? 2 : 1) * (q.sh[2] ? 2 : 1);
        int slot = atomicAdd(q_count, nq);
        if (slot + nq > qcap) {              // queue full: the whole particle goes to the list
            atomicMin(q_count + 1, slot);    // later requests start beyond: they do not fit either
            return false;
        }
#pragma unroll 1
        for (int v = 0; v < 8; ++v) {
            const int vx = v & 1, vy = (v >> 1) & 1, vz = v >> 2;
            if ((vx && !q.sh[0]) || (vy && !q.sh[1]) || (vz && !q.sh[2])) continue;
            queue[slot++] = make_int2((int)ip, v | ((q.t[0] + vx) << 3) | ((q.t[1] + vy) << 6) | ((q.t[2] + vz) << 9));
        }
        return true;
    }
    __device__ __forceinline__ void to_list(bool listed, long ip) const {   // for deposit_general_kernel (warp-aggregated append)
        const unsigned mm = __ballot_sync(DC_FULL, listed);
        if (mm) {
            int basei = 0;
            if (lane == 0) basei = atomicAdd(list_count, __popc(mm));
            basei = __shfl_sync(DC_FULL, basei, 0);
            if (listed) list[basei + __popc(mm & ((1u << lane) - 1u))] = (int)ip;
        }
    }
};

// ---- what a consumer warp does with one record buffer ----------------------------------------------------------
// component roles: acc[a][b][p] += cds[p] * (A[a].x B[b].x + A[a].y B[b].y)
//   Jx: a = y (Sy),  b = z (ABz), p = x     Jy: a = x (Sx), b = z (ABz), p = y     Jz: a = x (Sx), b = y (ABy), p = z
template <int N> struct CellsConsumer {
    using T = CellsCfg<N>;
    static constexpr int QS = T::QS, QP = T::QP, NCP = T::NCP, PX = T::PX, PY = T::PY;
    int comp, fA, fB, fC, sa, sb, sp;
    double* tl;
    int lx, lrow;
    double acc[QS][QS][QP];

    __device__ __forceinline__ void init(int comp_, double* tile, int lx_, int lrow_) {
        comp = comp_; lx = lx_; lrow = lrow_;
        fA = (comp == 0) ? T::F_SY : T::F_SX;
        fB = (comp == 2) ? T::F_ABY : T::F_ABZ;
        fC = T::F_CDS + comp * NCP;
        sa = (comp == 0) ? PX : 1;
        sb = (comp == 2) ? PX : PX * PY;
        sp = (comp == 0) ? 1 : ((comp == 1) ? PX : PX * PY);
        tl = tile + (size_t)comp * T::TS;
#pragma unroll
        for (int a = 0; a < QS; ++a)
#pragma unroll
            for (int b = 0; b < QS; ++b)
#pragma unroll
                for (int p = 0; p < QP; ++p) acc[a][b][p] = 0.0;
    }
    __device__ __forceinline__ void consume(const double2* r) {
        double cds[2 * NCP];
#pragma unroll
        for (int m = 0; m < NCP; ++m) {
            const double2 c2 = r[(fC + m) * 32];
            cds[2 * m] = c2.x; cds[2 * m + 1] = c2.y;
        }
        double2 B[QS];
#pragma unroll
        for (int b = 0; b < QS; ++b) B[b] = r[(fB + b) * 32];
#pragma unroll
        for (int a = 0; a < QS; ++a) {
            const double2 A = r[(fA + a) * 32];
#pragma unroll
            for (int b = 0; b < QS; ++b) {
                const double wab = A.x * B[b].x + A.y * B[b].y;
#pragma unroll
                for (int p = 0; p < QP; ++p) acc[a][b][p] += cds[p] * wab;
            }
        }
    }
    // last slice of group g: add the lane's sums into the CTA's J block of this component.  Lanes are distinct cells,
    // so one instruction (fixed stencil offset) touches distinct nodes; two offsets that differ along z never meet (the
    // cells of a group share z), the others are ordered by __syncwarp.
    __device__ __forceinline__ void retire_group(int g) {
        const int ly = ((g & 1) << 2) + lrow, lz = g >> 1;
        double* base = tl + lx + PX * (ly + PY * lz);
        if (comp == 2) {                 // z is the prefix direction
#pragma unroll
            for (int a = 0; a < QS; ++a)
#pragma unroll
                for (int b = 0; b < QS; ++b) {
                    double* q = base + a * sa + b * sb;
                    double v[QP];
#pragma unroll
                    for (int p = 0; p < QP; ++p) v[p] = q[p * sp];
#pragma unroll
                    for (int p = 0; p < QP; ++p) { q[p * sp] = v[p] + acc[a][b][p]; acc[a][b][p] = 0.0; }
                    __syncwarp();
                }
        } else {                         // z is line direction b
#pragma unroll
            for (int a = 0; a < QS; ++a)
#pragma unroll
                for (int p = 0; p < QP; ++p) {
                    double* q = base + a * sa + p * sp;
                    double v[QS];
#pragma unroll
                    for (int b = 0; b < QS; ++b) v[b] = q[b * sb];
#pragma unroll
                    for (int b = 0; b < QS; ++b) { q[b * sb] = v[b] + acc[a][b][p]; acc[a][b][p] = 0.0; }
                    __syncwarp();
                }
        }
    }
    // extra round: every lane carries one sub-particle of ITS OWN cell (distinct cells within the round): add at the
    // record's anchor, one stencil offset at a time (the cells differ in every direction now, so every step is ordered)
    __device__ __forceinline__ void retire_extra(const double2* r) {
        retire_extra_at(*reinterpret_cast<const int2*>(&r[T::F_META * 32]));
    }
    __device__ __forceinline__ void retire_extra_at(const int2 mt) {      // mt = {active, offset of the anchor cell}
        double* base = tl + mt.y;
        const bool active = mt.x != 0;
#pragma unroll
        for (int a = 0; a < QS; ++a)
#pragma unroll
            for (int b = 0; b < QS; ++b)
#pragma unroll
                for (int p = 0; p < QP; ++p) {
                    double* q = base + a * sa + b * sb + p * sp;
                    if (active) *q += acc[a][b][p];
                    acc[a][b][p] = 0.0;
                    __syncwarp();
                }
    }
};

// the J block goes to the arrays: one reduction per touched node
template <int N, int NT>
__device__ __forceinline__ void cells_flush(const double* tile, const BinsView& bins, const int tc[3], const J3& Jp) {
    using T = CellsCfg<N>;
    constexpr int PX = T::PX, PY = T::PY, TS = T::TS;
    const int org[3] = {bins.box_lo[0] + tc[0] * T::T + T::O0, bins.box_lo[1] + tc[1] * T::T + T::O0,
                        bins.box_lo[2] + tc[2] * T::T + T::O0};
    for (int n = threadIdx.x; n < 3 * TS; n += NT) {
        const double v = tile[n];
        if (v == 0.0) continue;
        const int c = n / TS, r = n - c * TS;
        const int tz = r / (PX * PY), r2 = r - tz * (PX * PY), ty = r2 / PX, tx = r2 - ty * PX;
        const FabView& F = Jp.v[c];
        const int gx = org[0] + tx, gy = org[1] + ty, gz = org[2] + tz;
        if (gx < F.lo0 || gy < F.lo1 || gz < F.lo2 || gx >= F.lo0 + F.n0 || gy >= F.lo1 + F.n1 || gz >= F.lo2 + F.n2) continue;
        atomicAdd(F.p + F.off(gx, gy, gz), v);
    }
}

// the cell of lane `lane` in group g, its bin, and the bin's particles
template <int N>
struct CellsGroup {
    int p0, n, maxn, lc[3];
    __device__ __forceinline__ void load(const BinsView& bins, long bin0, long np_lim, int g, int lx, int lrow) {
        using T = CellsCfg<N>;
        lc[0] = lx; lc[1] = ((g & 1) << 2) + lrow; lc[2] = g >> 1;
        const long b = bin0 + lx + T::T * (lc[1] + T::T * lc[2]);
        p0 = (int)min((long)bins.cell_start[b], np_lim);
        n = (int)min((long)bins.cell_start[b + 1], np_lim) - p0;
        maxn = n;
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) maxn = max(maxn, __shfl_xor_sync(DC_FULL, maxn, o));
    }
};

// ==================================================================================================================
// One producer, three consumers (128 threads)
// ==================================================================================================================
template <int N, int MINB>
__global__ void __launch_bounds__(128, MINB)
deposit_cells_kernel(SoaView P, long np_lim, BinsView bins, J3 Jp, DepositGeom dg,
                     int* __restrict__ list, int* __restrict__ list_count) {
    using T = CellsCfg<N>;
    constexpr int NF = T::NF, PX = T::PX, PY = T::PY, TS = T::TS;
    PIC_DYNAMIC_SMEM(double2, smem2);
    double2* rec = smem2;                                                  // [2][NF][32]
    double* tile = reinterpret_cast<double*>(smem2 + 2 * NF * 32);         // [3][TS]
    int2* queue = reinterpret_cast<int2*>(tile + 3 * TS);                  // [QCAP] (particle, code)
    CellsHeader* hdr = reinterpret_cast<CellsHeader*>(queue + T::QCAP);    // [2]
    int* q_count = reinterpret_cast<int*>(hdr + 2);      // [0] entries requested, [1] first slot that did not fit
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int role = (warp + blockIdx.x) & 3;                              // 0 producer, 1..3 consumer of component role-1
    int tc[3];
    tile_coords(bins, blockIdx.x, tc);                                     // supercell of this CTA
    const long bin0 = (long)blockIdx.x * (T::T * T::T * T::T);
    // lane -> cell of a group: 8 cells along x, rows 0,2,1,3 (rows r, r+2 share a half-warp: disjoint banks)
    const int lx = lane & 7, rsel = lane >> 3, lrow = ((rsel & 1) << 1) | (rsel >> 1);

    for (int n = threadIdx.x; n < 3 * TS; n += 128) tile[n] = 0.0;
    for (int n = threadIdx.x; n < 2 * NF * 32; n += 128) rec[n] = make_double2(0.0, 0.0);
    if (threadIdx.x == 0) { q_count[0] = 0; q_count[1] = T::QCAP; }
    __syncthreads();

    if (role == 0) {
        // ============================== producer ==============================
        CellsProducer<N> pr{P, dg, {tc[0] * T::T + bins.box_lo[0] - dg.lo[0] + T::O0, tc[1] * T::T + bins.box_lo[1] - dg.lo[1] + T::O0,
                                    tc[2] * T::T + bins.box_lo[2] - dg.lo[2] + T::O0}, list, list_count, lane};
        double pf[7] = {0, 0, 0, 0, 0, 0, 0};
        int it = 0;
        // ---------------- the groups: slice s = the s-th particle of each of the 32 cells ----------------
        for (int g = 0; g < 16; ++g) {
            CellsGroup<N> G;
            G.load(bins, bin0, np_lim, g, lx, lrow);
            for (int s = 0; s < G.maxn; ++s) {
                double2* r = rec + (size_t)(it & 1) * NF * 32 + lane;
                const bool valid = s < G.n;
                const long ip = (long)G.p0 + s;
                // this particle was requested during the previous slice (registers); the first of a cell is loaded here
                double v7[7];
                if (s == 0) {
                    if (valid) pr.load(ip, v7);
                    else { v7[0] = v7[1] = v7[2] = v7[3] = v7[4] = v7[5] = v7[6] = 0.0; }
                } else {
#pragma unroll
                    for (int c = 0; c < 7; ++c) v7[c] = pf[c];
                }
                if (s + 1 < G.n) pr.load(ip + 1, pf);
                bool listed = false, sent = false;
                if (valid) {
                    CellsPart<N> q;
                    pr.compute(v7, q);
                    // hot path: quiet in the lane's own cell.  Everything else -- every sub-particle of it -- waits
                    // in the queue for the extra rounds (or goes to the list when it reaches outside the supercell).
                    if (pr.simple(q, G.lc)) { pr.emit_simple(q, r); sent = true; }
                    else listed = !pr.enqueue(q, ip, queue, q_count);
                }
                if (!sent) pr.emit_nothing(r);
                pr.to_list(listed, ip);
                if (lane == 0) hdr[it & 1] = CellsHeader{DC_SLICE, s == G.maxn - 1 ? 1 : 0, g, 0};
                __syncthreads();
                ++it;
            }
        }
        // ---------------- extra rounds: the queued sub-particles, one per lane, distinct cells per round ----------------
        __syncwarp();
        const int nq_total = min(q_count[0], q_count[1]);
        for (int qb = 0; qb < nq_total; qb += 32) {
            bool pend = qb + lane < nq_total;
            const int2 e = pend ? queue[qb + lane] : make_int2(0, 0);
            const int akey = (e.y >> 3) & 511;
            while (__ballot_sync(DC_FULL, pend)) {
                const unsigned m = __match_any_sync(DC_FULL, pend ? akey : 512 + lane);
                const bool go = pend && lane == __ffs(m) - 1;
                double2* r = rec + (size_t)(it & 1) * NF * 32 + lane;
                if (go) {
                    CellsPart<N> q;
                    double v7[7];
                    pr.load(e.x, v7);
                    pr.compute(v7, q);
                    const int v[3] = {e.y & 1, (e.y >> 1) & 1, (e.y >> 2) & 1};
                    const int ax = (e.y >> 3) & 7, ay = (e.y >> 6) & 7, az = (e.y >> 9) & 7;
                    pr.emit(q, v, r, 1, ax + PX * (ay + PY * az));
                } else {
                    pr.emit_nothing(r);
                }
                if (lane == 0) hdr[it & 1] = CellsHeader{DC_EXTRA, 1, 0, 0};
                __syncthreads();
                ++it;
                pend = pend && !go;
            }
        }
        if (lane == 0) hdr[it & 1] = CellsHeader{DC_END, 0, 0, 0};
        __syncthreads();
    } else {
        // ============================== consumer of component role - 1 ==============================
        CellsConsumer<N> co;
        co.init(role - 1, tile, lx, lrow);
        int it = 0;
        while (true) {
            __syncthreads();             // the producer has filled buffer it & 1 and its header
            const CellsHeader h = hdr[it & 1];
            if (h.kind == DC_END) break;
            const double2* r = rec + (size_t)(it & 1) * NF * 32 + lane;
            co.consume(r);
            if (h.kind == DC_SLICE) { if (h.retire) co.retire_group(h.g); }
            else co.retire_extra(r);
            ++it;
        }
    }
    __syncthreads();
    cells_flush<N, 128>(tile, bins, tc, Jp);
}

// ==================================================================================================================
// Two producers, three consumers (160 threads).  profiles/r2_ncu_cells_1p.txt: with one producer the consumers spend
// 65 % of their time at the barrier -- the producer's ~400 instructions per slice (plus the latency of its loads) are the
// critical path.  Here the items (slices, then extra rounds) alternate between two producer warps, and each item takes
// TWO barrier intervals: part 1 (load, geometry, shape factors, classification, queue / list) in interval k, part 2
// (record and header into buffer k & 1) in interval k+1; the consumers take it in interval k+2.  In every interval one
// producer runs a part 1 and the other a part 2.  Producer 0 owns the extra rounds (their duplicate-cell bookkeeping lives
// in its registers): in that phase producer 1's items are empty.  `stop` (shared memory) ends the loop of every warp
// after the same barrier.
// ==================================================================================================================
constexpr int DC_NOP = 3;

template <int N, int MINB>
__global__ void __launch_bounds__(160, MINB)
deposit_cells2_kernel(SoaView P, long np_lim, BinsView bins, J3 Jp, DepositGeom dg,
                      int* __restrict__ list, int* __restrict__ list_count) {
    using T = CellsCfg<N>;
    constexpr int NF = T::NF, PX = T::PX, PY = T::PY, TS = T::TS;
    PIC_DYNAMIC_SMEM(double2, smem2);
    double2* rec = smem2;                                                  // [2][NF][32]
    double* tile = reinterpret_cast<double*>(smem2 + 2 * NF * 32);         // [3][TS]
    int2* queue = reinterpret_cast<int2*>(tile + 3 * TS);                  // [QCAP] (particle, code)
    CellsHeader* hdr = reinterpret_cast<CellsHeader*>(queue + T::QCAP);    // [2]
    int* q_count = reinterpret_cast<int*>(hdr + 2);      // [0] entries requested, [1] first slot that did not fit, [2] stop
    volatile int* stop = q_count + 2;                    // index of the END item once known
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int role = (warp + blockIdx.x) % 5;            // 0, 1 producers (even / odd items), 2..4 consumers
    int tc[3];
    tile_coords(bins, blockIdx.x, tc);
    const long bin0 = (long)blockIdx.x * (T::T * T::T * T::T);
    const int lx = lane & 7, rsel = lane >> 3, lrow = ((rsel & 1) << 1) | (rsel >> 1);

    for (int n = threadIdx.x; n < 3 * TS; n += 160) tile[n] = 0.0;
    for (int n = threadIdx.x; n < 2 * NF * 32; n += 160) rec[n] = make_double2(0.0, 0.0);
    if (threadIdx.x == 0) { q_count[0] = 0; q_count[1] = T::QCAP; q_count[2] = 0x7fffffff; }
    __syncthreads();

    if (role < 2) {
        // ============================== producer of the items with parity `role` ==============================
        CellsProducer<N> pr{P, dg, {tc[0] * T::T + bins.box_lo[0] - dg.lo[0] + T::O0, tc[1] * T::T + bins.box_lo[1] - dg.lo[1] + T::O0,
                                    tc[2] * T::T + bins.box_lo[2] - dg.lo[2] + T::O0}, list, list_count, lane};
        // the walk over the slices: (g, s) is item number `k`; exhausted: k = number of slices
        CellsGroup<N> G;
        int g = -1, s = 0, k = 0;
        bool slices_left = true;
        auto next_group = [&]() {
            while (true) {
                if (++g >= 16) { slices_left = false; return; }
                G.load(bins, bin0, np_lim, g, lx, lrow);
                if (G.maxn > 0) { s = 0; return; }
            }
        };
        auto step = [&]() { if (slices_left) { ++k; if (++s >= G.maxn) next_group(); } };
        next_group();
        if (role == 1) step();                           // producer 1 starts at item 1
        // what part 1 leaves for part 2
        CellsPart<N> q;
        int kind = DC_NOP, h_retire = 0, h_g = 0, x_base = 0, x_v = 0;
        bool send = false;
        double pf[7] = {0, 0, 0, 0, 0, 0, 0};
        bool pf_ok = false;                              // pf holds the particle of this producer's next slice
        // extra rounds (producer 0)
        int nq_total = -1, qb = 0;
        bool pend = false;
        int2 e = make_int2(0, 0);
        bool ending = false;

        for (int t = 0;; ++t) {
            if ((t & 1) == role) {
                // ------------------------------ part 1 of item t ------------------------------
                kind = DC_NOP; send = false;
                if (slices_left) {                       // the walk points at item t: a slice
                    const bool valid = s < G.n;
                    const long ip = (long)G.p0 + s;
                    double v7[7];
                    if (pf_ok) {
#pragma unroll
                        for (int c = 0; c < 7; ++c) v7[c] = pf[c];
                    } else if (valid) pr.load(ip, v7);
                    else { v7[0] = v7[1] = v7[2] = v7[3] = v7[4] = v7[5] = v7[6] = 0.0; }
                    // this producer's next slice is s + 2 of the same cells when the group has it
                    pf_ok = s + 2 < G.maxn;              // warp-uniform
                    if (s + 2 < G.n) pr.load(ip + 2, pf);
                    bool listed = false;
                    if (valid) {
                        pr.compute(v7, q);
                        if (pr.simple(q, G.lc)) send = true;
                        else listed = !pr.enqueue(q, ip, queue, q_count);
                    }
                    pr.to_list(listed, ip);
                    kind = DC_SLICE; h_retire = (s == G.maxn - 1) ? 1 : 0; h_g = g;
                    step(); step();                      // to this producer's next item
                } else if (role == 0 && !ending) {       // an extra round, or the end
                    if (nq_total < 0) { nq_total = min(q_count[0], q_count[1]); qb = -32; }
                    if (!__ballot_sync(DC_FULL, pend)) {             // next batch of 32 queued sub-particles
                        qb += 32;
                        pend = qb + lane < nq_total;
                        e = pend ? queue[qb + lane] : make_int2(0, 0);
                    }
                    if (qb >= nq_total) { ending = true; kind = DC_END; }
                    else {
                        const unsigned m = __match_any_sync(DC_FULL, pend ? ((e.y >> 3) & 511) : 512 + lane);
                        const bool go = pend && lane == __ffs(m) - 1;
                        if (go) {
                            double v7[7];
                            pr.load(e.x, v7);
                            pr.compute(v7, q);
                            x_v = e.y & 7;
                            x_base = ((e.y >> 3) & 7) + PX * (((e.y >> 6) & 7) + PY * ((e.y >> 9) & 7));
                            send = true;
                        }
                        pend = pend && !go;
                        kind = DC_EXTRA;
                    }
                }
            } else if (t >= 1) {
                // ------------------------------ part 2 of item t - 1 ------------------------------
                const int kk = t - 1;
                double2* r = rec + (size_t)(kk & 1) * NF * 32 + lane;
                if (kind == DC_SLICE) {
                    if (send) pr.emit_simple(q, r); else pr.emit_nothing(r);
                } else if (kind == DC_EXTRA) {
                    const int v[3] = {x_v & 1, (x_v >> 1) & 1, (x_v >> 2) & 1};
                    if (send) pr.emit(q, v, r, 1, x_base); else pr.emit_nothing(r);
                }
                if (lane == 0) {
                    hdr[kk & 1] = CellsHeader{kind == DC_END ? DC_NOP : kind, kind == DC_EXTRA ? 1 : h_retire, h_g, 0};
                    if (kind == DC_END) *stop = kk;
                }
            }
            __syncthreads();
            if (*stop <= t - 1) break;
        }
    } else {
        // ============================== consumer of component role - 2 ==============================
        CellsConsumer<N> co;
        co.init(role - 2, tile, lx, lrow);
        for (int t = 0;; ++t) {
            if (t >= 2) {                                // item t - 2 sits in buffer t & 1
                const CellsHeader h = hdr[t & 1];
                if (h.kind == DC_SLICE || h.kind == DC_EXTRA) {
                    const double2* r = rec + (size_t)(t & 1) * NF * 32 + lane;
                    co.consume(r);
                    if (h.kind == DC_SLICE) { if (h.retire) co.retire_group(h.g); }
                    else co.retire_extra(r);
                }
            }
            __syncthreads();
            if (*stop <= t - 1) break;
        }
    }
    __syncthreads();
    cells_flush<N, 160>(tile, bins, tc, Jp);
}

// ==================================================================================================================
// Two producers, three consumers, DECOUPLED (160 threads): no per-item __syncthreads.  Three record slots; producer and
// consumers meet on mbarriers -- full[slot] (32 producer lanes arrive after their stores), empty[slot] (96 consumer lanes
// arrive after their loads).  A producer computes an item (loads, geometry, shape factors, classification) BEFORE it
// waits for its slot, so a load stall of one warp no longer stalls the others; the consumers take the items in order.
// Items k = 0 .. K-1 are the slices (owner k mod 2), then producer 0 alone produces the extra rounds (it waits on
// `bdone` until producer 1 has classified its last slice: the queue is complete) and the END item.
// ==================================================================================================================
#ifdef PIC_SIMT_HOST      // tests/host_harness: a counter the fibers poll cooperatively
struct DcBar { int count, arrived, phase, pad; };
__device__ __forceinline__ void dc_bar_init(DcBar* b, int count) { b->count = count; b->arrived = 0; b->phase = 0; }
__device__ __forceinline__ void dc_bar_fence_init() {}
__device__ __forceinline__ void dc_bar_arrive(DcBar* b) { if (++b->arrived == b->count) { b->arrived = 0; b->phase ^= 1; } }
__device__ __forceinline__ void dc_bar_wait(DcBar* b, int parity) { while (b->phase == parity) ::simt::yield(); }
#else
struct DcBar { unsigned long long v, pad; };
__device__ __forceinline__ unsigned dc_smem(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void dc_bar_init(DcBar* b, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(dc_smem(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void dc_bar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void dc_bar_arrive(DcBar* b) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(dc_smem(b)) : "memory");
}
__device__ __forceinline__ void dc_bar_wait(DcBar* b, int parity) {      // returns when the phase of that parity is complete
    unsigned done = 0;
    for (unsigned spins = 0; !done; ++spins) {
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}"
                     : "=r"(done) : "r"(dc_smem(b)), "r"(parity) : "memory");
        if (spins > (1u << 26)) __trap();       // a protocol bug must end the kernel with an error, not hang the device
    }
}
#endif

template <int N> struct Cells3Cfg {
    using T = CellsCfg<N>;
    static constexpr int NB = 3;                   // record slots
    static constexpr int QCAP = 512;
    static constexpr size_t smem_bytes = sizeof(double2) * NB * T::NF * 32 + sizeof(double) * 3 * T::TS + sizeof(int2) * QCAP +
                                         sizeof(CellsHeader) * NB + sizeof(DcBar) * (2 * NB + 1) + 16;
};

template <int N, int MINB>
__global__ void __launch_bounds__(160, MINB)
deposit_cells3_kernel(SoaView P, long np_lim, BinsView bins, J3 Jp, DepositGeom dg,
                      int* __restrict__ list, int* __restrict__ list_count) {
    using T = CellsCfg<N>;
    using T3 = Cells3Cfg<N>;
    constexpr int NF = T::NF, PX = T::PX, PY = T::PY, TS = T::TS, NB = T3::NB;
    PIC_DYNAMIC_SMEM(double2, smem2);
    double2* rec = smem2;                                                  // [NB][NF][32]
    double* tile = reinterpret_cast<double*>(smem2 + NB * NF * 32);        // [3][TS]
    int2* queue = reinterpret_cast<int2*>(tile + 3 * TS);                  // [QCAP]
    CellsHeader* hdr = reinterpret_cast<CellsHeader*>(queue + T3::QCAP);   // [NB]
    DcBar* full = reinterpret_cast<DcBar*>(hdr + NB);                      // [NB]
    DcBar* empty = full + NB;                                              // [NB]
    DcBar* bdone = empty + NB;
    int* q_count = reinterpret_cast<int*>(bdone + 1);                      // [0] requested, [1] first slot that did not fit
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int role = (warp + blockIdx.x) % 5;            // 0, 1 producers (even / odd slices), 2..4 consumers
    int tc[3];
    tile_coords(bins, blockIdx.x, tc);
    const long bin0 = (long)blockIdx.x * (T::T * T::T * T::T);
    const int lx = lane & 7, rsel = lane >> 3, lrow = ((rsel & 1) << 1) | (rsel >> 1);

    for (int n = threadIdx.x; n < 3 * TS; n += 160) tile[n] = 0.0;
    for (int n = threadIdx.x; n < NB * NF * 32; n += 160) rec[n] = make_double2(0.0, 0.0);
    if (threadIdx.x == 0) {
        q_count[0] = 0; q_count[1] = T3::QCAP;
        for (int b = 0; b < NB; ++b) { dc_bar_init(full + b, 32); dc_bar_init(empty + b, 96); }
        dc_bar_init(bdone, 32);
        dc_bar_fence_init();
    }
    __syncthreads();

    if (role < 2) {
        // ============================== producer ==============================
        CellsProducer<N> pr{P, dg, {tc[0] * T::T + bins.box_lo[0] - dg.lo[0] + T::O0, tc[1] * T::T + bins.box_lo[1] - dg.lo[1] + T::O0,
                                    tc[2] * T::T + bins.box_lo[2] - dg.lo[2] + T::O0}, list, list_count, lane};
        // hand an item over: wait until the consumers have released the slot's previous use, store, publish
        auto slot_of = [&](int k) -> double2* {
            const int slot = k % NB, use = k / NB;
            if (use >= 1) dc_bar_wait(empty + slot, (use - 1) & 1);
            return rec + (size_t)slot * NF * 32 + lane;
        };
        auto publish = [&](int k, int kind, int retire, int g) {
            const int slot = k % NB;
            if (lane == 0) hdr[slot] = CellsHeader{kind, retire, g, 0};
            dc_bar_arrive(full + slot);
        };
        CellsGroup<N> G;
        int g = -1, s = 0, k = 0;
        bool slices_left = true;
        auto next_group = [&]() {
            while (true) {
                if (++g >= 16) { slices_left = false; return; }
                G.load(bins, bin0, np_lim, g, lx, lrow);
                if (G.maxn > 0) { s = 0; return; }
            }
        };
        auto step = [&]() { if (slices_left) { ++k; if (++s >= G.maxn) next_group(); } };
        next_group();
        if (role == 1) step();
        double pf[7] = {0, 0, 0, 0, 0, 0, 0};
        bool pf_ok = false;
        // ---------------- this producer's slices ----------------
        while (slices_left) {
            const bool valid = s < G.n;
            const long ip = (long)G.p0 + s;
            double v7[7];
            if (pf_ok) {
#pragma unroll
                for (int c = 0; c < 7; ++c) v7[c] = pf[c];
            } else if (valid) pr.load(ip, v7);
            else { v7[0] = v7[1] = v7[2] = v7[3] = v7[4] = v7[5] = v7[6] = 0.0; }
            pf_ok = s + 2 < G.maxn;                      // this producer's next slice belongs to the same group
            if (s + 2 < G.n) pr.load(ip + 2, pf);
            bool listed = false, send = false;
            CellsPart<N> q;
            if (valid) {
                pr.compute(v7, q);
                if (pr.simple(q, G.lc)) send = true;
                else listed = !pr.enqueue(q, ip, queue, q_count, T3::QCAP);
            }
            pr.to_list(listed, ip);
            double2* r = slot_of(k);
            if (send) pr.emit_simple(q, r); else pr.emit_nothing(r);
            publish(k, DC_SLICE, s == G.maxn - 1 ? 1 : 0, g);
            step(); step();
        }
        if (role == 1) {
            dc_bar_arrive(bdone);                        // every slice of producer 1 is classified: the queue is complete
        } else {
            // ---------------- producer 0: the extra rounds, then END; item numbers continue at k = number of slices ----------------
            dc_bar_wait(bdone, 0);
            const int nq_total = min(q_count[0], q_count[1]);
            for (int qb = 0; qb < nq_total; qb += 32) {
                bool pend = qb + lane < nq_total;
                const int2 e = pend ? queue[qb + lane] : make_int2(0, 0);
                while (__ballot_sync(DC_FULL, pend)) {
                    const unsigned m = __match_any_sync(DC_FULL, pend ? ((e.y >> 3) & 511) : 512 + lane);
                    const bool go = pend && lane == __ffs(m) - 1;
                    CellsPart<N> q;
                    if (go) {
                        double v7[7];
                        pr.load(e.x, v7);
                        pr.compute(v7, q);
                    }
                    double2* r = slot_of(k);
                    if (go) {
                        const int v[3] = {e.y & 1, (e.y >> 1) & 1, (e.y >> 2) & 1};
                        pr.emit(q, v, r, 1, ((e.y >> 3) & 7) + PX * (((e.y >> 6) & 7) + PY * ((e.y >> 9) & 7)));
                    } else pr.emit_nothing(r);
                    publish(k, DC_EXTRA, 1, 0);
                    ++k;
                    pend = pend && !go;
                }
            }
            slot_of(k);
            publish(k, DC_END, 0, 0);
        }
    } else {
        // ============================== consumer of component role - 2 ==============================
        CellsConsumer<N> co;
        co.init(role - 2, tile, lx, lrow);
        for (int k = 0;; ++k) {
            const int slot = k % NB;
            dc_bar_wait(full + slot, (k / NB) & 1);
            const CellsHeader h = hdr[slot];
            if (h.kind == DC_END) break;
            const double2* r = rec + (size_t)slot * NF * 32 + lane;
            co.consume(r);
            int2 mt = make_int2(0, 0);
            if (h.kind == DC_EXTRA) mt = *reinterpret_cast<const int2*>(&r[T::F_META * 32]);
            dc_bar_arrive(empty + slot);                 // the record is in registers: the slot may be refilled
            if (h.kind == DC_SLICE) { if (h.retire) co.retire_group(h.g); }
            else co.retire_extra_at(mt);
        }
    }
    __syncthreads();
    cells_flush<N, 160>(tile, bins, tc, Jp);
}

// deposit_runs.cu: the listed particles (full stencil)
int deposit_general_launch(SoaView P, const int* list, const int* list_count, const pic_fab J[3], const DepositGeom& dg,
                           int nox, cudaStream_t s);

int g_cells_two_producers = 0;      // 1: PIC_DEPOSIT_CELLS2 (three CTAs per SM, 128 registers), 2: PIC_DEPOSIT_CELLS2_WIDE (two CTAs),
                                    // 3 / 4: PIC_DEPOSIT_CELLS3 / _WIDE (decoupled pipeline)

template <int N>
static int launch_cells(SoaView P, long np, const pic_fab J[3], const DepositGeom& dg, const pic_bins* pb, cudaStream_t s) {
    using T = CellsCfg<N>;
    BinsView bins = make_bins(*pb);
    if (bins.tile[0] != T::T || bins.tile[1] != T::T || bins.tile[2] != T::T)
        return fail("pic_deposit_esirkepov(cells): the bins must use 8 x 8 x 8 supercells");
    // the listed particles go through deposit_general_kernel, whose cell keys take 10 bits per direction: refuse
    // before the cell kernel has deposited anything (launch_general would refuse only after it)
    for (int d = 0; d < 3; ++d)
        for (int c = 0; c < 3; ++c)
            if (J[c].hi[d] - J[c].lo[d] + 2 > 1022) return fail("pic_deposit_esirkepov: J extent > 1020 points per rank");
    const long np_lim = np < (long)bins.np_limit ? np : (long)bins.np_limit;
    const unsigned grid = (unsigned)(bins.nt[0] * bins.nt[1] * bins.nt[2]);
    J3 j3; j3.v[0] = make_view(J[0]); j3.v[1] = make_view(J[1]); j3.v[2] = make_view(J[2]);
    constexpr int MINB = 3;
    const int two = g_cells_two_producers;
    auto k = two == 4 ? deposit_cells3_kernel<N, 2> : two == 3 ? deposit_cells3_kernel<N, MINB>
           : two == 2 ? deposit_cells2_kernel<N, 2> : two == 1 ? deposit_cells2_kernel<N, MINB> : deposit_cells_kernel<N, MINB>;
    const int nthreads = two ? 160 : 128;
    const size_t smem_bytes = two >= 3 ? Cells3Cfg<N>::smem_bytes : T::smem_bytes;
#ifndef PIC_SIMT_HOST
    int* scratch = nullptr;
    if (cudaMallocAsync((void**)&scratch, sizeof(int) * (size_t)(np + 1), s) != cudaSuccess)
        return fail("pic_deposit_esirkepov: cannot allocate %ld B of scratch", (long)(sizeof(int) * (np + 1)));
    cudaMemsetAsync(scratch, 0, sizeof(int), s);
    static bool attr_done[5] = {false, false, false, false, false};
    if (!attr_done[two]) {
        cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
        attr_done[two] = true;
    }
    k<<<grid, nthreads, smem_bytes, s>>>(P, np_lim, bins, j3, dg, scratch + 1, scratch);
    count_launch();
    int rc = check_launch("pic_deposit_esirkepov(cells)") ? 0 : 1;
    if (!rc) rc = deposit_general_launch(P, scratch + 1, scratch, J, dg, N, s);
    cudaFreeAsync(scratch, s);
    return rc;
#else
    std::vector<int> scratch_h((size_t)np + 1, 0);
    int* scratch = scratch_h.data();
    k<<<grid, nthreads, smem_bytes, s>>>(P, np_lim, bins, j3, dg, scratch + 1, scratch);
    return deposit_general_launch(P, scratch + 1, scratch, J, dg, N, s);
#endif
}

// particles [0, min(np, np_binned)) through the cell kernel + the general kernel; the caller deposits the rest
int deposit_cells_launch(const pic_soa* p, long offset, long np, const pic_fab J[3], const DepositGeom& dg, int nox,
                         const pic_bins* bins, cudaStream_t s) {
    SoaView P = make_soa(*p, offset);
    if (nox == 1) return launch_cells<1>(P, np, J, dg, bins, s);
    return launch_cells<3>(P, np, J, dg, bins, s);
}

}  // namespace pic
