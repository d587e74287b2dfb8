// Esirkepov deposition for cell-sorted particles by warp-segmented register reduction
// (the timed path; replaces doEsirkepovDepositionShapeN, CurrentDeposition.H:642-907).
//
// For one particle the Esirkepov stencil is an outer product,
//     Jx[i][j][k] += cdsx[i] * Wx[j][k],   cdsx[i] = sum_{i'<=i} wq/(dt dy dz) (Sx_old[i'] - Sx_new[i']),
//     Wx[j][k]    = Sy_new[j] Az[k] + Sy_old[j] Bz[k],  Az = Sz_new/3 + Sz_old/6, Bz = Sz_old/3 + Sz_new/6
// (cyclically for Jy, Jz).  A warp alternates two phases over chunks of 32 consecutive particles:
//   phase 1 (lane = particle): positions, shape factors, prefix sums -> per-particle record in smem;
//   phase 2 (lane = stencil line): every lane owns stencil lines of all three components and keeps
//       their partial sums in REGISTERS while the warp walks the particles.  All particles of a
//       run with the same stencil anchor (same new cell) accumulate into the same registers: the
//       segment of the segmented reduction is the run of cell-sorted particles, and the reduction
//       costs no atomic and no shuffle.
// Two kernels:
//   deposit_quiet_kernel  -- particles whose old and new position lie in the same cell in all three
//       directions (the overwhelming majority in a thermal plasma).  Their stencil is (N+1)^2
//       lines x N prefix entries, so 32/(N+1)^2 particles are processed per warp pass.  Cells are
//       visited along x, and a lane owns the Jy/Jz lines of a fixed ABSOLUTE x (ring mapping): when
//       the anchor advances by one cell only the plane leaving the window is retired -- 40 fp64
//       reductions per cell instead of the reference's (N+2)(N+3)^2*3 = 540 per PARTICLE.
//       Particles that changed cell are appended to a list.
//   deposit_general_kernel -- the listed particles with the full (N+3)^2 x (N+2) stencil.
// Retired sums go to J with fp64 red.global (L2 reductions, no return value).  PIC_DEPOSIT_RUNS_SLAB (ZS > 0
// below) retires them into a per-warp shared-memory J slab instead: one supercell's 8 x 8 cells
// in x, y and ZS cell layers in z, grown by the stencil reach.  A warp's 512 particles cover about 64
// cells -- one z layer of a supercell -- so the slab is rebased rarely; a rebase and the end of the
// warp's span add the slab to J with fp64 red.global along x rows, zeros skipped.  The slab takes plain
// read-modify-writes: its one writer is the warp, inside one retire instruction the sender lanes own
// distinct lines and so touch distinct nodes, and retires are ordered by __syncwarp (no shared fp64
// atomicAdd: on sm_90a that is a CAS loop).  On the H100 the slab variant is slower (DESIGN.md section
// 3.3): the slab halves the resident warps and a shared read-modify-write waits where red.global does
// not.  Any particle order is CORRECT (a run may be a single particle); cell-sorted order is FAST.
#include "pic_common.cuh"
#include "deposit_common.cuh"
#ifdef PIC_SIMT_HOST
#include <vector>
#endif

namespace pic {

// bit 0: two v-lines per lane where N+1 is even; bit 1: per-slot reductions instead of the shuffle fold;
// bit 2: four v-lines per lane (order 3 only; 168 registers -> 3 CTAs of 4 warps per SM); bit 3: the J slab
int g_runs_variant = 0;

constexpr int DR_CH = 32;          // particles per chunk
constexpr int DR_CHP = DR_CH + 1;  // record pitch (odd: conflict-free column access)
constexpr unsigned FULL = 0xffffffffu;

#ifdef PIC_DEPOSIT_COUNTERS
// What the quiet kernel does, counted under the host emulator (tests/host_harness, one OS thread); the
// library build never defines PIC_DEPOSIT_COUNTERS.
struct RunsCounters {
    long chunks, particles, movers, runs, slides, jumps, lones, lones_outside, rebases, cells;
    long red_retire, red_lone, red_slab;      // fp64 reductions sent to J by the three paths
};
RunsCounters g_runs_counters;
#define DR_COUNT(field, v) (::pic::g_runs_counters.field += (v))
extern "C" void pic_runs_counters(long* out, int reset) {     // the fields in declaration order
    constexpr int n = sizeof(RunsCounters) / sizeof(long);
    for (int i = 0; i < n; ++i) out[i] = reinterpret_cast<const long*>(&g_runs_counters)[i];
    if (reset) g_runs_counters = RunsCounters{};
}
#else
#define DR_COUNT(field, v) ((void)0)
#endif

// ---- per-direction weights without dynamic indexing -------------------------------------------
// shifted (old-position) weights: slot s holds w[s-1-sh], sh in {-1,0,1}  (ShapeFactors.H:93-156)
template <int N>
__device__ __forceinline__ void dr_place_old(double* so /*N+3*/, const double* w /*N+1*/, int sh) {
#pragma unroll
    for (int s = 0; s < N + 3; ++s) {
        const double wm = (s <= N) ? w[s] : 0.0;
        const double w0 = (s >= 1 && s - 1 <= N) ? w[s - 1] : 0.0;
        const double wp = (s >= 2) ? w[s - 2] : 0.0;
        so[s] = (sh < 0) ? wm : ((sh == 0) ? w0 : wp);
    }
}

// ================================================================================================
// quiet particles
// ================================================================================================
// VL = lines along role Z that one lane owns ("v" values per lane).  VL = 1: one lane per line,
// QS*QS lanes per particle.  VL = 2 (experiment, pic_set_deposit_mode(PIC_DEPOSIT_RUNS2)): a lane owns
// the lines of two consecutive v, so the pairs (Sx, Sy) and the prefix sums are fetched once for
// twice the lines -- the kernel is bound by the shared-memory return path (DESIGN.md section 8).
template <int N, int VL = 1> struct QuietCfg {
    static constexpr int QS = N + 1;          // slots 1..N+1 of the (N+3)-slot window
    static_assert(QS % VL == 0, "VL must divide N+1");
    static constexpr int QL = QS * (QS / VL); // lanes per particle
    static constexpr int NG = 32 / QL;        // particles per warp pass
    static constexpr int QP = N;              // live prefix entries (slots 1..N)
    // The record is an array of double2 (one LDS.128 fetches a pair the lane always needs together):
    //   (Sx_new, Sx_old)[QS], (Sy_new, Sy_old)[QS], (Ay, By)[QS], (Az, Bz)[QS], then the 3*QP prefix
    //   sums packed two per element.
    static constexpr int F_SX = 0, F_SY = QS, F_ABY = 2 * QS, F_ABZ = 3 * QS;
    static constexpr int F_CDS = 4 * QS;
    static constexpr int NCDS = (3 * QP + 1) / 2;
    static constexpr int NF = 4 * QS + NCDS;  // double2 elements per particle
    // record pitch (double2 elements): a pass reads rows r < QS of a field family at NG consecutive
    // columns; with pitch = NG (mod 8) the 16-byte words pitch*r + c fall into distinct bank groups
    static constexpr int CHP = DR_CH + NG;
};

// Direction roles.  The kernel is written for "role" directions X (the direction along which
// consecutive cells are visited and the register window slides), Y and Z; R0/R1/R2 say which
// physical direction plays each role (the bins are numbered x-fastest, so X = x).
__device__ __forceinline__ long fab_stride(const FabView& F, int d) { return d == 0 ? 1 : (d == 1 ? F.sj : F.sk); }

// SLOTRED = true: the NG particle slots of a pass are not summed by shuffles before a plane is retired --
// every slot sends its own partial sums to L2 (NG times the reductions, no SHFL; experiment).
// ZS > 0: retire into the per-warp slab of ZS cell layers (dynamic shared memory after the NW records).
template <int N, int ZS> struct SlabCfg {
    static constexpr int SX = 8 + N, SY = 8 + N, SZ = ZS + N;    // nodes per direction (N+1 per quiet line)
    static constexpr int SN = SX * SY * SZ;                      // doubles per component
};
template <int N, int NW, int MINB, int R0, int R1, int R2, int VL = 1, bool SLOTRED = false, int ZS = 0>
__global__ void __launch_bounds__(NW * 32, MINB)
deposit_quiet_kernel(SoaView P, long np, int chunks_per_warp, J3 Jp, DepositGeom dg, KeyBase kbp,
                     int* __restrict__ list, int* __restrict__ list_count) {
    // role views of the physical arrays / geometry
    const FabView& Jx = Jp.v[R0]; const FabView& Jy = Jp.v[R1]; const FabView& Jz = Jp.v[R2];
    const int kbb[3] = {kbp.b0, kbp.b1, kbp.b2};
    const KeyBase kb = {kbb[R0], kbb[R1], kbb[R2]};
    using T = QuietCfg<N, VL>;
    constexpr int QS = T::QS, QL = T::QL, NG = T::NG, QP = T::QP, NF = T::NF, CHP = T::CHP;
    constexpr bool SLAB = ZS > 0;
    static_assert(!SLAB || (VL == 1 && !SLOTRED), "the slab takes one sender lane per line");
    using SC = SlabCfg<N, (SLAB ? ZS : 1)>;
    constexpr int SX = SC::SX, SY = SC::SY, SN = SC::SN;
    PIC_DYNAMIC_SMEM(double2, smem2);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double2* rec = smem2 + (size_t)warp * NF * CHP;
    double* slab = reinterpret_cast<double*>(smem2 + (size_t)NW * NF * CHP) + (size_t)warp * 3 * SN;
    // strides of the window's lines: along its own role in the slab or in J, and along role X for Jy / Jz
    const long stX = SLAB ? 1 : fab_stride(Jx, R0), stY = SLAB ? SX : fab_stride(Jy, R1);
    const long stZ = SLAB ? (long)SX * SY : fab_stride(Jz, R2);
    const long xY = SLAB ? 1 : fab_stride(Jy, R0), xZ = SLAB ? 1 : fab_stride(Jz, R0);

    const long nchunks = (np + DR_CH - 1) / DR_CH;
    const long wg = (long)blockIdx.x * NW + warp;
    const long c_begin = wg * chunks_per_warp;
    const long c_end = min(nchunks, c_begin + chunks_per_warp);
    if (c_begin >= c_end) return;

    // lane (g, u, h): particle slot g of the pass; the lane owns the VL values v = h*VL + m, m < VL:
    //   Jx line (j, k) = (1+u, 1+v);  Jy line (i, k) = (1+ur, 1+v);  Jz line (i, j) = (1+ur, 1+v),
    //   ur = (u - (ax+1)) mod QS  (ring mapping: a lane keeps the Jy/Jz lines of one absolute x)
    const int g = lane / QL, ql = lane % QL, qu = ql % QS, qv0 = (ql / QS) * VL;
    const bool active_q = g < NG;
    double acc[VL][3][QP];
#pragma unroll
    for (int m = 0; m < VL; ++m)
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int i = 0; i < QP; ++i) acc[m][c][i] = 0.0;
    int cur = -1;

    auto ring = [&](int ax) -> int {
        int r = (qu - (ax + 1)) % QS;
        return r < 0 ? r + QS : r;
    };
    auto fold = [&](double v) -> double {          // sum over the particle slots of the pass
        if constexpr (SLOTRED) return v;
        double r = v;
        if constexpr ((NG & (NG - 1)) == 0) {       // power of two: butterfly, log2(NG) steps; slot 0 ends with the sum
#pragma unroll
            for (int off = NG / 2; off >= 1; off >>= 1) r += __shfl_down_sync(FULL, r, off * QL);
        } else {
#pragma unroll
            for (int gg = 1; gg < NG; ++gg) {
                const double o = __shfl_down_sync(FULL, v, gg * QL);
                if (lane + gg * QL < NG * QL) r += o;
            }
        }
        return r;
    };
    // which lanes send retired sums to J: slot 0 after the fold, or every slot with its own partial sum
    const bool sender = SLOTRED ? active_q : (lane < QL);
    // Running state of the current anchor: this lane's ring index and the J addresses of its lines
    //   px -> Jx(gx+1, gy+1+u, gz+1+v) (entries along x: +i), py -> Jy(gx+1+ur, gy+1, gz+1+v) (+i*sj),
    //   pz -> Jz(gx+1+ur, gy+1+v, gz+1) (+i*sk)
    int ur = 0;
    double *px[VL], *py[VL], *pz[VL];
#pragma unroll
    for (int m = 0; m < VL; ++m) { px[m] = nullptr; py[m] = nullptr; pz[m] = nullptr; }
    auto at = [&](const FabView& F, int ix, int iy, int iz) -> double* {   // role indices -> element
        int q[3];
        q[R0] = ix; q[R1] = iy; q[R2] = iz;
        return F.p + F.off(q[0], q[1], q[2]);
    };
    // The slab holds the nodes (bx.., by.., bz..) of role component c at slab[c*SN + (z*SY + y)*SX + x]; it
    // takes the anchors gx+1 - bx in [0, 8), gy+1 - by in [0, 8), gz+1 - bz in [0, ZS).  No base yet: bx huge.
    int bx = 1 << 28, by = 0, bz = 0;
    auto slab_at = [&](int c, int ix, int iy, int iz) -> double* {       // role indices -> slab node
        return slab + c * SN + ((iz - bz) * SY + (iy - by)) * SX + (ix - bx);
    };
    auto covers = [&](int k) -> bool {
        const int gx = (k & 1023) + kb.b0, gy = ((k >> 10) & 1023) + kb.b1, gz = (k >> 20) + kb.b2;
        return (unsigned)(gx + 1 - bx) < 8u && (unsigned)(gy + 1 - by) < 8u && (unsigned)(gz + 1 - bz) < (unsigned)ZS;
    };
    // add the slab to J (red.global along x rows, zeros skipped), zero it and base it at anchor k: x and y at
    // the supercell of k's cell (gx + 2 for order 3), z at k's own layer
    auto rebase = [&](int k) {
        if (bx != (1 << 28)) {
            DR_COUNT(rebases, lane == 0);
#pragma unroll 1
            for (int c = 0; c < 3; ++c) {
                const FabView& F = c == 0 ? Jx : (c == 1 ? Jy : Jz);
#pragma unroll 1
                for (int e = lane; e < SN; e += 32) {
                    const double v = slab[c * SN + e];
                    if (v != 0.0) { atomicAdd(at(F, bx + e % SX, by + (e / SX) % SY, bz + e / (SX * SY)), v); DR_COUNT(red_slab, 1); }
                }
            }
            __syncwarp();                          // every node read before any lane zeroes it
        }
        if (k >= 0) {
            const int gx = (k & 1023) + kb.b0, gy = ((k >> 10) & 1023) + kb.b1, gz = (k >> 20) + kb.b2;
            bx = ((gx + 2) & ~7) - 1; by = ((gy + 2) & ~7) - 1; bz = gz + 1;
#pragma unroll 1
            for (int e = lane; e < 3 * SN; e += 32) slab[e] = 0.0;
        }
        __syncwarp();
    };
    auto set_anchor = [&](int k) {
        const int ax = (k & 1023), gx = ax + kb.b0, gy = ((k >> 10) & 1023) + kb.b1, gz = (k >> 20) + kb.b2;
        ur = ring(ax);
        DR_COUNT(cells, lane == 0);
#pragma unroll
        for (int m = 0; m < VL; ++m) {
            const int qv = qv0 + m;
            if constexpr (SLAB) {
                px[m] = slab_at(0, gx + 1, gy + 1 + qu, gz + 1 + qv);
                py[m] = slab_at(1, gx + 1 + ur, gy + 1, gz + 1 + qv);
                pz[m] = slab_at(2, gx + 1 + ur, gy + 1 + qv, gz + 1);
            } else {
                px[m] = at(Jx, gx + 1, gy + 1 + qu, gz + 1 + qv);
                py[m] = at(Jy, gx + 1 + ur, gy + 1, gz + 1 + qv);
                pz[m] = at(Jz, gx + 1 + ur, gy + 1 + qv, gz + 1);
            }
        }
    };
    auto put = [&](double* p, double v) {         // retire one partial sum
        if constexpr (SLAB) *p += v;
        else { atomicAdd(p, v); DR_COUNT(red_retire, 1); }
    };
    // the anchor advances one cell along x: only the plane x = gx+1 leaves the window
    auto slide = [&]() {
        const bool leaving = (ur == 0);
        DR_COUNT(slides, lane == 0);
        DR_COUNT(cells, lane == 0);
#pragma unroll
        for (int m = 0; m < VL; ++m) {
            const double vx = fold(acc[m][0][0]);
            if (sender) put(px[m], vx);
#pragma unroll
            for (int i = 0; i + 1 < QP; ++i) acc[m][0][i] = acc[m][0][i + 1];
            acc[m][0][QP - 1] = 0.0;
#pragma unroll
            for (int i = 0; i < QP; ++i) {
                const double vy = fold(acc[m][1][i]), vz = fold(acc[m][2][i]);
                if (sender && leaving) { put(py[m] + i * stY, vy); put(pz[m] + i * stZ, vz); }
                if (leaving) { acc[m][1][i] = 0.0; acc[m][2][i] = 0.0; }
            }
            px[m] += stX;                               // next X plane
            if (leaving) { py[m] += QS * xY; pz[m] += QS * xZ; }   // now owns X = gx + 1 + QS
        }
        if (leaving) ur = QS - 1;
        else ur -= 1;                                   // same absolute x, one slot lower
        if constexpr (SLAB) __syncwarp();
    };
    auto flush_all = [&]() {                        // the anchor jumps: retire the whole window
        DR_COUNT(jumps, lane == 0);
#pragma unroll
        for (int m = 0; m < VL; ++m)
#pragma unroll
            for (int i = 0; i < QP; ++i) {
                const double vx = fold(acc[m][0][i]), vy = fold(acc[m][1][i]), vz = fold(acc[m][2][i]);
                if (sender) { put(px[m] + i * stX, vx); put(py[m] + i * stY, vy); put(pz[m] + i * stZ, vz); }
                acc[m][0][i] = 0.0; acc[m][1][i] = 0.0; acc[m][2][i] = 0.0;
            }
        if constexpr (SLAB) __syncwarp();
    };

    // one particle (record column pq) of anchor k, deposited without the register window: into the slab when it
    // covers k, else straight to J
    auto deposit_lone = [&](int k, int pq) {
        const bool in_slab = SLAB && covers(k);
        DR_COUNT(lones, lane == 0);
        DR_COUNT(lones_outside, lane == 0 && !in_slab);
        if (lane < QL) {
            const int ax = (k & 1023), gx = ax + kb.b0, gy = ((k >> 10) & 1023) + kb.b1, gz = (k >> 20) + kb.b2;
            const int us = ring(ax);
            const double2 sx = rec[(T::F_SX + us) * CHP + pq];
            const double2 sy = rec[(T::F_SY + qu) * CHP + pq];
            const long lX = in_slab ? 1 : fab_stride(Jx, R0), lY = in_slab ? SX : fab_stride(Jy, R1);
            const long lZ = in_slab ? (long)SX * SY : fab_stride(Jz, R2);
#pragma unroll
            for (int mv = 0; mv < VL; ++mv) {
                const int qv = qv0 + mv;
                double* qx = in_slab ? slab_at(0, gx + 1, gy + 1 + qu, gz + 1 + qv) : at(Jx, gx + 1, gy + 1 + qu, gz + 1 + qv);
                double* qy = in_slab ? slab_at(1, gx + 1 + us, gy + 1, gz + 1 + qv) : at(Jy, gx + 1 + us, gy + 1, gz + 1 + qv);
                double* qz = in_slab ? slab_at(2, gx + 1 + us, gy + 1 + qv, gz + 1) : at(Jz, gx + 1 + us, gy + 1 + qv, gz + 1);
                auto add = [&](double* q, double v) {
                    if (in_slab) *q += v;
                    else { atomicAdd(q, v); DR_COUNT(red_lone, 1); }
                };
                const double2 aby = rec[(T::F_ABY + qv) * CHP + pq];
                const double2 abz = rec[(T::F_ABZ + qv) * CHP + pq];
                const double wx = sy.x * abz.x + sy.y * abz.y;
                const double wy = sx.x * abz.x + sx.y * abz.y;
                const double wz = sx.x * aby.x + sx.y * aby.y;
#pragma unroll
                for (int m = 0; m < T::NCDS; ++m) {
                    const double2 c2 = rec[(T::F_CDS + m) * CHP + pq];
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int e = 2 * m + h;                 // entry e = component (e / QP), prefix index (e % QP)
                        if (e < 3 * QP) {
                            const double cv = h ? c2.y : c2.x;
                            const int c = e / QP, i = e % QP;
                            if (c == 0) add(qx + i * lX, cv * wx);
                            else if (c == 1) add(qy + i * lY, cv * wy);
                            else add(qz + i * lZ, cv * wz);
                        }
                    }
                }
            }
        }
        if constexpr (SLAB) __syncwarp();
    };

    // software prefetch: chunk ch+1 is requested before chunk ch is processed
    double pf[7] = {0, 0, 0, 0, 0, 0, 0};
    auto prefetch = [&](long ch) {
        const long ip = ch * DR_CH + lane;
        if (ch < c_end && ip < np) {
            pf[0] = P.x[ip]; pf[1] = P.y[ip]; pf[2] = P.z[ip]; pf[3] = P.w[ip];
            pf[4] = P.ux[ip]; pf[5] = P.uy[ip]; pf[6] = P.uz[ip];
        }
    };
    prefetch(c_begin);

    for (long ch = c_begin; ch < c_end; ++ch) {
        const long base = ch * DR_CH;
        const int nval = (int)min((long)DR_CH, np - base);
        const double xp = pf[0], yp = pf[1], zp = pf[2], wp = pf[3], uxp = pf[4], uyp = pf[5], uzp = pf[6];
        prefetch(ch + 1);
        // ---------------- phase 1: lane = particle ----------------
        int key = -2;
        bool moved = false;
        if (lane < nval) {
            const ParticleGeom pg = particle_geom(xp, yp, zp, wp, uxp, uyp, uzp, dg);
            double wn[3][N + 1], wo[3][N + 1];
            int inew[3], sh[3];
#pragma unroll
            for (int d = 0; d < 3; ++d) inew[d] = dr_dir<N>(pg.pos_new[d], pg.pos_old[d], wn[d], wo[d], sh[d]);
            moved = (sh[0] != 0) || (sh[1] != 0) || (sh[2] != 0);
            if (!moved) {
                key = pack_key(dg.lo[R0] + inew[R0] - 1, dg.lo[R1] + inew[R1] - 1, dg.lo[R2] + inew[R2] - 1, kb);
                // slots 1..N+1 hold wn[0..N] (new) and wo[0..N] (old, no shift); role X/Y/Z = dir R0/R1/R2
#pragma unroll
                for (int s = 0; s < QS; ++s) {
                    rec[(T::F_SX + s) * CHP + lane] = make_double2(wn[R0][s], wo[R0][s]);
                    rec[(T::F_SY + s) * CHP + lane] = make_double2(wn[R1][s], wo[R1][s]);
                    rec[(T::F_ABY + s) * CHP + lane] = make_double2((1.0 / 3.0) * wn[R1][s] + (1.0 / 6.0) * wo[R1][s],
                                                                    (1.0 / 3.0) * wo[R1][s] + (1.0 / 6.0) * wn[R1][s]);
                    rec[(T::F_ABZ + s) * CHP + lane] = make_double2((1.0 / 3.0) * wn[R2][s] + (1.0 / 6.0) * wo[R2][s],
                                                                    (1.0 / 3.0) * wo[R2][s] + (1.0 / 6.0) * wn[R2][s]);
                }
                // prefix sums over slots 1..N (slot 0 is empty; the sum over 1..N+1 vanishes and is
                // not deposited -- loop trimming of CurrentDeposition.H:777-788 with dl = du = 1)
                double cds[3 * QP + 1];
                cds[3 * QP] = 0.0;
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    constexpr int RR[3] = {R0, R1, R2};
                    const int d = RR[r];                 // role r component = physical component d
                    const double wqd = pg.wq * dg.invdtd[d];
                    double run = 0.0;
#pragma unroll
                    for (int i = 0; i < QP; ++i) {
                        run += wqd * (wo[d][i] - wn[d][i]);
                        cds[r * QP + i] = run;
                    }
                }
#pragma unroll
                for (int m = 0; m < T::NCDS; ++m)
                    rec[(T::F_CDS + m) * CHP + lane] = make_double2(cds[2 * m], cds[2 * m + 1]);
            } else {
                key = -1;
            }
        }
        // particles that changed cell: append to the list (warp-aggregated)
        {
            const unsigned mm = __ballot_sync(FULL, moved);
            if (mm) {
                int basei = 0;
                if (lane == 0) basei = atomicAdd(list_count, __popc(mm));
                basei = __shfl_sync(FULL, basei, 0);
                if (moved) list[basei + __popc(mm & ((1u << lane) - 1u))] = (int)(base + lane);
            }
            DR_COUNT(chunks, lane == 0);
            DR_COUNT(particles, lane < nval);
            DR_COUNT(movers, moved);
        }
        __syncwarp();
        // ---------------- phase 2: lane = stencil lines ----------------
        {
            const int prev = __shfl_up_sync(FULL, key, 1);
            const int next = __shfl_down_sync(FULL, key, 1);
            const bool head = (lane < nval) && (lane == 0 || key != prev);
            unsigned heads = __ballot_sync(FULL, head);
            // A lone particle of another cell between two particles of the same (or of consecutive)
            // cells moved there after the last sort.  As a run of its own it would retire the whole
            // register window twice; instead its 3 x QP x QL contributions go straight to J and the
            // surrounding run continues untouched.
            const bool lone = lane > 0 && lane < nval - 1 && key >= 0 && prev >= 0 && next >= 0 && key != prev &&
                              key != next && (next == prev || next == prev + 1);
            const unsigned lones = __ballot_sync(FULL, lone);
            while (heads) {
                const int start = __ffs(heads) - 1;
                heads &= heads - 1;
                const int end = heads ? (__ffs(heads) - 1) : nval;
                const int k = __shfl_sync(FULL, key, start);
                if ((lones >> start) & 1u) { deposit_lone(k, start); continue; }
                if (k < 0) continue;
                DR_COUNT(runs, lane == 0);
                if (k != cur) {
                    const bool inside = !SLAB || covers(k);
                    if (cur >= 0 && k == cur + 1 && inside) slide();
                    else {
                        if (cur >= 0) flush_all();
                        if (!inside) rebase(k);
                        set_anchor(k);
                    }
                    cur = k;
                }
                auto accumulate = [&](int pq) {
                    const double2 sx = rec[(T::F_SX + ur) * CHP + pq];     // (Sx_new, Sx_old)[1+ur]
                    const double2 sy = rec[(T::F_SY + qu) * CHP + pq];     // (Sy_new, Sy_old)[1+u]
                    double cds[2 * T::NCDS];
#pragma unroll
                    for (int m = 0; m < T::NCDS; ++m) {
                        const double2 c2 = rec[(T::F_CDS + m) * CHP + pq];
                        cds[2 * m] = c2.x; cds[2 * m + 1] = c2.y;
                    }
#pragma unroll
                    for (int mv = 0; mv < VL; ++mv) {
                        const double2 aby = rec[(T::F_ABY + qv0 + mv) * CHP + pq];   // (Ay, By)[1+v]
                        const double2 abz = rec[(T::F_ABZ + qv0 + mv) * CHP + pq];   // (Az, Bz)[1+v]
                        double w3[3];
                        w3[0] = sy.x * abz.x + sy.y * abz.y;    // Jx line (j, k) = (1+u, 1+v)
                        w3[1] = sx.x * abz.x + sx.y * abz.y;    // Jy line (i, k) = (1+ur, 1+v)
                        w3[2] = sx.x * aby.x + sx.y * aby.y;    // Jz line (i, j) = (1+ur, 1+v)
#pragma unroll
                        for (int c = 0; c < 3; ++c)
#pragma unroll
                            for (int i = 0; i < QP; ++i) acc[mv][c][i] += cds[c * QP + i] * w3[c];
                    }
                };
                // the run [start, end) is contiguous (moved particles have their own key): slot g of
                // the pass takes particles start+g, start+g+NG, ...
                if (active_q)
                    for (int pq = start + g; pq < end; pq += NG) accumulate(pq);
            }
        }
        __syncwarp();
    }
    if (cur >= 0) flush_all();
    if constexpr (SLAB) rebase(-1);
}

// ================================================================================================
// particles that changed cell: full stencil
// ================================================================================================
template <int N> struct GeneralCfg {
    static constexpr int S = N + 3;                 // window slots per direction
    static constexpr int PN = N + 2;                // prefix entries deposited
    static constexpr int NB = (S * S + 31) / 32;    // b values per lane
    static constexpr int BH = (S + NB - 1) / NB;
    static constexpr int NLANES = S * BH;
    static constexpr int F_SNX = 0, F_SOX = S, F_SNY = 2 * S, F_SOY = 3 * S;
    static constexpr int F_AY = 4 * S, F_BY = 5 * S, F_AZ = 6 * S, F_BZ = 7 * S;
    static constexpr int F_CDS = 8 * S;
    static constexpr int NF = 8 * S + 3 * PN;
    static constexpr int NJX = S * S * PN;          // Jx of one stencil, staged x-fastest before it goes to J
    static constexpr int WARP_DOUBLES = NF * DR_CHP + NJX;   // shared memory per warp
};

template <int N, int NW>
__global__ void __launch_bounds__(NW * 32, (NW <= 4 ? 3 : 1))
deposit_general_kernel(SoaView P, const int* __restrict__ list, const int* __restrict__ list_count,
                       FabView Jx, FabView Jy, FabView Jz, DepositGeom dg, KeyBase kb) {
    using T = GeneralCfg<N>;
    constexpr int S = T::S, PN = T::PN, NB = T::NB, NF = T::NF, CHP = DR_CHP;
    PIC_DYNAMIC_SMEM(double, smem);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double* rec = smem + (size_t)warp * T::WARP_DOUBLES;
    double* xs = rec + NF * CHP;
    const int count = *list_count;
    const int nchunks = (count + DR_CH - 1) / DR_CH;
    // lane (a, bh) owns lines (a, b), b = bh + nb*BH:  Jx (j=a,k=b), Jy (i=a,k=b), Jz (i=a,j=b)
    const int a = lane % S, bh = lane / S;
    const bool active = lane < T::NLANES;
    double acc[NB][3][PN];
#pragma unroll
    for (int nb = 0; nb < NB; ++nb)
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int i = 0; i < PN; ++i) acc[nb][c][i] = 0.0;

    // Called by the whole warp (k is warp-uniform).  Jy and Jz go to J from the lines: the lanes of one
    // reduction differ in x by a, so S of them share a row.  The Jx lines run along x themselves, so one
    // reduction would touch 18 different rows; Jx is staged in xs instead and sent x-fastest, a warp
    // instruction then covering rows of PN consecutive nodes.
    auto flush = [&](int k) {
        if (k < 0) return;
        const int gx = (k & 1023) + kb.b0, gy = ((k >> 10) & 1023) + kb.b1, gz = (k >> 20) + kb.b2;
        if (active) {
#pragma unroll
            for (int nb = 0; nb < NB; ++nb) {
                const int b = bh + nb * T::BH;
                if (b < S) {
                    double* py = &Jy(gx + a, gy, gz + b);
                    double* pz = &Jz(gx + a, gy + b, gz);
#pragma unroll
                    for (int i = 0; i < PN; ++i) {
                        const double vy = acc[nb][1][i], vz = acc[nb][2][i];
                        xs[(b * S + a) * PN + i] = acc[nb][0][i];        // Jx(gx + i, gy + a, gz + b)
                        if (vy != 0.0) atomicAdd(py + i * Jy.sj, vy);
                        if (vz != 0.0) atomicAdd(pz + i * Jz.sk, vz);
                        acc[nb][0][i] = 0.0; acc[nb][1][i] = 0.0; acc[nb][2][i] = 0.0;
                    }
                }
            }
        }
        __syncwarp();
#pragma unroll 1
        for (int e = lane; e < T::NJX; e += 32) {
            const double v = xs[e];
            if (v != 0.0) atomicAdd(&Jx(gx + e % PN, gy + (e / PN) % S, gz + e / (PN * S)), v);
        }
        __syncwarp();                                  // xs read by every lane before the next flush writes it
    };

    for (int ch = blockIdx.x * NW + warp; ch < nchunks; ch += gridDim.x * NW) {
        const int base = ch * DR_CH;
        const int nval = min(DR_CH, count - base);
        int key = -2;
        if (lane < nval) {
            const long ip = list[base + lane];
            const ParticleGeom pg = particle_geom(P.x[ip], P.y[ip], P.z[ip], P.w[ip], P.ux[ip], P.uy[ip], P.uz[ip], dg);
            double sn[3][S], so[3][S];
            int inew[3], sh[3];
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                double wn[N + 1], wo[N + 1];
                inew[d] = dr_dir<N>(pg.pos_new[d], pg.pos_old[d], wn, wo, sh[d]);
                sn[d][0] = 0.0; sn[d][N + 2] = 0.0;
#pragma unroll
                for (int s = 0; s <= N; ++s) sn[d][s + 1] = wn[s];
                dr_place_old<N>(so[d], wo, sh[d]);
            }
            key = pack_key(dg.lo[0] + inew[0] - 1, dg.lo[1] + inew[1] - 1, dg.lo[2] + inew[2] - 1, kb);
#pragma unroll
            for (int s = 0; s < S; ++s) {
                rec[(T::F_SNX + s) * CHP + lane] = sn[0][s];
                rec[(T::F_SOX + s) * CHP + lane] = so[0][s];
                rec[(T::F_SNY + s) * CHP + lane] = sn[1][s];
                rec[(T::F_SOY + s) * CHP + lane] = so[1][s];
                rec[(T::F_AY + s) * CHP + lane] = (1.0 / 3.0) * sn[1][s] + (1.0 / 6.0) * so[1][s];
                rec[(T::F_BY + s) * CHP + lane] = (1.0 / 3.0) * so[1][s] + (1.0 / 6.0) * sn[1][s];
                rec[(T::F_AZ + s) * CHP + lane] = (1.0 / 3.0) * sn[2][s] + (1.0 / 6.0) * so[2][s];
                rec[(T::F_BZ + s) * CHP + lane] = (1.0 / 3.0) * so[2][s] + (1.0 / 6.0) * sn[2][s];
            }
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                const double wqd = pg.wq * dg.invdtd[d];
                // loop trimming of the reference (:777-788): entries outside [dl, N+1-du] are not deposited
                const int dl = (sh[d] < 0) ? 0 : 1, du = (sh[d] > 0) ? 0 : 1;
                double run = 0.0;
#pragma unroll
                for (int i = 0; i < PN; ++i) {
                    run += wqd * (so[d][i] - sn[d][i]);
                    const bool live = (i >= dl) && (i <= N + 1 - du);
                    rec[(T::F_CDS + d * PN + i) * CHP + lane] = live ? run : 0.0;
                }
            }
        }
        __syncwarp();
        int cur = -1;
        for (int pp = 0; pp < nval; ++pp) {
            const int k = __shfl_sync(FULL, key, pp);
            if (k != cur) { flush(cur); cur = k; }
            if (active) {
                const double snx = rec[(T::F_SNX + a) * CHP + pp], sox = rec[(T::F_SOX + a) * CHP + pp];
                const double sny = rec[(T::F_SNY + a) * CHP + pp], soy = rec[(T::F_SOY + a) * CHP + pp];
                double cds[3][PN];
#pragma unroll
                for (int c = 0; c < 3; ++c)
#pragma unroll
                    for (int i = 0; i < PN; ++i) cds[c][i] = rec[(T::F_CDS + c * PN + i) * CHP + pp];
#pragma unroll
                for (int nb = 0; nb < NB; ++nb) {
                    const int b = bh + nb * T::BH;
                    if (b < S) {
                        const double ay_ = rec[(T::F_AY + b) * CHP + pp], by_ = rec[(T::F_BY + b) * CHP + pp];
                        const double az_ = rec[(T::F_AZ + b) * CHP + pp], bz_ = rec[(T::F_BZ + b) * CHP + pp];
                        const double wx = sny * az_ + soy * bz_;
                        const double wy = snx * az_ + sox * bz_;
                        const double wz = snx * ay_ + sox * by_;
#pragma unroll
                        for (int i = 0; i < PN; ++i) {
                            acc[nb][0][i] += cds[0][i] * wx;
                            acc[nb][1][i] += cds[1][i] * wy;
                            acc[nb][2][i] += cds[2][i] * wz;
                        }
                    }
                }
            }
        }
        flush(cur);
        __syncwarp();
    }
}

template <int N>
static int launch_runs(SoaView P, long np, const pic_fab J[3], const DepositGeom& dg, cudaStream_t s) {
    constexpr int NWQ = 4, MINB = 4, NWG = 4;        // general kernel: 4 warps x 3 CTAs per SM (was 8 x 1: latency bound)
    using TQ = QuietCfg<N>;
    using TG = GeneralCfg<N>;
    for (int d = 0; d < 3; ++d)
        for (int c = 0; c < 3; ++c)
            if (J[c].hi[d] - J[c].lo[d] + 2 > 1022) return fail("pic_deposit_esirkepov: J extent > 1020 points per rank");
    KeyBase kb;
    kb.b0 = min(J[0].lo[0], min(J[1].lo[0], J[2].lo[0])) - 1;
    kb.b1 = min(J[0].lo[1], min(J[1].lo[1], J[2].lo[1])) - 1;
    kb.b2 = min(J[0].lo[2], min(J[1].lo[2], J[2].lo[2])) - 1;
#ifndef PIC_SIMT_HOST
    // list of particles that changed cell + its counter (stream-ordered scratch, freed after use).
    // Keep the pool's memory across host synchronisations (default threshold 0 would unmap it).
    static bool pool_done = false;
    if (!pool_done) {
        int dev = 0; cudaGetDevice(&dev);
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
            unsigned long long thr = ~0ull;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
        }
        pool_done = true;
    }
    int* scratch = nullptr;
    if (cudaMallocAsync((void**)&scratch, sizeof(int) * (size_t)(np + 1), s) != cudaSuccess)
        return fail("pic_deposit_esirkepov: cannot allocate %ld B of scratch", (long)(sizeof(int) * (np + 1)));
    int* list_count = scratch;
    int* list = scratch + 1;
    cudaMemsetAsync(list_count, 0, sizeof(int), s);
    // roles X,Y,Z = x,y,z: bins are x-fastest, the window slides along x.  (Sliding along z with lanes
    // along x -- <2,0,1> with z-fastest bins -- coalesces the retired planes but was measured no
    // faster for the deposition and 2.2x slower for the gather: 4-way bank conflicts between the
    // cells of a warp in the shared E/B block.)
    constexpr int VL2 = ((N + 1) % 2 == 0) ? 2 : 1;
    using TQ2 = QuietCfg<N, VL2>;
    const bool four = (g_runs_variant & 4) && N == 3;
    const bool two = !four && (g_runs_variant & 1) && VL2 == 2, slotred = (g_runs_variant & 2) != 0;
    constexpr int VL4 = (N == 3) ? 4 : 1;
    using TQ4 = QuietCfg<N, VL4>;
    // J slab: 2 cell layers, 4 warps x 2 CTAs per SM (104 KB of shared memory per CTA, 154 registers, no spills;
    // 3 warps x 3 CTAs with one layer and 2 warps x 4 CTAs measured the same)
    const bool slab = !four && !two && !slotred && (g_runs_variant & 8);
    using TS2 = SlabCfg<N, 2>;
    auto kq = four ? (slotred ? deposit_quiet_kernel<N, NWQ, 3, 0, 1, 2, VL4, true> : deposit_quiet_kernel<N, NWQ, 3, 0, 1, 2, VL4, false>)
            : two ? (slotred ? deposit_quiet_kernel<N, NWQ, MINB, 0, 1, 2, VL2, true> : deposit_quiet_kernel<N, NWQ, MINB, 0, 1, 2, VL2, false>)
            : slotred ? deposit_quiet_kernel<N, NWQ, MINB, 0, 1, 2, 1, true>
            : !slab ? deposit_quiet_kernel<N, NWQ, MINB, 0, 1, 2, 1, false>
            : deposit_quiet_kernel<N, 4, 2, 0, 1, 2, 1, false, 2>;
    const int nwq = 4;
    auto kg = deposit_general_kernel<N, NWG>;
    const size_t smem_q = (size_t)nwq * TQ::NF * (four ? TQ4::CHP : two ? TQ2::CHP : TQ::CHP) * sizeof(double2) +
                          (slab ? (size_t)nwq * 3 * TS2::SN * sizeof(double) : 0);
    const size_t smem_g = (size_t)NWG * TG::WARP_DOUBLES * sizeof(double);
    static bool attr_done[16] = {false};
    const int vidx = (two ? 1 : 0) + (slotred ? 2 : 0) + (four ? 4 : 0) + (slab ? 8 : 0);
    if (!attr_done[vidx]) {
        cudaFuncSetAttribute(kq, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_q);
        cudaFuncSetAttribute(kg, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_g);
        attr_done[vidx] = true;
    }
    const long nchunks = (np + DR_CH - 1) / DR_CH;
    const int cpw = 16;   // 512 consecutive particles per warp: long runs, few boundaries
    const long nwarps = (nchunks + cpw - 1) / cpw;
    const unsigned grid_q = (unsigned)((nwarps + nwq - 1) / nwq);
    J3 j3; j3.v[0] = make_view(J[0]); j3.v[1] = make_view(J[1]); j3.v[2] = make_view(J[2]);
    kq<<<grid_q, nwq * 32, smem_q, s>>>(P, np, cpw, j3, dg, kb, list, list_count);
    kg<<<NUM_SMS * 3, NWG * 32, smem_g, s>>>(P, list, list_count, make_view(J[0]), make_view(J[1]), make_view(J[2]), dg, kb);
    count_launch(2);
    cudaFreeAsync(scratch, s);
    return check_launch("pic_deposit_esirkepov(runs)") ? 0 : 1;
}
#else
    // tests/host_harness: the same two kernels under the SIMT emulator (host memory, no CUDA runtime)
    std::vector<int> scratch_h((size_t)np + 1, 0);
    int* list_count = scratch_h.data();
    int* list = scratch_h.data() + 1;
    constexpr int VL2 = ((N + 1) % 2 == 0) ? 2 : 1;
    using TQ2 = QuietCfg<N, VL2>;
    const bool four = (g_runs_variant & 4) && N == 3;
    const bool two = !four && (g_runs_variant & 1) && VL2 == 2, slotred = (g_runs_variant & 2) != 0;
    constexpr int VL4 = (N == 3) ? 4 : 1;
    using TQ4 = QuietCfg<N, VL4>;
    const bool slab = !four && !two && !slotred && (g_runs_variant & 8);
    using TS2 = SlabCfg<N, 2>;
    const int nwq = 4;
    const size_t smem_q = (size_t)nwq * TQ::NF * (four ? TQ4::CHP : two ? TQ2::CHP : TQ::CHP) * sizeof(double2) +
                          (slab ? (size_t)nwq * 3 * TS2::SN * sizeof(double) : 0);
    const size_t smem_g = (size_t)NWG * TG::WARP_DOUBLES * sizeof(double);
    const long nchunks = (np + DR_CH - 1) / DR_CH;
    const int cpw = 16;
    const long nwarps = (nchunks + cpw - 1) / cpw;
    const unsigned grid_q = (unsigned)((nwarps + nwq - 1) / nwq);
    J3 j3; j3.v[0] = make_view(J[0]); j3.v[1] = make_view(J[1]); j3.v[2] = make_view(J[2]);
    const FabView v0 = make_view(J[0]), v1 = make_view(J[1]), v2 = make_view(J[2]);
    (void)s;
    ::simt::launch(dim3(grid_q), dim3(nwq * 32), smem_q, [&] {
        if (four && slotred) deposit_quiet_kernel<N, NWQ, 3, 0, 1, 2, VL4, true>(P, np, cpw, j3, dg, kb, list, list_count);
        else if (four) deposit_quiet_kernel<N, NWQ, 3, 0, 1, 2, VL4, false>(P, np, cpw, j3, dg, kb, list, list_count);
        else if (two && slotred) deposit_quiet_kernel<N, NWQ, MINB, 0, 1, 2, VL2, true>(P, np, cpw, j3, dg, kb, list, list_count);
        else if (two) deposit_quiet_kernel<N, NWQ, MINB, 0, 1, 2, VL2, false>(P, np, cpw, j3, dg, kb, list, list_count);
        else if (slotred) deposit_quiet_kernel<N, NWQ, MINB, 0, 1, 2, 1, true>(P, np, cpw, j3, dg, kb, list, list_count);
        else if (!slab) deposit_quiet_kernel<N, NWQ, MINB, 0, 1, 2, 1, false>(P, np, cpw, j3, dg, kb, list, list_count);
        else deposit_quiet_kernel<N, 4, 2, 0, 1, 2, 1, false, 2>(P, np, cpw, j3, dg, kb, list, list_count);
    });
    ::simt::launch(dim3(4), dim3(NWG * 32), smem_g,
                   [&] { deposit_general_kernel<N, NWG>(P, list, list_count, v0, v1, v2, dg, kb); });
    return 0;
}
#endif

// The listed particles of another deposition kernel (deposit_cells.cu) through deposit_general_kernel.
template <int N>
static int launch_general(SoaView P, const int* list, const int* list_count, const pic_fab J[3], const DepositGeom& dg,
                          cudaStream_t s) {
    constexpr int NWG = 8;
    using TG = GeneralCfg<N>;
    for (int d = 0; d < 3; ++d)
        for (int c = 0; c < 3; ++c)
            if (J[c].hi[d] - J[c].lo[d] + 2 > 1022) return fail("pic_deposit_esirkepov: J extent > 1020 points per rank");
    KeyBase kb;
    kb.b0 = min(J[0].lo[0], min(J[1].lo[0], J[2].lo[0])) - 1;
    kb.b1 = min(J[0].lo[1], min(J[1].lo[1], J[2].lo[1])) - 1;
    kb.b2 = min(J[0].lo[2], min(J[1].lo[2], J[2].lo[2])) - 1;
    const size_t smem_g = (size_t)NWG * TG::WARP_DOUBLES * sizeof(double);
    auto kg = deposit_general_kernel<N, NWG>;
#ifndef PIC_SIMT_HOST
    static bool attr_done = false;
    if (!attr_done) {
        cudaFuncSetAttribute(kg, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_g);
        attr_done = true;
    }
    kg<<<NUM_SMS, NWG * 32, smem_g, s>>>(P, list, list_count, make_view(J[0]), make_view(J[1]), make_view(J[2]), dg, kb);
    count_launch();
    return check_launch("pic_deposit_esirkepov(general)") ? 0 : 1;
#else       // tests/host_harness (this file is also compiled untransformed): the emulator's launch
    (void)s; (void)kg;
    const FabView v0 = make_view(J[0]), v1 = make_view(J[1]), v2 = make_view(J[2]);
    ::simt::launch(dim3(4), dim3(NWG * 32), smem_g, [&] { deposit_general_kernel<N, NWG>(P, list, list_count, v0, v1, v2, dg, kb); });
    return 0;
#endif
}
int deposit_general_launch(SoaView P, const int* list, const int* list_count, const pic_fab J[3], const DepositGeom& dg,
                           int nox, cudaStream_t s) {
    if (nox == 1) return launch_general<1>(P, list, list_count, J, dg, s);
    if (nox == 2) return launch_general<2>(P, list, list_count, J, dg, s);
    return launch_general<3>(P, list, list_count, J, dg, s);
}

int deposit_runs_launch(const pic_soa* p, long offset, long np, const pic_fab J[3],
                        const DepositGeom& dg, int nox, cudaStream_t s) {
    SoaView P = make_soa(*p, offset);
    if (nox == 1) return launch_runs<1>(P, np, J, dg, s);
    if (nox == 2) return launch_runs<2>(P, np, J, dg, s);
    return launch_runs<3>(P, np, J, dg, s);
}

}  // namespace pic
