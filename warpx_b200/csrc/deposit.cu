// Esirkepov charge-conserving current deposition.
//
// Replaces WarpXParticleContainer::DepositCurrent -> doEsirkepovDepositionShapeN<N>
// (reference: Source/Particles/WarpXParticleContainer.cpp:352-827,
//  Source/Particles/Deposition/CurrentDeposition.H:642-907; 3D loops :792-824).
//
// Two kernels:
//  * deposit_global -- order-agnostic: one thread per particle, fp64 red.global per grid point.
//    This is the reference's GPU strategy (Gpu::Atomic::AddNoRet, :799,810,821) and is kept as the
//    drop-in for callers that cannot provide cell bins.
//  * deposit_runs.cu (default with bins) -- cell-sorted particles: runs of same-cell particles are
//    reduced in registers by a warp whose lanes own stencil lines; retired planes go to J with
//    fp64 L2 reductions (~7 per particle instead of 540).  PIC_DEPOSIT_RUNS_SLAB retires them into a
//    per-warp shared-memory J slab first (slower on the H100, DESIGN.md 3.3).
//  * deposit_tile.cu (pic_set_deposit_mode(PIC_DEPOSIT_TILE)) -- same reduction, staged through a shared-memory J block
//    per supercell; kept for comparison (slower on sm_90a: shared fp64 atomics are CAS loops).
#include "pic_common.cuh"
#include "deposit_common.cuh"

namespace pic {

template <int N>
__global__ void __launch_bounds__(128)
deposit_global(SoaView P, long np, FabView Jx, FabView Jy, FabView Jz, DepositGeom dg) {
    const long ip = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (ip >= np) return;
    // a weightless particle deposits nothing and is not required to lie inside the fab: the replicated antenna of a
    // multi-rank run carries zero weights outside the brick that owns each particle (engine.cu, lasers)
    if (P.w[ip] == 0.0) return;
    EsirkepovWeights<N> ew;
    ew.compute(P.x[ip], P.y[ip], P.z[ip], P.w[ip], P.ux[ip], P.uy[ip], P.uz[ip], dg);
    const int bi = dg.lo[0] + ew.i_new - 1, bj = dg.lo[1] + ew.j_new - 1, bk = dg.lo[2] + ew.k_new - 1;
#ifdef PIC_DEBUG_BOUNDS
    if (bi < Jx.lo0 || bi + N + 2 >= Jx.lo0 + Jx.n0 || bj < Jx.lo1 || bj + N + 2 >= Jx.lo1 + Jx.n1 || bk < Jx.lo2 ||
        bk + N + 2 >= Jx.lo2 + Jx.n2)
        printf("deposit_global: ip %ld of %ld base %d %d %d fab lo %d %d %d n %d %d %d  x %.17g %.17g %.17g u %g %g %g w %g xyzmin %g %g %g\n",
               ip, np, bi, bj, bk, Jx.lo0, Jx.lo1, Jx.lo2, Jx.n0, Jx.n1, Jx.n2, P.x[ip], P.y[ip], P.z[ip], P.ux[ip], P.uy[ip], P.uz[ip], P.w[ip],
               dg.xyzmin[0], dg.xyzmin[1], dg.xyzmin[2]);
#endif
    constexpr double one_third = 1.0 / 3.0, one_sixth = 1.0 / 6.0;
    // Same loop nests, trimming and accumulation order as CurrentDeposition.H:792-824.
    for (int k = ew.dkl; k <= N + 2 - ew.dku; ++k)
        for (int j = ew.djl; j <= N + 2 - ew.dju; ++j) {
            double sdxi = 0.0;
            const double wjk = one_third * (ew.sy_new[j] * ew.sz_new[k] + ew.sy_old[j] * ew.sz_old[k])
                             + one_sixth * (ew.sy_new[j] * ew.sz_old[k] + ew.sy_old[j] * ew.sz_new[k]);
            for (int i = ew.dil; i <= N + 1 - ew.diu; ++i) {
                sdxi += ew.wqx * (ew.sx_old[i] - ew.sx_new[i]) * wjk;
                atomicAdd(&Jx(bi + i, bj + j, bk + k), sdxi);
            }
        }
    for (int k = ew.dkl; k <= N + 2 - ew.dku; ++k)
        for (int i = ew.dil; i <= N + 2 - ew.diu; ++i) {
            double sdyj = 0.0;
            const double wik = one_third * (ew.sx_new[i] * ew.sz_new[k] + ew.sx_old[i] * ew.sz_old[k])
                             + one_sixth * (ew.sx_new[i] * ew.sz_old[k] + ew.sx_old[i] * ew.sz_new[k]);
            for (int j = ew.djl; j <= N + 1 - ew.dju; ++j) {
                sdyj += ew.wqy * (ew.sy_old[j] - ew.sy_new[j]) * wik;
                atomicAdd(&Jy(bi + i, bj + j, bk + k), sdyj);
            }
        }
    for (int j = ew.djl; j <= N + 2 - ew.dju; ++j)
        for (int i = ew.dil; i <= N + 2 - ew.diu; ++i) {
            double sdzk = 0.0;
            const double wij = one_third * (ew.sx_new[i] * ew.sy_new[j] + ew.sx_old[i] * ew.sy_old[j])
                             + one_sixth * (ew.sx_new[i] * ew.sy_old[j] + ew.sx_old[i] * ew.sy_new[j]);
            for (int k = ew.dkl; k <= N + 1 - ew.dku; ++k) {
                sdzk += ew.wqz * (ew.sz_old[k] - ew.sz_new[k]) * wij;
                atomicAdd(&Jz(bi + i, bj + j, bk + k), sdzk);
            }
        }
}

int deposit_tile_launch(const pic_soa* p, long offset, long np, const pic_fab J[3],
                        const DepositGeom& dg, int nox, const pic_bins* bins, cudaStream_t s);
int deposit_runs_launch(const pic_soa* p, long offset, long np, const pic_fab J[3],
                        const DepositGeom& dg, int nox, cudaStream_t s);
int deposit_cells_launch(const pic_soa* p, long offset, long np, const pic_fab J[3], const DepositGeom& dg, int nox,
                         const pic_bins* bins, cudaStream_t s);

static int g_deposit_mode = PIC_DEPOSIT_RUNS;
extern int g_runs_variant;      // deposit_runs.cu
extern int g_cells_two_producers;   // deposit_cells.cu

}  // namespace pic

using namespace pic;

extern "C" void pic_set_deposit_mode(int mode) {
    g_deposit_mode = mode;
    g_cells_two_producers = (mode >= PIC_DEPOSIT_CELLS2 && mode <= PIC_DEPOSIT_CELLS3_WIDE) ? mode - PIC_DEPOSIT_CELLS2 + 1 : 0;
    if (g_cells_two_producers) g_deposit_mode = PIC_DEPOSIT_CELLS;
    g_runs_variant = (mode == PIC_DEPOSIT_RUNS2) ? 1 : (mode == PIC_DEPOSIT_RUNS_SLOTRED) ? 2 : (mode == PIC_DEPOSIT_RUNS2_SLOTRED) ? 3
                   : (mode == PIC_DEPOSIT_RUNS4) ? 4 : (mode == PIC_DEPOSIT_RUNS4_SLOTRED) ? 6
                   : (mode == PIC_DEPOSIT_RUNS_SLAB) ? 8 : 0;
}

extern "C" int pic_deposit_esirkepov(const pic_soa* p, long offset, long np, const pic_fab J[3],
                                     const double dinv[3], const double xyzmin[3], const int lo[3],
                                     double q, double dt, double relative_time, int nox,
                                     const pic_bins* bins, void* stream) {
    if (np == 0 || q == 0.0) return 0;                 // WarpXParticleContainer.cpp:367-370
    PIC_REQUIRE(nox >= 1 && nox <= 4, "pic_deposit_esirkepov: particle shape order %d not in 1..4", nox);
    PIC_REQUIRE(offset >= 0 && offset + np <= p->np, "pic_deposit_esirkepov: range outside the tile");
    PIC_REQUIRE(p->w != nullptr, "pic_deposit_esirkepov: weights missing");
    for (int c = 0; c < 3; ++c)
        for (int d = 0; d < 3; ++d) {
            // guard-cell sanity as WarpXParticleContainer.cpp:375-405: shape + half-step displacement
            PIC_REQUIRE(J[c].ng[d] >= nox, "pic_deposit_esirkepov: J needs more guard cells (ng_J)");
        }
    DepositGeom dg;
    for (int d = 0; d < 3; ++d) { dg.dinv[d] = dinv[d]; dg.xyzmin[d] = xyzmin[d]; dg.lo[d] = lo[d]; }
    dg.q = q; dg.dt = dt; dg.tshift = relative_time + 0.5 * dt;
    dg.invdtd[0] = (1.0 / dt) * dinv[1] * dinv[2];     // CurrentDeposition.H:671-673
    dg.invdtd[1] = (1.0 / dt) * dinv[0] * dinv[2];
    dg.invdtd[2] = (1.0 / dt) * dinv[0] * dinv[1];
    cudaStream_t s = (cudaStream_t)stream;
    if (bins && nox <= 3) {        // order 4: order-agnostic kernel (the run kernels are built for orders 1..3)
        // (the run kernels do not read the bins and accept any range; the bin-driven ones need the whole tile)
        // cell-sorted particles: warp-segmented register reduction (deposit_runs.cu).  The
        // shared-memory-block variant (deposit_tile.cu) is kept for comparison: pic_set_deposit_mode().
        PIC_REQUIRE(np < (1L << 31), "pic_deposit_esirkepov: more than 2^31 particles in one tile");
        const bool cells = g_deposit_mode == PIC_DEPOSIT_CELLS && (nox == 1 || nox == 3) && offset == 0 &&
                           bins->tile[0] == 8 && bins->tile[1] == 8 && bins->tile[2] == 8;
        if (g_deposit_mode != PIC_DEPOSIT_TILE && !cells) return deposit_runs_launch(p, offset, np, J, dg, nox, s);
        // the two bin-driven kernels cover [0, np_binned) of the tile
        PIC_REQUIRE(offset == 0, "pic_deposit_esirkepov: the bin-driven kernels take the whole tile (offset 0)");
        if (cells) { if (int rc = deposit_cells_launch(p, offset, np, J, dg, nox, bins, s)) return rc; }
        else if (int rc = deposit_tile_launch(p, offset, np, J, dg, nox, bins, s)) return rc;
        if (bins->np_binned >= np) return 0;
        offset = bins->np_binned;           // particles appended after the last sort
        np -= bins->np_binned;
    }
    SoaView P = make_soa(*p, offset);
    const int tpb = 128;
    const unsigned nblk = (unsigned)((np + tpb - 1) / tpb);
    FabView jx = make_view(J[0]), jy = make_view(J[1]), jz = make_view(J[2]);
    if (nox == 1) deposit_global<1><<<nblk, tpb, 0, s>>>(P, np, jx, jy, jz, dg);
    else if (nox == 2) deposit_global<2><<<nblk, tpb, 0, s>>>(P, np, jx, jy, jz, dg);
    else if (nox == 3) deposit_global<3><<<nblk, tpb, 0, s>>>(P, np, jx, jy, jz, dg);
    else deposit_global<4><<<nblk, tpb, 0, s>>>(P, np, jx, jy, jz, dg);
    count_launch();
    return check_launch("pic_deposit_esirkepov") ? 0 : 1;
}
