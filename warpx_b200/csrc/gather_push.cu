// Fused field gather + momentum push + position push (PushPX) and momentum-only push (PushP).
//
// Replaces PhysicalParticleContainer::PushPX (reference: Source/Particles/PhysicalParticleContainer.cpp
// :2549-2786) and PushP (:2368-2513): per particle doGatherShapeN (Gather/FieldGather.H:36-424),
// doParticleMomentumPush (Pusher/PushSelector.H:38-102), UpdatePosition (Pusher/UpdatePosition.H:24-45).
//
// Two kernels:
//  * gather_push_global  -- order-agnostic, one thread per particle, fields read through the
//                           read-only path (what the reference does, minus AMReX dispatch);
//  * gather_push_tile    -- cell-sorted particles (pic_bins): one CTA per supercell, the E/B
//                           sub-blocks (supercell + stencil halo) are staged in shared memory once
//                           and every particle of the supercell gathers from shared memory.
#include "pic_common.cuh"
#include "gather_common.cuh"

namespace pic {

template <int N, int G, bool YEE>
__global__ void __launch_bounds__(128)
gather_push_global(SoaView P, long np, GlobalFields fld, GatherGeom gg, double qdt2m /*0.5*q*dt/m*/,
                   double dt, int pusher, int push_position, EscapeView esc, long ip0) {
    const long ip = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (ip >= np) return;
    double xp = P.x[ip], yp = P.y[ip], zp = P.z[ip];
    double F[6];
    gather_fields<N, G, YEE>(fld, gg, xp, yp, zp, F);
    double ux = P.ux[ip], uy = P.uy[ip], uz = P.uz[ip];
    push_particle(xp, yp, zp, ux, uy, uz, F, qdt2m, dt, pusher, push_position);
    P.ux[ip] = ux; P.uy[ip] = uy; P.uz[ip] = uz;
    if (push_position) { P.x[ip] = xp; P.y[ip] = yp; P.z[ip] = zp; esc.note(ip0 + ip, xp, yp, zp); }
}

}  // namespace pic

using namespace pic;

namespace pic {
int gather_push_tile_launch(const pic_soa* p, long offset, long np, const pic_fab E[3],
                            const pic_fab B[3], const GatherGeom& gg, double qdt2m, double dt,
                            int nox, int galerkin, int pusher, int push_position,
                            const pic_bins* bins, const EscapeView& esc, cudaStream_t s);
int gather_push_tile_launch(const pic_soa* p, long offset, long np, const pic_fab E[3],
                            const pic_fab B[3], const GatherGeom& gg, double qdt2m, double dt,
                            int nox, int galerkin, int pusher, int push_position,
                            const pic_bins* bins, const EscapeView& esc, const PermSrc& perm, cudaStream_t s);

static GatherGeom make_gather_geom(const pic_fab E[3], const pic_fab B[3], const double dinv[3], const double xyzmin[3],
                                   const int lo[3]) {
    GatherGeom gg;
    for (int d = 0; d < 3; ++d) { gg.dinv[d] = dinv[d]; gg.xyzmin[d] = xyzmin[d]; gg.lo[d] = lo[d]; }
    for (int c = 0; c < 3; ++c)
        for (int d = 0; d < 3; ++d) { gg.stag[c][d] = E[c].stag[d]; gg.stag[3 + c][d] = B[c].stag[d]; }
    return gg;
}
}

namespace pic {
extern int g_gather_mode;      // gather_push_tile.cu
// Whether pic_gather_push_permuted serves shape order nox: only the default supercell kernel, built for orders 1..3,
// carries out a pending cell sort.
bool gather_push_carries_permutation(int nox) { return nox >= 1 && nox <= 3 && g_gather_mode == PIC_GATHER_TILE; }
}
extern "C" void pic_set_gather_mode(int mode) { pic::g_gather_mode = (mode >= PIC_GATHER_PAIRS && mode <= PIC_GATHER_PAIRS_192) ? mode : 0; }

extern "C" int pic_gather_push(const pic_soa* p, long offset, long np, const pic_fab E[3],
                               const pic_fab B[3], const double dinv[3], const double xyzmin[3],
                               const int lo[3], double q, double m, double dt, int nox,
                               int galerkin, int pusher, int push_position, const pic_bins* bins,
                               const pic_escape_list* escaped, void* stream) {
    if (np == 0) return 0;                                   // PhysicalParticleContainer.cpp:2568
    PIC_REQUIRE(nox >= 1 && nox <= 4, "pic_gather_push: particle shape order %d not in 1..4", nox);
    PIC_REQUIRE(galerkin == 0 || galerkin == 1, "pic_gather_push: galerkin must be 0/1");
    PIC_REQUIRE(pusher >= 0 && pusher <= 2, "pic_gather_push: unknown particle pusher %d", pusher);
    PIC_REQUIRE(offset >= 0 && offset + np <= p->np, "pic_gather_push: range outside the tile");
    const GatherGeom gg = make_gather_geom(E, B, dinv, xyzmin, lo);
    const double qdt2m = 0.5 * q * dt / m;
    cudaStream_t s = (cudaStream_t)stream;
    const EscapeView esc = make_escape(escaped, push_position);
    if (bins && nox <= 3) {        // the supercell kernel is built for orders 1..3; order 4 takes the order-agnostic one
        // the bins index the whole tile: a sub-range would push particles outside it (or the tail twice)
        PIC_REQUIRE(offset == 0 && np == p->np, "pic_gather_push: with cell bins the call must cover the whole tile (offset 0, np = %ld)", (long)p->np);
        if (int rc = gather_push_tile_launch(p, offset, np, E, B, gg, qdt2m, dt, nox, galerkin, pusher,
                                             push_position, bins, esc, s)) return rc;
        if (bins->np_binned >= np) return 0;
        // particles appended after the last sort (neighbour migration): order-agnostic kernel
        offset = bins->np_binned;
        np -= bins->np_binned;
    }
    GlobalFields fld;
    for (int c = 0; c < 3; ++c) { fld.v[c] = make_view(E[c]); fld.v[3 + c] = make_view(B[c]); }
    SoaView P = make_soa(*p, offset);
    const int tpb = 128;
    const unsigned nblk = (unsigned)((np + tpb - 1) / tpb);
    const bool yee = is_yee(E, B);
#define PIC_GP(N, G) do { if (yee) gather_push_global<N, G, true><<<nblk, tpb, 0, s>>>(P, np, fld, gg, qdt2m, dt, pusher, push_position, esc, offset); \
                          else gather_push_global<N, G, false><<<nblk, tpb, 0, s>>>(P, np, fld, gg, qdt2m, dt, pusher, push_position, esc, offset); } while (0)
    if (nox == 1 && galerkin) PIC_GP(1, 1);
    else if (nox == 1) PIC_GP(1, 0);
    else if (nox == 2 && galerkin) PIC_GP(2, 1);
    else if (nox == 2) PIC_GP(2, 0);
    else if (nox == 3 && galerkin) PIC_GP(3, 1);
    else if (nox == 3) PIC_GP(3, 0);
    else if (galerkin) PIC_GP(4, 1);
    else PIC_GP(4, 0);
#undef PIC_GP
    count_launch();
    return check_launch("pic_gather_push") ? 0 : 1;
}

extern "C" int pic_gather_push_permuted(const pic_soa* in, const pic_soa* out, const int* src, const pic_fab E[3],
                                        const pic_fab B[3], const double dinv[3], const double xyzmin[3],
                                        const int lo[3], double q, double m, double dt, int nox, int galerkin,
                                        int pusher, const pic_bins* bins, const pic_escape_list* escaped, void* stream) {
    PIC_REQUIRE(in && out && src && bins, "pic_gather_push_permuted: null argument");
    PIC_REQUIRE(out->np == in->np && bins->np_binned == in->np, "pic_gather_push_permuted: the permutation covers every particle (in %ld, out %ld, binned %ld)",
                (long)in->np, (long)out->np, (long)bins->np_binned);
    PIC_REQUIRE(in->x != out->x, "pic_gather_push_permuted: in and out must be different buffers");
    PIC_REQUIRE(nox >= 1 && nox <= 3, "pic_gather_push_permuted: the supercell kernel serves orders 1..3, not %d", nox);
    PIC_REQUIRE(galerkin == 0 || galerkin == 1, "pic_gather_push_permuted: galerkin must be 0/1");
    PIC_REQUIRE(pusher >= 0 && pusher <= 2, "pic_gather_push_permuted: unknown particle pusher %d", pusher);
    PIC_REQUIRE(pic::gather_push_carries_permutation(nox), "pic_gather_push_permuted: only the default gather kernel permutes (gather mode %d is set)", pic::g_gather_mode);
    if (in->np == 0) return 0;
    PermSrc perm;
    perm.in = make_soa(*in, 0); perm.src = src; perm.id_in = in->idcpu; perm.id_out = out->idcpu;
    return gather_push_tile_launch(out, 0, out->np, E, B, make_gather_geom(E, B, dinv, xyzmin, lo), 0.5 * q * dt / m, dt,
                                   nox, galerkin, pusher, 1, bins, make_escape(escaped, 1), perm, (cudaStream_t)stream);
}
