// Per-particle field gather shared by the order-agnostic and the supercell kernels.
// Follows Source/Particles/Gather/FieldGather.H:36-424 (3D branch :368-422).
#ifndef PIC_GATHER_COMMON_CUH_
#define PIC_GATHER_COMMON_CUH_
#include "pic_common.cuh"

namespace pic {

struct GatherGeom {
    double dinv[3];
    double xyzmin[3];
    int lo[3];
    int stag[6][3];   // Ex Ey Ez Bx By Bz
};

// by-product of the position push: particles whose new position left [lo, hi] (pic_escape_list)
struct EscapeView {
    int* idx; int* count; int cap;
    double lo[3], hi[3];
    __device__ __forceinline__ void note(long ip, double x, double y, double z) const {
        if (idx == nullptr) return;
        if (x < lo[0] || x > hi[0] || y < lo[1] || y > hi[1] || z < lo[2] || z > hi[2]) {
            const int n = atomicAdd(count, 1);      // rare: a thin layer next to the domain faces
            if (n < cap) idx[n] = (int)ip;
        }
    }
};
// A pending cell sort for the push to carry out (pic_gather_push_permuted): slot i of the binned order is particle
// src[i] of `in`.  src == nullptr: no permutation, the push works in place.
struct PermSrc {
    SoaView in;
    const int* __restrict__ src;
    const uint64_t* __restrict__ id_in;
    uint64_t* __restrict__ id_out;
};
inline EscapeView make_escape(const pic_escape_list* e, int push_position) {
    EscapeView v;
    v.idx = nullptr; v.count = nullptr; v.cap = 0;
    for (int d = 0; d < 3; ++d) { v.lo[d] = 0.0; v.hi[d] = 0.0; }
    if (e && push_position) {
        v.idx = e->idx; v.count = e->count; v.cap = e->capacity;
        for (int d = 0; d < 3; ++d) { v.lo[d] = e->lo[d]; v.hi[d] = e->hi[d]; }
    }
    return v;
}

// Weights of one particle along one direction for the four (centering, order) combinations the
// gather needs (FieldGather.H:98-121): [0] node/full, [1] cell/full, [2] node/lowered, [3] cell/lowered.
template <int N, int G>
struct DirWeights {
    double s[4][N + 1];
    int j0[4];
    __device__ __forceinline__ void compute(double pos) {
        constexpr int M = N - G;
#pragma unroll
        for (int t = 0; t < 4; ++t)
#pragma unroll
            for (int n = 0; n <= N; ++n) s[t][n] = 0.0;
        j0[0] = shape_factor<N>(s[0], pos);
        j0[1] = shape_factor<N>(s[1], pos - 0.5);
        j0[2] = shape_factor<M>(s[2], pos);
        j0[3] = shape_factor<M>(s[3], pos - 0.5);
    }
};

// Field access policies -----------------------------------------------------------------------
// A field policy hands out, per component, an accessor positioned at the first stencil point;
// the accessor is then indexed with the (compile-time) stencil offsets.
struct GlobalFields {
    FabView v[6];
    struct Acc {
        const double* __restrict__ b; long sj, sk;
        __device__ __forceinline__ double operator()(int ix, int iy, int iz) const { return __ldg(b + ix + iy * sj + iz * sk); }
    };
    __device__ __forceinline__ Acc at(int c, int i0, int j0, int k0) const {
        return Acc{v[c].p + v[c].off(i0, j0, k0), v[c].sj, v[c].sk};
    }
};

// Gathers the six components at one particle.  Accumulation order as the reference:
// iz outer, iy, ix inner; components Ex,Ey,Ez,Bz,By,Bx (FieldGather.H:368-422).
// YEE = true folds the staggering (Source/WarpX.cpp:2117-2125) into compile-time constants so
// that every weight-array index is static (registers, no local memory).
__host__ __device__ constexpr int yee_stag(int c, int d) { return c < 3 ? (d != c) : (d == c - 3); }

template <int N, int G, bool YEE, class Fields>
__device__ __forceinline__ void gather_fields(const Fields& fld, const GatherGeom& gg, double xp,
                                              double yp, double zp, double F[6]) {
    constexpr int M = N - G;
    DirWeights<N, G> wx, wy, wz;
    wx.compute((xp - gg.xyzmin[0]) * gg.dinv[0]);
    wy.compute((yp - gg.xyzmin[1]) * gg.dinv[1]);
    wz.compute((zp - gg.xyzmin[2]) * gg.dinv[2]);
#pragma unroll
    for (int oc = 0; oc < 6; ++oc) {
        const int c = (oc < 3) ? oc : (8 - oc);   // 0,1,2,5,4,3
        // lowered order along: E_c -> its own direction; B_c -> the two transverse directions
        const bool lx = (c < 3) ? (c == 0) : (c != 3);
        const bool ly = (c < 3) ? (c == 1) : (c != 4);
        const bool lz = (c < 3) ? (c == 2) : (c != 5);
        const int tx = (lx ? 2 : 0) + ((YEE ? yee_stag(c, 0) : gg.stag[c][0]) ? 0 : 1);
        const int ty = (ly ? 2 : 0) + ((YEE ? yee_stag(c, 1) : gg.stag[c][1]) ? 0 : 1);
        const int tz = (lz ? 2 : 0) + ((YEE ? yee_stag(c, 2) : gg.stag[c][2]) ? 0 : 1);
        const int nx = lx ? M : N, ny = ly ? M : N, nz = lz ? M : N;
        const auto F3 = fld.at(c, gg.lo[0] + wx.j0[tx], gg.lo[1] + wy.j0[ty], gg.lo[2] + wz.j0[tz]);
        // separable contraction: sum_z sz ( sum_y sy ( sum_x sx F ) ) -- (n+1)^2 + (n+1) + 1 fewer
        // multiplies than the reference's sx*sy*sz*F form, identical up to rounding (1e-16 relative)
        double acc = 0.0;
#pragma unroll
        for (int iz = 0; iz <= N; ++iz) {
            if (iz > nz) break;
            double accy = 0.0;
#pragma unroll
            for (int iy = 0; iy <= N; ++iy) {
                if (iy > ny) break;
                double accx = 0.0;
#pragma unroll
                for (int ix = 0; ix <= N; ++ix) {
                    if (ix > nx) break;
                    accx += wx.s[tx][ix] * F3(ix, iy, iz);
                }
                accy += wy.s[ty][iy] * accx;
            }
            acc += wz.s[tz][iz] * accy;
        }
        F[c] = acc;
    }
}


// ---- two particles per lane ------------------------------------------------------------------
// Weight type (index into DirWeights::s / j0) and order of component c along direction d, exactly
// as gather_fields selects them.
template <bool YEE>
__device__ __forceinline__ int weight_type(const GatherGeom& gg, int c, int d, bool lowered) {
    return (lowered ? 2 : 0) + ((YEE ? yee_stag(c, d) : gg.stag[c][d]) ? 0 : 1);
}
__host__ __device__ constexpr bool lowered_along(int c, int d) { return (c < 3) ? (c == d) : (c != d + 3); }

// Do the stencils of two particles start at the same grid points for every component?  (Always true
// for two particles of one cell at order 3 or 1 with the Galerkin gather on the Yee grid: node weights
// of order N and cell weights of order N - 1 both start at cell - 1, resp. cell.)
template <int N, int G, bool YEE>
__device__ __forceinline__ bool same_stencils(const GatherGeom& gg, const DirWeights<N, G>& ax, const DirWeights<N, G>& ay,
                                              const DirWeights<N, G>& az, const DirWeights<N, G>& bx,
                                              const DirWeights<N, G>& by, const DirWeights<N, G>& bz) {
    bool same = true;
#pragma unroll
    for (int c = 0; c < 6; ++c) {
        const int tx = weight_type<YEE>(gg, c, 0, lowered_along(c, 0));
        const int ty = weight_type<YEE>(gg, c, 1, lowered_along(c, 1));
        const int tz = weight_type<YEE>(gg, c, 2, lowered_along(c, 2));
        same = same && ax.j0[tx] == bx.j0[tx] && ay.j0[ty] == by.j0[ty] && az.j0[tz] == bz.j0[tz];
    }
    return same;
}

// The six components at two particles with identical stencil points (same_stencils): each grid value is
// loaded once and contracted with both weight sets.  Same accumulation order per particle as gather_fields.
template <int N, int G, bool YEE, class Fields>
__device__ __forceinline__ void gather_fields_pair(const Fields& fld, const GatherGeom& gg,
                                                   const DirWeights<N, G>& ax, const DirWeights<N, G>& ay,
                                                   const DirWeights<N, G>& az, const DirWeights<N, G>& bx,
                                                   const DirWeights<N, G>& by, const DirWeights<N, G>& bz,
                                                   double FA[6], double FB[6]) {
    constexpr int M = N - G;
#pragma unroll
    for (int oc = 0; oc < 6; ++oc) {
        const int c = (oc < 3) ? oc : (8 - oc);   // 0,1,2,5,4,3
        const bool lx = lowered_along(c, 0), ly = lowered_along(c, 1), lz = lowered_along(c, 2);
        const int tx = weight_type<YEE>(gg, c, 0, lx), ty = weight_type<YEE>(gg, c, 1, ly), tz = weight_type<YEE>(gg, c, 2, lz);
        const int nx = lx ? M : N, ny = ly ? M : N, nz = lz ? M : N;
        const auto F3 = fld.at(c, gg.lo[0] + ax.j0[tx], gg.lo[1] + ay.j0[ty], gg.lo[2] + az.j0[tz]);
        double accA = 0.0, accB = 0.0;
#pragma unroll
        for (int iz = 0; iz <= N; ++iz) {
            if (iz > nz) break;
            double accyA = 0.0, accyB = 0.0;
#pragma unroll
            for (int iy = 0; iy <= N; ++iy) {
                if (iy > ny) break;
                double accxA = 0.0, accxB = 0.0;
#pragma unroll
                for (int ix = 0; ix <= N; ++ix) {
                    if (ix > nx) break;
                    const double f = F3(ix, iy, iz);
                    accxA += ax.s[tx][ix] * f;
                    accxB += bx.s[tx][ix] * f;
                }
                accyA += ay.s[ty][iy] * accxA;
                accyB += by.s[ty][iy] * accxB;
            }
            accA += az.s[tz][iz] * accyA;
            accB += bz.s[tz][iz] * accyB;
        }
        FA[c] = accA; FB[c] = accB;
    }
}

// momentum + position update of one particle (PushSelector.H:88-102, UpdatePosition.H:36-44)
__device__ __forceinline__ void push_particle(double& xp, double& yp, double& zp, double& ux,
                                              double& uy, double& uz, const double F[6],
                                              double qdt2m, double dt, int pusher, int push_position) {
    if (pusher == PIC_PUSHER_BORIS) push_boris(ux, uy, uz, F[0], F[1], F[2], F[3], F[4], F[5], qdt2m);
    else if (pusher == PIC_PUSHER_VAY) push_vay(ux, uy, uz, F[0], F[1], F[2], F[3], F[4], F[5], qdt2m);
    else push_hc(ux, uy, uz, F[0], F[1], F[2], F[3], F[4], F[5], qdt2m);
    if (push_position) {
        const double ig = 1.0 / sqrt(1.0 + (ux * ux + uy * uy + uz * uz) * INV_C2);
        xp += ux * ig * dt; yp += uy * ig * dt; zp += uz * ig * dt;
    }
}

}  // namespace pic
#endif
