// Shared device/host helpers of the PIC kernels (sm_90a, H100, only; no multi-arch paths).
#ifndef PIC_COMMON_CUH_
#define PIC_COMMON_CUH_

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include "../../include/pic_b200.h"

namespace pic {

// CODATA-2018 as used by the reference (Source/ablastr/constant.H:44-54)
constexpr double C_LIGHT = 299792458.0;
constexpr double MU0 = 1.25663706212e-06;
constexpr double EP0 = 8.8541878128e-12;
constexpr double INV_C2 = 1.0 / (C_LIGHT * C_LIGHT);

constexpr int NUM_SMS = 132;  // H100 SXM

// ---- error handling (mirrors amrex::Abort unless tests ask for return codes) ---------------
int fail(const char* fmt, ...);
void count_launch(long n = 1);
bool check_launch(const char* what);  // cudaGetLastError after a launch

#define PIC_REQUIRE(cond, ...) do { if (!(cond)) return ::pic::fail(__VA_ARGS__); } while (0)

// Dynamic shared memory of a kernel.  PIC_SIMT_HOST is only ever defined by tests/host_harness (the SIMT
// emulator that runs the kernel source on the host, see tests/host_harness/simt_host.h).
#ifdef PIC_SIMT_HOST
#define PIC_DYNAMIC_SMEM(T, name) T* name = reinterpret_cast<T*>(::simt::dynamic_smem())
#define PIC_STATIC_SMEM(T, name, n) T* name = reinterpret_cast<T*>(::simt::block_static(#name, sizeof(T) * (n)))
#else
#define PIC_DYNAMIC_SMEM(T, name) extern __shared__ T name[]
#define PIC_STATIC_SMEM(T, name, n) __shared__ T name[n]
#endif

// ---- array view: amrex::Array4 indexing (Fortran order, arbitrary lower bound) --------------
struct FabView {
    double* __restrict__ p;
    int lo0, lo1, lo2;
    int n0, n1, n2;       // allocated extents
    long sj, sk;          // strides
    __host__ __device__ __forceinline__ long off(int i, int j, int k) const {
        return (long)(i - lo0) + (long)(j - lo1) * sj + (long)(k - lo2) * sk;
    }
    __device__ __forceinline__ double& operator()(int i, int j, int k) const { return p[off(i, j, k)]; }
    __device__ __forceinline__ double ld(int i, int j, int k) const { return __ldg(p + off(i, j, k)); }
};

inline FabView make_view(const pic_fab& f) {
    FabView v;
    v.p = f.p;
    v.lo0 = f.lo[0]; v.lo1 = f.lo[1]; v.lo2 = f.lo[2];
    v.n0 = f.hi[0] - f.lo[0] + 1; v.n1 = f.hi[1] - f.lo[1] + 1; v.n2 = f.hi[2] - f.lo[2] + 1;
    v.sj = v.n0; v.sk = (long)v.n0 * v.n1;
    return v;
}
inline int vlo(const pic_fab& f, int d) { return f.lo[d] + f.ng[d]; }
inline int vhi(const pic_fab& f, int d) { return f.hi[d] - f.ng[d]; }
inline long fab_size(const pic_fab& f) {
    return (long)(f.hi[0] - f.lo[0] + 1) * (f.hi[1] - f.lo[1] + 1) * (f.hi[2] - f.lo[2] + 1);
}
inline bool is_yee(const pic_fab E[3], const pic_fab B[3]) {
    static const int se[3][3] = {{0, 1, 1}, {1, 0, 1}, {1, 1, 0}};
    static const int sb[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int c = 0; c < 3; ++c)
        for (int d = 0; d < 3; ++d)
            if (E[c].stag[d] != se[c][d] || B[c].stag[d] != sb[c][d]) return false;
    return true;
}

struct SoaView {
    double* __restrict__ x; double* __restrict__ y; double* __restrict__ z; double* __restrict__ w;
    double* __restrict__ ux; double* __restrict__ uy; double* __restrict__ uz;
};
inline SoaView make_soa(const pic_soa& p, long offset) {
    SoaView s;
    s.x = p.x + offset; s.y = p.y + offset; s.z = p.z + offset; s.w = p.w ? p.w + offset : nullptr;
    s.ux = p.ux + offset; s.uy = p.uy + offset; s.uz = p.uz + offset;
    return s;
}

// ---- products / sums rounded separately (no FMA contraction) ----------------------------------
// The deposition coordinates x_new, x_old (CurrentDeposition.H:725-736) are evaluated by the CPU
// reference as individually rounded operations; where a particle's displacement per step is below
// the spacing of doubles at its grid coordinate (test_3d_pec_particle) a fused multiply-add changes
// x_old by one unit in the last place and with it the deposited current.  These helpers keep nvcc
// from contracting (the host build of the harness compiles with -ffp-contract=off anyway).
__host__ __device__ __forceinline__ double mul_rn(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ __forceinline__ double add_rn(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
__host__ __device__ __forceinline__ double sub_rn(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}
// x_new = (xp - xmin + tshift*u*gaminv)*dinv ; x_old = x_new - dt*dinv*u*gaminv, left to right
__host__ __device__ __forceinline__ void deposit_coords(double xp, double xmin, double tshift, double u, double gaminv,
                                                        double dinv, double dt, double& x_new, double& x_old) {
    x_new = mul_rn(add_rn(sub_rn(xp, xmin), mul_rn(mul_rn(tshift, u), gaminv)), dinv);
    x_old = sub_rn(x_new, mul_rn(mul_rn(mul_rn(dt, dinv), u), gaminv));
}

// ---- B-spline shape factors (Source/Particles/ShapeFactors.H:27-84) --------------------------
// Written for the evaluation order of the reference; returns the leftmost index.
// Quartic spline around the nearest node, d in [-1/2, 1/2] (ShapeFactors.H:66-77).
__host__ __device__ __forceinline__ void quartic_weights(double* s, double d) {
    const double a = 0.5 - d, b = 0.5 + d;        // products left to right, as the reference evaluates them
    s[0] = (1.0 / 24.0) * a * a * a * a;
    s[1] = (1.0 / 24.0) * (4.75 - 11.0 * d + 4.0 * d * d * (1.5 + d - d * d));
    s[2] = (1.0 / 24.0) * (14.375 + 6.0 * d * d * (d * d - 2.5));
    s[3] = (1.0 / 24.0) * (4.75 + 11.0 * d + 4.0 * d * d * (1.5 - d - d * d));
    s[4] = (1.0 / 24.0) * b * b * b * b;
}
template <int N>
__host__ __device__ __forceinline__ int shape_factor(double* s, double xmid) {
    if constexpr (N == 0) {
        const int j = (int)(xmid + 0.5);
        s[0] = 1.0;
        return j;
    } else if constexpr (N == 1) {
        const int j = (int)xmid;
        const double d = xmid - (double)j;
        s[0] = 1.0 - d; s[1] = d;
        return j;
    } else if constexpr (N == 2) {
        const int j = (int)(xmid + 0.5);
        const double d = xmid - (double)j;
        const double a = 0.5 - d, b = 0.5 + d;
        s[0] = 0.5 * a * a; s[1] = 0.75 - d * d; s[2] = 0.5 * b * b;
        return j - 1;
    } else if constexpr (N == 3) {
        const int j = (int)xmid;
        const double d = xmid - (double)j;
        const double e = 1.0 - d;
        s[0] = (1.0 / 6.0) * e * e * e;
        s[1] = (2.0 / 3.0) - d * d * (1.0 - d / 2.0);
        s[2] = (2.0 / 3.0) - e * e * (1.0 - 0.5 * e);
        s[3] = (1.0 / 6.0) * d * d * d;
        return j - 1;
    } else {
        static_assert(N == 4, "orders 0..4");
        quartic_weights(s, xmid - (double)(int)(xmid + 0.5));
        return (int)(xmid + 0.5) - 2;
    }
}

// Shifted shape factor of the OLD position (ShapeFactors.H:93-156): slot 1 of the (N+3)-slot
// array is the leftmost point of the NEW position's stencil.  s must be pre-zeroed.
template <int N>
__host__ __device__ __forceinline__ int shifted_shape_factor(double* s, double x_old, int i_new) {
    if constexpr (N == 1) {
        const int i = (int)floor(x_old);
        const int sh = i - i_new;
        const double d = x_old - (double)i;
        s[1 + sh] = 1.0 - d; s[2 + sh] = d;
        return i;
    } else if constexpr (N == 2) {
        const int i = (int)(x_old + 0.5);
        const int sh = i - (i_new + 1);
        const double d = x_old - (double)i;
        const double a = 0.5 - d, b = 0.5 + d;
        s[1 + sh] = 0.5 * a * a; s[2 + sh] = 0.75 - d * d; s[3 + sh] = 0.5 * b * b;
        return i - 1;
    } else if constexpr (N == 3) {
        const int i = (int)x_old;
        const int sh = i - (i_new + 1);
        const double d = x_old - (double)i;
        const double e = 1.0 - d;
        s[1 + sh] = (1.0 / 6.0) * e * e * e;
        s[2 + sh] = (2.0 / 3.0) - d * d * (1.0 - d / 2.0);
        s[3 + sh] = (2.0 / 3.0) - e * e * (1.0 - 0.5 * e);
        s[4 + sh] = (1.0 / 6.0) * d * d * d;
        return i - 1;
    } else {
        static_assert(N == 4, "orders 1..4");
        const int i = (int)(x_old + 0.5);
        const int sh = i - (i_new + 2);
        quartic_weights(s + 1 + sh, x_old - (double)i);
        return i - 2;
    }
}

// ---- momentum pushers (Source/Particles/Pusher/UpdateMomentum{Boris,Vay,HigueraCary}.H) -----
__device__ __forceinline__ void push_boris(double& ux, double& uy, double& uz, double Ex, double Ey,
                                           double Ez, double Bx, double By, double Bz, double ec) {
    // ec = 0.5*q*dt/m
    ux += ec * Ex; uy += ec * Ey; uz += ec * Ez;
    const double ig = 1.0 / sqrt(1.0 + (ux * ux + uy * uy + uz * uz) * INV_C2);
    const double tx = ec * ig * Bx, ty = ec * ig * By, tz = ec * ig * Bz;
    const double tsqi = 2.0 / (1.0 + tx * tx + ty * ty + tz * tz);
    const double sx = tx * tsqi, sy = ty * tsqi, sz = tz * tsqi;
    const double px = ux + uy * tz - uz * ty;
    const double py = uy + uz * tx - ux * tz;
    const double pz = uz + ux * ty - uy * tx;
    ux += py * sz - pz * sy;
    uy += pz * sx - px * sz;
    uz += px * sy - py * sx;
    ux += ec * Ex; uy += ec * Ey; uz += ec * Ez;
}

__device__ __forceinline__ void push_vay(double& ux, double& uy, double& uz, double Ex, double Ey,
                                         double Ez, double Bx, double By, double Bz, double bc) {
    // bc = 0.5*q*dt/m ; econst = 2*bc
    const double ec = 2.0 * bc;
    constexpr double ic = 1.0 / C_LIGHT;
    const double ig = 1.0 / sqrt(1.0 + (ux * ux + uy * uy + uz * uz) * INV_C2);
    const double ax = bc * Bx, ay = bc * By, az = bc * Bz;
    const double a2 = ax * ax + ay * ay + az * az;
    const double px = ux + ec * Ex + (uy * az - uz * ay) * ig;
    const double py = uy + ec * Ey + (uz * ax - ux * az) * ig;
    const double pz = uz + ec * Ez + (ux * ay - uy * ax) * ig;
    const double gp2 = (1.0 + (px * px + py * py + pz * pz) * INV_C2);
    const double ust = (px * ax + py * ay + pz * az) * ic;
    const double sig = gp2 - a2;
    const double gi2 = 2.0 / (sig + sqrt(sig * sig + 4.0 * (a2 + ust * ust)));
    const double bg = bc * sqrt(gi2);
    const double tx = bg * Bx, ty = bg * By, tz = bg * Bz;
    const double s = 1.0 / (1.0 + a2 * gi2);
    const double tu = tx * px + ty * py + tz * pz;
    ux = s * (px + tx * tu + py * tz - pz * ty);
    uy = s * (py + ty * tu + pz * tx - px * tz);
    uz = s * (pz + tz * tu + px * ty - py * tx);
}

__device__ __forceinline__ void push_hc(double& ux, double& uy, double& uz, double Ex, double Ey,
                                        double Ez, double Bx, double By, double Bz, double h) {
    // h = 0.5*q*dt/m
    constexpr double ic = 1.0 / C_LIGHT;
    const double mx = ux + h * Ex, my = uy + h * Ey, mz = uz + h * Ez;
    double g = 1.0 + (mx * mx + my * my + mz * mz) * INV_C2;
    const double bx = h * Bx, by = h * By, bz = h * Bz;
    const double b2 = bx * bx + by * by + bz * bz;
    const double sig = g - b2;
    const double ust = (mx * bx + my * by + mz * bz) * ic;
    g = 1.0 / sqrt(0.5 * (sig + sqrt(sig * sig + 4.0 * (b2 + ust * ust))));
    const double tx = g * bx, ty = g * by, tz = g * bz;
    const double s = 1.0 / (1.0 + (tx * tx + ty * ty + tz * tz));
    const double mt = mx * tx + my * ty + mz * tz;
    const double px = s * (mx + mt * tx + my * tz - mz * ty);
    const double py = s * (my + mt * ty + mz * tx - mx * tz);
    const double pz = s * (mz + mt * tz + mx * ty - my * tx);
    ux = px + h * Ex + py * tz - pz * ty;
    uy = py + h * Ey + pz * tx - px * tz;
    uz = pz + h * Ez + px * ty - py * tx;
}

}  // namespace pic
#endif
