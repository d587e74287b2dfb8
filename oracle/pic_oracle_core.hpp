// TEST INFRASTRUCTURE -- CPU oracle of the explicit EM-PIC step (fp64), templated on the leaf
// arithmetic (leaf_restated.hpp = hand restatement, leaf_reference.hpp = reference headers
// compiled verbatim).  Every routine cites the reference lines it follows (paths relative to
// Source/ of ECP-WarpX/WarpX).  Loop order and accumulation order follow the reference's CPU path.
//
// Only tests/, __graft_entry__.smoke() and the cpu_baseline / --impl reference legs of bench.py
// may use this; the product (warpx_b200/) never links, imports or executes anything in oracle/.
#ifndef PIC_ORACLE_CORE_HPP_
#define PIC_ORACLE_CORE_HPP_

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#endif
#include "../include/pic_b200.h"

namespace orc {

constexpr double C_LIGHT = 299792458.0;        // ablastr/constant.H:44
constexpr double MU0 = 1.25663706212e-06;      // ablastr/constant.H:48
constexpr double EP0 = 8.8541878128e-12;       // ablastr/constant.H:46

inline int vlo(const pic_fab& f, int d) { return f.lo[d] + f.ng[d]; }
inline int vhi(const pic_fab& f, int d) { return f.hi[d] - f.ng[d]; }
inline long fab_size(const pic_fab& f) {
    return (long)(f.hi[0] - f.lo[0] + 1) * (f.hi[1] - f.lo[1] + 1) * (f.hi[2] - f.lo[2] + 1);
}
struct W {  // writable view
    double* p; int l0, l1, l2; long sj, sk;
    explicit W(const pic_fab& f) : p(f.p), l0(f.lo[0]), l1(f.lo[1]), l2(f.lo[2]),
        sj(f.hi[0] - f.lo[0] + 1), sk(sj * (long)(f.hi[1] - f.lo[1] + 1)) {}
    double& operator()(int i, int j, int k) const { return p[(i - l0) + (j - l1) * sj + (k - l2) * sk]; }
};

// ============================================================================================
// FDTD.  FiniteDifferenceSolver::EvolveBCartesian (FieldSolver/FiniteDifferenceSolver/EvolveB.cpp:164-186)
// over mfi.tilebox(ixType) = valid points of each component (:159-161).
// ============================================================================================
template <class L>
void evolve_b(const pic_fab B[3], const pic_fab E[3], const pic_stencil& st, double dt) {
    const int a = st.algo;
    auto Ex = L::arr(E[0]); auto Ey = L::arr(E[1]); auto Ez = L::arr(E[2]);
    W Bx(B[0]), By(B[1]), Bz(B[2]);
#pragma omp parallel
    {
#pragma omp for nowait
        for (int k = vlo(B[0], 2); k <= vhi(B[0], 2); ++k)
            for (int j = vlo(B[0], 1); j <= vhi(B[0], 1); ++j)
                for (int i = vlo(B[0], 0); i <= vhi(B[0], 0); ++i)
                    Bx(i, j, k) += dt * L::template upward<2>(a, Ey, st.cz, i, j, k)
                                 - dt * L::template upward<1>(a, Ez, st.cy, i, j, k);
#pragma omp for nowait
        for (int k = vlo(B[1], 2); k <= vhi(B[1], 2); ++k)
            for (int j = vlo(B[1], 1); j <= vhi(B[1], 1); ++j)
                for (int i = vlo(B[1], 0); i <= vhi(B[1], 0); ++i)
                    By(i, j, k) += dt * L::template upward<0>(a, Ez, st.cx, i, j, k)
                                 - dt * L::template upward<2>(a, Ex, st.cz, i, j, k);
#pragma omp for nowait
        for (int k = vlo(B[2], 2); k <= vhi(B[2], 2); ++k)
            for (int j = vlo(B[2], 1); j <= vhi(B[2], 1); ++j)
                for (int i = vlo(B[2], 0); i <= vhi(B[2], 0); ++i)
                    Bz(i, j, k) += dt * L::template upward<1>(a, Ex, st.cy, i, j, k)
                                 - dt * L::template upward<0>(a, Ey, st.cx, i, j, k);
    }
}

// FiniteDifferenceSolver::EvolveECartesian (EvolveE.cpp:179-216): E += c^2 dt (curl B - mu0 J),
// c2 = PhysConst::c*PhysConst::c (:134); no EB, no F term.
template <class L>
void evolve_e(const pic_fab E[3], const pic_fab B[3], const pic_fab J[3], const pic_stencil& st,
              double dt) {
    const int a = st.algo;
    constexpr double c2 = C_LIGHT * C_LIGHT;
    auto Bx = L::arr(B[0]); auto By = L::arr(B[1]); auto Bz = L::arr(B[2]);
    W Ex(E[0]), Ey(E[1]), Ez(E[2]);
    W jx(J[0]), jy(J[1]), jz(J[2]);
#pragma omp parallel
    {
#pragma omp for nowait
        for (int k = vlo(E[0], 2); k <= vhi(E[0], 2); ++k)
            for (int j = vlo(E[0], 1); j <= vhi(E[0], 1); ++j)
                for (int i = vlo(E[0], 0); i <= vhi(E[0], 0); ++i)
                    Ex(i, j, k) += c2 * dt * (-L::template downward<2>(a, By, st.cz, i, j, k)
                                              + L::template downward<1>(a, Bz, st.cy, i, j, k)
                                              - MU0 * jx(i, j, k));
#pragma omp for nowait
        for (int k = vlo(E[1], 2); k <= vhi(E[1], 2); ++k)
            for (int j = vlo(E[1], 1); j <= vhi(E[1], 1); ++j)
                for (int i = vlo(E[1], 0); i <= vhi(E[1], 0); ++i)
                    Ey(i, j, k) += c2 * dt * (-L::template downward<0>(a, Bz, st.cx, i, j, k)
                                              + L::template downward<2>(a, Bx, st.cz, i, j, k)
                                              - MU0 * jy(i, j, k));
#pragma omp for nowait
        for (int k = vlo(E[2], 2); k <= vhi(E[2], 2); ++k)
            for (int j = vlo(E[2], 1); j <= vhi(E[2], 1); ++j)
                for (int i = vlo(E[2], 0); i <= vhi(E[2], 0); ++i)
                    Ez(i, j, k) += c2 * dt * (-L::template downward<1>(a, Bx, st.cy, i, j, k)
                                              + L::template downward<0>(a, By, st.cx, i, j, k)
                                              - MU0 * jz(i, j, k));
    }
}

// ============================================================================================
// Gather.  doGatherShapeN<order,galerkin> (Particles/Gather/FieldGather.H:36-424, 3D branch
// :368-422).  Per direction two centerings (node: x, cell: x-0.5, :98-109) times two orders
// (full, and order-galerkin for the component's own direction, :110-121).  Accumulation order:
// iz outer, iy, ix inner; Ex, Ey, Ez, Bz, By, Bx.
// ============================================================================================
template <class L, int N, int G>
inline void gather_one(double xp, double yp, double zp, double F[6] /*Ex,Ey,Ez,Bx,By,Bz*/,
                       const W* A /*6 views, same order*/, const int (*stag)[3],
                       const double dinv[3], const double xyzmin[3], const int lo[3]) {
    constexpr int M = N - G;  // galerkin-lowered order
    const double pos[3] = {(xp - xyzmin[0]) * dinv[0], (yp - xyzmin[1]) * dinv[1],
                           (zp - xyzmin[2]) * dinv[2]};
    // [dim][0 = node full, 1 = cell full, 2 = node lowered, 3 = cell lowered]; like the reference
    // (FieldGather.H:98-109,134-145,170-181) only the combinations some component needs are computed
    double s[3][4][N + 1];
    int j0[3][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}, {0, 0, 0, 0}};
    bool need[3][4] = {{false, false, false, false}, {false, false, false, false}, {false, false, false, false}};
    int sel[6][3], cnt[6][3];
    for (int c = 0; c < 6; ++c)
        for (int d = 0; d < 3; ++d) {
            // lowered order along: E_c its own direction; B_c the two transverse directions
            const bool lowered = (c < 3) ? (d == c) : (d != (c - 3));
            sel[c][d] = (lowered ? 2 : 0) + (stag[c][d] == 1 ? 0 : 1);
            cnt[c][d] = lowered ? M : N;
            need[d][sel[c][d]] = true;
        }
    for (int d = 0; d < 3; ++d) {
        if (need[d][0]) j0[d][0] = L::template shape<N>(s[d][0], pos[d]);
        if (need[d][1]) j0[d][1] = L::template shape<N>(s[d][1], pos[d] - 0.5);
        if (need[d][2]) j0[d][2] = L::template shape<M>(s[d][2], pos[d]);
        if (need[d][3]) j0[d][3] = L::template shape<M>(s[d][3], pos[d] - 0.5);
    }
    const int order_of_comp[6] = {0, 1, 2, 5, 4, 3};  // Ex,Ey,Ez,Bz,By,Bx (:368-422)
    for (int oc = 0; oc < 6; ++oc) {
        const int c = order_of_comp[oc];
        const int tx = sel[c][0], ty = sel[c][1], tz = sel[c][2];
        const int nx = cnt[c][0], ny = cnt[c][1], nz = cnt[c][2];
        const double* sx = s[0][tx]; const double* sy = s[1][ty]; const double* sz = s[2][tz];
        const double* base = &A[c](lo[0] + j0[0][tx], lo[1] + j0[1][ty], lo[2] + j0[2][tz]);
        const long sj = A[c].sj, sk = A[c].sk;
        double acc = F[c];
        for (int iz = 0; iz <= nz; ++iz)
            for (int iy = 0; iy <= ny; ++iy) {
                const double* row = base + iy * sj + iz * sk;
                for (int ix = 0; ix <= nx; ++ix)
                    acc += sx[ix] * sy[iy] * sz[iz] * row[ix];
            }
        F[c] = acc;
    }
}

// PhysicalParticleContainer::PushPX (Particles/PhysicalParticleContainer.cpp:2693-2749) and
// PushP (:2454-2510, push_position = 0).  doParticleMomentumPush: Pusher/PushSelector.H:88-102.
template <class L, int N, int G>
void gather_push_t(const pic_soa& P, long offset, long np, const pic_fab E[3], const pic_fab B[3],
                   const double dinv[3], const double xyzmin[3], const int lo[3], double q,
                   double m, double dt, int pusher, int push_position) {
    const W A[6] = {W(E[0]), W(E[1]), W(E[2]), W(B[0]), W(B[1]), W(B[2])};
    int stag[6][3];
    for (int c = 0; c < 3; ++c)
        for (int d = 0; d < 3; ++d) { stag[c][d] = E[c].stag[d]; stag[3 + c][d] = B[c].stag[d]; }
#pragma omp parallel for schedule(static)
    for (long ip = offset; ip < offset + np; ++ip) {
        double xp = P.x[ip], yp = P.y[ip], zp = P.z[ip];
        double F[6] = {0, 0, 0, 0, 0, 0};  // m_E/B_external_particle = 0 (:2589-2594)
        gather_one<L, N, G>(xp, yp, zp, F, A, stag, dinv, xyzmin, lo);
        double ux = P.ux[ip], uy = P.uy[ip], uz = P.uz[ip];
        if (pusher == PIC_PUSHER_BORIS) L::boris(ux, uy, uz, F[0], F[1], F[2], F[3], F[4], F[5], q, m, dt);
        else if (pusher == PIC_PUSHER_VAY) L::vay(ux, uy, uz, F[0], F[1], F[2], F[3], F[4], F[5], q, m, dt);
        else L::higuera_cary(ux, uy, uz, F[0], F[1], F[2], F[3], F[4], F[5], q, m, dt);
        P.ux[ip] = ux; P.uy[ip] = uy; P.uz[ip] = uz;
        if (push_position) {
            L::update_position(xp, yp, zp, ux, uy, uz, dt);
            P.x[ip] = xp; P.y[ip] = yp; P.z[ip] = zp;
        }
    }
}

template <class L>
int gather_push(const pic_soa& P, long offset, long np, const pic_fab E[3], const pic_fab B[3],
                const double dinv[3], const double xyzmin[3], const int lo[3], double q, double m,
                double dt, int nox, int galerkin, int pusher, int push_position) {
    // runtime -> compile-time dispatch as FieldGather.H:1590-1664
#define ORC_GP(N, G) gather_push_t<L, N, G>(P, offset, np, E, B, dinv, xyzmin, lo, q, m, dt, pusher, push_position)
    if (nox == 1 && galerkin) ORC_GP(1, 1);
    else if (nox == 1) ORC_GP(1, 0);
    else if (nox == 2 && galerkin) ORC_GP(2, 1);
    else if (nox == 2) ORC_GP(2, 0);
    else if (nox == 3 && galerkin) ORC_GP(3, 1);
    else if (nox == 3) ORC_GP(3, 0);
    else if (nox == 4 && galerkin) ORC_GP(4, 1);
    else if (nox == 4) ORC_GP(4, 0);
    else return 1;
#undef ORC_GP
    return 0;
}

// ============================================================================================
// Esirkepov deposition of one particle into jx/jy/jz views.
// doEsirkepovDepositionShapeN<N> (Particles/Deposition/CurrentDeposition.H:683-906, 3D :792-824).
// ============================================================================================
template <class L, int N>
inline void deposit_one(double xp, double yp, double zp, double wp, double uxp, double uyp,
                        double uzp, const W& Jx, const W& Jy, const W& Jz, double dt,
                        double relative_time, const double dinv[3], const double xyzmin[3],
                        const int lo[3], double q) {
    const double invdtd[3] = {(1.0 / dt) * dinv[1] * dinv[2], (1.0 / dt) * dinv[0] * dinv[2],
                              (1.0 / dt) * dinv[0] * dinv[1]};                    // :671-673
    constexpr double clightsq = 1.0 / (C_LIGHT * C_LIGHT);                         // :675
    constexpr double one_third = 1.0 / 3.0, one_sixth = 1.0 / 6.0;
    const double gaminv = 1.0 / std::sqrt(1.0 + uxp * uxp * clightsq + uyp * uyp * clightsq
                                          + uzp * uzp * clightsq);                 // :687-689
    const double wq = q * wp;                                                      // :691
    // positions in grid units, double (:725-736)
    const double x_new = (xp - xyzmin[0] + (relative_time + 0.5 * dt) * uxp * gaminv) * dinv[0];
    const double x_old = x_new - dt * dinv[0] * uxp * gaminv;
    const double y_new = (yp - xyzmin[1] + (relative_time + 0.5 * dt) * uyp * gaminv) * dinv[1];
    const double y_old = y_new - dt * dinv[1] * uyp * gaminv;
    const double z_new = (zp - xyzmin[2] + (relative_time + 0.5 * dt) * uzp * gaminv) * dinv[2];
    const double z_old = z_new - dt * dinv[2] * uzp * gaminv;
    double sx_new[N + 3] = {0.}, sx_old[N + 3] = {0.};                             // :759-773
    double sy_new[N + 3] = {0.}, sy_old[N + 3] = {0.};
    double sz_new[N + 3] = {0.}, sz_old[N + 3] = {0.};
    const int i_new = L::template shape<N>(sx_new + 1, x_new);
    const int i_old = L::template shifted_shape<N>(sx_old, x_old, i_new);
    const int j_new = L::template shape<N>(sy_new + 1, y_new);
    const int j_old = L::template shifted_shape<N>(sy_old, y_old, j_new);
    const int k_new = L::template shape<N>(sz_new + 1, z_new);
    const int k_old = L::template shifted_shape<N>(sz_old, z_old, k_new);
    int dil = 1, diu = 1, djl = 1, dju = 1, dkl = 1, dku = 1;                      // :777-788
    if (i_old < i_new) dil = 0;
    if (i_old > i_new) diu = 0;
    if (j_old < j_new) djl = 0;
    if (j_old > j_new) dju = 0;
    if (k_old < k_new) dkl = 0;
    if (k_old > k_new) dku = 0;
    const int bi = lo[0] + i_new - 1, bj = lo[1] + j_new - 1, bk = lo[2] + k_new - 1;
    for (int k = dkl; k <= N + 2 - dku; ++k)                                       // :792-802
        for (int j = djl; j <= N + 2 - dju; ++j) {
            double sdxi = 0.0;
            for (int i = dil; i <= N + 1 - diu; ++i) {
                sdxi += wq * invdtd[0] * (sx_old[i] - sx_new[i]) * (
                    one_third * (sy_new[j] * sz_new[k] + sy_old[j] * sz_old[k])
                    + one_sixth * (sy_new[j] * sz_old[k] + sy_old[j] * sz_new[k]));
                Jx(bi + i, bj + j, bk + k) += sdxi;
            }
        }
    for (int k = dkl; k <= N + 2 - dku; ++k)                                       // :803-813
        for (int i = dil; i <= N + 2 - diu; ++i) {
            double sdyj = 0.0;
            for (int j = djl; j <= N + 1 - dju; ++j) {
                sdyj += wq * invdtd[1] * (sy_old[j] - sy_new[j]) * (
                    one_third * (sx_new[i] * sz_new[k] + sx_old[i] * sz_old[k])
                    + one_sixth * (sx_new[i] * sz_old[k] + sx_old[i] * sz_new[k]));
                Jy(bi + i, bj + j, bk + k) += sdyj;
            }
        }
    for (int j = djl; j <= N + 2 - dju; ++j)                                       // :814-824
        for (int i = dil; i <= N + 2 - diu; ++i) {
            double sdzk = 0.0;
            for (int k = dkl; k <= N + 1 - dku; ++k) {
                sdzk += wq * invdtd[2] * (sz_old[k] - sz_new[k]) * (
                    one_third * (sx_new[i] * sy_new[j] + sx_old[i] * sy_old[j])
                    + one_sixth * (sx_new[i] * sy_old[j] + sx_old[i] * sy_new[j]));
                Jz(bi + i, bj + j, bk + k) += sdzk;
            }
        }
}

// WarpXParticleContainer::DepositCurrent, CPU strategy (Particles/WarpXParticleContainer.cpp:451-470,
// 819-826): each OpenMP thread deposits its particles into a thread-local array, then adds it to
// the global J under a lock.  Here the thread-local array covers the bounding box of the cells its
// (contiguous) particle chunk touches.
template <class L, int N>
void deposit_t(const pic_soa& P, long offset, long np, const pic_fab J[3], const double dinv[3],
               const double xyzmin[3], const int lo[3], double q, double dt, double relative_time) {
    int nthreads = 1;
#ifdef _OPENMP
    nthreads = omp_get_max_threads();
#endif
    if (nthreads == 1 || np < 4096) {
        W Jx(J[0]), Jy(J[1]), Jz(J[2]);
        for (long ip = offset; ip < offset + np; ++ip)
            deposit_one<L, N>(P.x[ip], P.y[ip], P.z[ip], P.w[ip], P.ux[ip], P.uy[ip], P.uz[ip],
                              Jx, Jy, Jz, dt, relative_time, dinv, xyzmin, lo, q);
        return;
    }
    // thread-local tiles (WarpXParticleContainer.cpp:455-470) ...
    std::vector<pic_fab> tiles((size_t)3 * nthreads);
    std::vector<std::vector<double>> bufs((size_t)3 * nthreads);
    std::vector<char> used((size_t)nthreads, 0);
#pragma omp parallel num_threads(nthreads)
    {
#ifdef _OPENMP
        const int t = omp_get_thread_num();
#else
        const int t = 0;
#endif
        const long b = offset + np * t / nthreads, e = offset + np * (t + 1) / nthreads;
        if (e > b) {
            // bounding box (grid units relative to lo) of this chunk, with the stencil margin
            double mn[3] = {1e300, 1e300, 1e300}, mx[3] = {-1e300, -1e300, -1e300};
            for (long ip = b; ip < e; ++ip) {
                const double r[3] = {(P.x[ip] - xyzmin[0]) * dinv[0], (P.y[ip] - xyzmin[1]) * dinv[1],
                                     (P.z[ip] - xyzmin[2]) * dinv[2]};
                for (int d = 0; d < 3; ++d) { mn[d] = std::min(mn[d], r[d]); mx[d] = std::max(mx[d], r[d]); }
            }
            pic_fab* T = &tiles[(size_t)3 * t];
            for (int c = 0; c < 3; ++c) {
                T[c] = J[c];
                for (int d = 0; d < 3; ++d) {
                    // a particle moves < 1 cell (CFL) and its stencil spans N+3 slots from i_new-1
                    T[c].lo[d] = std::max(J[c].lo[d], lo[d] + (int)std::floor(mn[d]) - (N + 3));
                    T[c].hi[d] = std::min(J[c].hi[d], lo[d] + (int)std::floor(mx[d]) + (N + 3));
                }
                bufs[(size_t)3 * t + c].assign((size_t)fab_size(T[c]), 0.0);
                T[c].p = bufs[(size_t)3 * t + c].data();
            }
            W Jx(T[0]), Jy(T[1]), Jz(T[2]);
            for (long ip = b; ip < e; ++ip)
                deposit_one<L, N>(P.x[ip], P.y[ip], P.z[ip], P.w[ip], P.ux[ip], P.uy[ip],
                                  P.uz[ip], Jx, Jy, Jz, dt, relative_time, dinv, xyzmin, lo, q);
            used[t] = 1;
        }
#pragma omp barrier
        // ... then added to the global J (the reference's lockAdd, :819-826), here k-plane by k-plane
        // so that the reduction scales with the thread count
        for (int c = 0; c < 3; ++c) {
            W G(J[c]);
#pragma omp for schedule(static)
            for (int k = J[c].lo[2]; k <= J[c].hi[2]; ++k)
                for (int tt = 0; tt < nthreads; ++tt) {
                    if (!used[tt]) continue;
                    const pic_fab& T = tiles[(size_t)3 * tt + c];
                    if (k < T.lo[2] || k > T.hi[2]) continue;
                    W S(T);
                    for (int j = T.lo[1]; j <= T.hi[1]; ++j)
                        for (int i = T.lo[0]; i <= T.hi[0]; ++i) G(i, j, k) += S(i, j, k);
                }
        }
    }
}

template <class L>
int deposit(const pic_soa& P, long offset, long np, const pic_fab J[3], const double dinv[3],
            const double xyzmin[3], const int lo[3], double q, double dt, double relative_time,
            int nox) {
    if (nox == 1) deposit_t<L, 1>(P, offset, np, J, dinv, xyzmin, lo, q, dt, relative_time);
    else if (nox == 2) deposit_t<L, 2>(P, offset, np, J, dinv, xyzmin, lo, q, dt, relative_time);
    else if (nox == 3) deposit_t<L, 3>(P, offset, np, J, dinv, xyzmin, lo, q, dt, relative_time);
    else if (nox == 4) deposit_t<L, 4>(P, offset, np, J, dinv, xyzmin, lo, q, dt, relative_time);
    else return 1;
    return 0;
}

// ============================================================================================
// Charge deposition (diagnostic: the `rho` of the golden checksum files).
// doChargeDepositionShapeN<N> (Particles/Deposition/ChargeDeposition.H:37-157, 3D :146-155) into a
// nodal rho: wq = q w / dV, weights = Compute_shape_factor at (x - xyzmin) * dinv.
// ============================================================================================
template <class L, int N>
void deposit_charge_t(const pic_soa& P, const pic_fab& rho, const double dinv[3], const double xyzmin[3],
                      const int lo[3], double q) {
    W R(rho);
    const double invvol = dinv[0] * dinv[1] * dinv[2];
    for (long ip = 0; ip < P.np; ++ip) {
        const double wq = q * P.w[ip] * invvol;
        double sx[N + 1] = {0.}, sy[N + 1] = {0.}, sz[N + 1] = {0.};
        const double x = (P.x[ip] - xyzmin[0]) * dinv[0], y = (P.y[ip] - xyzmin[1]) * dinv[1],
                     z = (P.z[ip] - xyzmin[2]) * dinv[2];
        const int i = L::template shape<N>(sx, rho.stag[0] ? x : x - 0.5);
        const int j = L::template shape<N>(sy, rho.stag[1] ? y : y - 0.5);
        const int k = L::template shape<N>(sz, rho.stag[2] ? z : z - 0.5);
        for (int iz = 0; iz <= N; ++iz)
            for (int iy = 0; iy <= N; ++iy)
                for (int ix = 0; ix <= N; ++ix)
                    R(lo[0] + i + ix, lo[1] + j + iy, lo[2] + k + iz) += sx[ix] * sy[iy] * sz[iz] * wq;
    }
}
template <class L>
int deposit_charge(const pic_soa& P, const pic_fab& rho, const double dinv[3], const double xyzmin[3],
                   const int lo[3], double q, int nox) {
    if (nox == 1) deposit_charge_t<L, 1>(P, rho, dinv, xyzmin, lo, q);
    else if (nox == 2) deposit_charge_t<L, 2>(P, rho, dinv, xyzmin, lo, q);
    else if (nox == 3) deposit_charge_t<L, 3>(P, rho, dinv, xyzmin, lo, q);
    else if (nox == 4) deposit_charge_t<L, 4>(P, rho, dinv, xyzmin, lo, q);
    else return 1;
    return 0;
}

// ============================================================================================
// Guard cells on a set of boxes tiling a periodic domain (semantics of AMReX FabArray
// FillBoundary / SumBoundary, AMReX 24.10 @62c2a81 -- un-vendored dependency; call sites
// ablastr/utils/Communication.cpp:71-115 and :148-175).
//
// A "location" is a global index wrapped into [0, n_cell) per periodic dimension (nodal index N
// is the periodic duplicate of index 0).  Brute force: correctness oracle, not fast.
// ============================================================================================
inline int wrap(int i, int n) { int r = i % n; return r < 0 ? r + n : r; }

// Location map of one dimension: periodic -> index wrapped into [0, n_cell); non-periodic -> the
// index itself, offset so that guard points beyond the domain have their own (unshared) location.
struct LocMap {
    int n[3], per[3], off[3], size[3];
    LocMap(const pic_geom& g, const pic_fab* fabs, int nfab) {
        for (int d = 0; d < 3; ++d) {
            n[d] = g.n_cell[d]; per[d] = g.periodic[d];
            int mg = 0;
            for (int b = 0; b < nfab; ++b) mg = std::max(mg, fabs[b].ng[d]);
            off[d] = per[d] ? 0 : mg;
            size[d] = per[d] ? n[d] : n[d] + 1 + 2 * mg;
        }
    }
    int at(int i, int d) const { return per[d] ? wrap(i, n[d]) : i + off[d]; }
    size_t idx(int i, int j, int k) const {
        return at(i, 0) + (size_t)size[0] * (at(j, 1) + (size_t)size[1] * at(k, 2));
    }
    size_t total() const { return (size_t)size[0] * size[1] * size[2]; }
};

// FillBoundary(ng): every guard point within ng of the valid region receives the value of a
// valid point at the same location (any box; duplicates hold equal values by construction).
// Guard points beyond a non-periodic domain face have no valid image and are left untouched
// (AMReX FabArray::FillBoundary with a Periodicity that is off in that direction).
inline void fill_boundary(const pic_fab* fabs, int nfab, const int ng[3], const pic_geom& g) {
    const LocMap M(g, fabs, nfab);
    const bool all_periodic = g.periodic[0] && g.periodic[1] && g.periodic[2];
    // canonical value of a location = the valid point of the box that OWNS it (a box owns the
    // points of its cells, i.e. its valid points minus the upper nodal layer; along a non-periodic
    // direction the upper nodal layer is a location of its own and is owned too); within one box
    // every location is written exactly once, so the fill is race-free.
    std::vector<double> canon(M.total(), 0.0);
    std::vector<char> have(all_periodic ? 0 : M.total(), 0);
    for (int b = 0; b < nfab; ++b) {
        const pic_fab& f = fabs[b]; W v(f);
        const int h0 = vhi(f, 0) - (g.periodic[0] ? f.stag[0] : 0), h1 = vhi(f, 1) - (g.periodic[1] ? f.stag[1] : 0),
                  h2 = vhi(f, 2) - (g.periodic[2] ? f.stag[2] : 0);
#pragma omp parallel for schedule(static)
        for (int k = vlo(f, 2); k <= h2; ++k)
            for (int j = vlo(f, 1); j <= h1; ++j)
                for (int i = vlo(f, 0); i <= h0; ++i) {
                    const size_t c = M.idx(i, j, k);
                    canon[c] = v(i, j, k);
                    if (!all_periodic) have[c] = 1;
                }
    }
    for (int b = 0; b < nfab; ++b) {
        const pic_fab& f = fabs[b]; W v(f);
#pragma omp parallel for schedule(static)
        for (int k = vlo(f, 2) - ng[2]; k <= vhi(f, 2) + ng[2]; ++k)
            for (int j = vlo(f, 1) - ng[1]; j <= vhi(f, 1) + ng[1]; ++j)
                for (int i = vlo(f, 0) - ng[0]; i <= vhi(f, 0) + ng[0]; ++i) {
                    const bool valid = i >= vlo(f, 0) && i <= vhi(f, 0) && j >= vlo(f, 1) &&
                                       j <= vhi(f, 1) && k >= vlo(f, 2) && k <= vhi(f, 2);
                    if (valid) continue;
                    const size_t c = M.idx(i, j, k);
                    if (!all_periodic && !have[c]) continue;
                    v(i, j, k) = canon[c];
                }
    }
}

// SumBoundary(src_ng, dst_ng): every point (valid + dst_ng guards) receives the sum over ALL
// copies (valid + src_ng guards of every box) at the same location (AMReX FabArray::SumBoundary:
// copy to a temporary, zero valid + dst_ng, ParallelAdd the temporary back).  Along a non-periodic
// direction a guard point beyond the domain face only has itself as a copy.
inline void sum_boundary(const pic_fab* fabs, int nfab, const int src_ng[3], const int dst_ng[3],
                         const pic_geom& g) {
    const LocMap M(g, fabs, nfab);
    const int n2 = g.n_cell[2];
    std::vector<double> canon(M.total(), 0.0);
    for (int b = 0; b < nfab; ++b) {
        const pic_fab& f = fabs[b]; W v(f);
        // planes k that wrap onto each other (k, k +- n2) are visited in separate sweeps, so each
        // sweep can run in parallel over k without atomics
        const int kbeg = vlo(f, 2) - src_ng[2], kend = vhi(f, 2) + src_ng[2];
        const int first_period = g.periodic[2] ? (int)std::floor((double)kbeg / n2) : 0;
        const int last_period = g.periodic[2] ? (int)std::floor((double)kend / n2) : 0;
        for (int per = first_period; per <= last_period; ++per) {
            const int ka = g.periodic[2] ? std::max(kbeg, per * n2) : kbeg;
            const int kb = g.periodic[2] ? std::min(kend, per * n2 + n2 - 1) : kend;
#pragma omp parallel for schedule(static)
            for (int k = ka; k <= kb; ++k)
                for (int j = vlo(f, 1) - src_ng[1]; j <= vhi(f, 1) + src_ng[1]; ++j)
                    for (int i = vlo(f, 0) - src_ng[0]; i <= vhi(f, 0) + src_ng[0]; ++i)
                        canon[M.idx(i, j, k)] += v(i, j, k);
        }
    }
    for (int b = 0; b < nfab; ++b) {
        const pic_fab& f = fabs[b]; W v(f);
#pragma omp parallel for schedule(static)
        for (int k = vlo(f, 2) - dst_ng[2]; k <= vhi(f, 2) + dst_ng[2]; ++k)
            for (int j = vlo(f, 1) - dst_ng[1]; j <= vhi(f, 1) + dst_ng[1]; ++j)
                for (int i = vlo(f, 0) - dst_ng[0]; i <= vhi(f, 0) + dst_ng[0]; ++i)
                    v(i, j, k) = canon[M.idx(i, j, k)];
    }
}

// ============================================================================================
// Bilinear (binomial) current filter.  Stencil: BilinearFilter.cpp:26-62 (compute_stencil: the
// (1,2,1)/4 kernel convolved npass times, element 0 halved because it is used twice); application:
// Filter::DoFilter, Filter/Filter.cpp:92-133 (3D), over the grown box, source zero-padded outside
// the fab (:103-107).  dst and src must be different arrays (WarpX::ApplyFilterJ filters into a
// temporary and copies back, Parallelization/WarpXComm.cpp:1357-1374).
// ============================================================================================
inline std::vector<double> filter_stencil(int npass) {
    std::vector<double> old_s(1 + npass, 0.0), new_s(1 + npass, 0.0);
    old_s[0] = 1.0;
    int jmax = 1;
    for (int ipass = 1; ipass < npass + 1; ++ipass) {
        new_s[0] = 0.5 * old_s[0];
        if (1 < jmax) new_s[0] += 0.5 * old_s[1];
        for (int j = 1; j < jmax + 1; ++j) {
            double loc = 0.5 * old_s[j];
            loc += 0.25 * old_s[j - 1];
            if (j < jmax) loc += 0.25 * old_s[j + 1];
            new_s[j] = loc;
        }
        old_s = new_s;
        jmax += 1;
    }
    old_s[0] *= 0.5;
    return old_s;
}

inline void apply_filter(const pic_fab& src, const pic_fab& dst, const int npass[3]) {
    const std::vector<double> s0 = filter_stencil(npass[0]), s1 = filter_stencil(npass[1]), s2 = filter_stencil(npass[2]);
    const int l0 = npass[0] + 1, l1 = npass[1] + 1, l2 = npass[2] + 1;      // stencil_length_each_dir
    W S(src), D(dst);
    auto pad = [&](int i, int j, int k) -> double {
        const bool in = i >= src.lo[0] && i <= src.hi[0] && j >= src.lo[1] && j <= src.hi[1] && k >= src.lo[2] && k <= src.hi[2];
        return in ? S(i, j, k) : 0.0;
    };
#pragma omp parallel for schedule(static)
    for (int k = dst.lo[2]; k <= dst.hi[2]; ++k)               // growntilebox: valid + guards
        for (int j = dst.lo[1]; j <= dst.hi[1]; ++j)
            for (int i = dst.lo[0]; i <= dst.hi[0]; ++i) {
                double d = 0.0;
                for (int i2 = 0; i2 < l2; ++i2)
                    for (int i1 = 0; i1 < l1; ++i1)
                        for (int i0 = 0; i0 < l0; ++i0) {
                            const double sss = s0[i0] * s1[i1] * s2[i2];
                            d += sss * (pad(i - i0, j - i1, k - i2) + pad(i + i0, j - i1, k - i2)
                                      + pad(i - i0, j + i1, k - i2) + pad(i + i0, j + i1, k - i2)
                                      + pad(i - i0, j - i1, k + i2) + pad(i + i0, j - i1, k + i2)
                                      + pad(i - i0, j + i1, k + i2) + pad(i + i0, j + i1, k + i2));
                        }
                D(i, j, k) = d;
            }
}

// ---------------------------------------------------------------------------------------------
// Godfrey's NCI corrector (particles.use_fdtd_nci_corr): a 5-point filter along z applied to a copy
// of E and B before the gather.
// NCIGodfreyFilter::ComputeStencils (Filter/NCIGodfreyFilter.cpp:49-120): the four coefficients are
// interpolated linearly in c dt / dz between two lines of the reference's tables
// (Utils/NCIGodfreyTables.H, tab_length = 101 lines, tab_width = 4; fitted data the caller supplies),
// then combined into the stencil; coefficient 0 is halved because of the way DoFilter sums.
inline int nci_table_index(double cdtodz, int tab_length) {
    int index = static_cast<int>(tab_length * cdtodz);                            // :61-63
    index = std::min(index, tab_length - 2);
    index = std::max(index, 0);
    return index;
}
inline void nci_godfrey_stencil(const double* row_lo /*4: table[index]*/, const double* row_hi /*4: table[index+1]*/,
                                int index, int tab_length, double cdtodz, double* stencil_z /*5*/) {
    const double weight_right = cdtodz - double(index) / double(tab_length);      // :64
    double prestencil[4];
    for (int i = 0; i < 4; ++i) prestencil[i] = (1.0 - weight_right) * row_lo[i] + weight_right * row_hi[i];   // :69-104
    stencil_z[0] =  (256 + 128 * prestencil[0] + 96 * prestencil[1] + 80 * prestencil[2] + 70 * prestencil[3]) / 256;   // :107-111
    stencil_z[1] = -(       64 * prestencil[0] + 64 * prestencil[1] + 60 * prestencil[2] + 56 * prestencil[3]) / 256;
    stencil_z[2] =  (                            16 * prestencil[1] + 24 * prestencil[2] + 28 * prestencil[3]) / 256;
    stencil_z[3] = -(                                                  4 * prestencil[2] +  8 * prestencil[3]) / 256;
    stencil_z[4] =  (                                                                       1 * prestencil[3]) / 256;
    stencil_z[0] /= 2.0;                                                          // :125-129
}

// Filter::ApplyStencil(FArrayBox) -> DoFilter (Filter/Filter.cpp:78-133) with the NCI stencils
// s0 = s1 = {1/2}, s2 = stencil_z (slen = {1,1,5}), over tbx = [tlo, thi] in the index space of the
// component (PhysicalParticleContainer::applyNCIFilter, PhysicalParticleContainer.cpp:2097-2169:
// the tile box grown by the shape order, converted to the component's index type).
inline void apply_nci_filter(const pic_fab& src, const pic_fab& dst, const double* stencil_z, const int tlo[3], const int thi[3]) {
    W S(src), D(dst);
    auto pad = [&](int i, int j, int k) -> double {
        const bool in = i >= src.lo[0] && i <= src.hi[0] && j >= src.lo[1] && j <= src.hi[1] && k >= src.lo[2] && k <= src.hi[2];
        return in ? S(i, j, k) : 0.0;
    };
    const double s0 = 1.0 / 2.0, s1 = 1.0 / 2.0;
#pragma omp parallel for schedule(static)
    for (int k = tlo[2]; k <= thi[2]; ++k)
        for (int j = tlo[1]; j <= thi[1]; ++j)
            for (int i = tlo[0]; i <= thi[0]; ++i) {
                double d = 0.0;
                for (int i2 = 0; i2 < 5; ++i2) {
                    const double sss = s0 * s1 * stencil_z[i2];
                    d += sss * (pad(i, j, k - i2) + pad(i, j, k - i2) + pad(i, j, k - i2) + pad(i, j, k - i2)
                              + pad(i, j, k + i2) + pad(i, j, k + i2) + pad(i, j, k + i2) + pad(i, j, k + i2));
                }
                D(i, j, k) = d;
            }
}

// amrex::enforcePeriodic (AMReX_ParticleUtil.H, AMReX 24.10) as applied by Redistribute
// (WarpXEvolve.cpp:550-559): shift by the domain length until inside, then clamp round-off.
inline void wrap_periodic(const pic_soa& P, const pic_geom& g) {
    double* X[3] = {P.x, P.y, P.z};
    for (int d = 0; d < 3; ++d) {
        if (!g.periodic[d]) continue;
        const double lo = g.prob_lo[d], hi = g.prob_hi[d], len = hi - lo;
        double* x = X[d];
#pragma omp parallel for schedule(static)
        for (long ip = 0; ip < P.np; ++ip) {
            double v = x[ip];
            if (v > hi) {
                while (v > hi) v -= len;
                if (v < lo) v = lo;
            } else if (v < lo) {
                while (v < lo) v += len;
                if (v > hi) v = hi;
            }
            x[ip] = v;
        }
    }
}

// ============================================================================================
// Diagnostics used as parity metrics
// ============================================================================================
// MultiFab::norm2(0, periodicity)^2: sum of squares counting each periodic/nodal duplicate once
// (Diagnostics/ReducedDiags/FieldEnergy.cpp:123-144).
inline double sum_squares_unique(const pic_fab* fabs, int nfab, const pic_geom& g) {
    const LocMap M(g, fabs, nfab);
    std::vector<char> seen(M.total(), 0);
    double s = 0.0;
    for (int b = 0; b < nfab; ++b) {
        const pic_fab& f = fabs[b]; W v(f);
        for (int k = vlo(f, 2); k <= vhi(f, 2); ++k)
            for (int j = vlo(f, 1); j <= vhi(f, 1); ++j)
                for (int i = vlo(f, 0); i <= vhi(f, 0); ++i) {
                    const size_t c = M.idx(i, j, k);
                    if (seen[c]) continue;
                    seen[c] = 1;
                    s += v(i, j, k) * v(i, j, k);
                }
    }
    return s;
}

// ParticleEnergy (Diagnostics/ReducedDiags/ParticleEnergy.cpp:86-170) with Algorithms::KineticEnergy
// (Particles/Algorithms/KineticEnergy.H:31-46): out = {sum w * m u^2 / (1 + gamma), sum w}.
inline void particle_energy(const pic_soa& P, double mass, double out[2]) {
    constexpr double inv_c2 = 1.0 / (C_LIGHT * C_LIGHT);
    double e = 0.0, ws = 0.0;
    for (long ip = 0; ip < P.np; ++ip) {
        const double u2 = P.ux[ip] * P.ux[ip] + P.uy[ip] * P.uy[ip] + P.uz[ip] * P.uz[ip];
        const double gamma = std::sqrt(1.0 + u2 * inv_c2);
        e += P.w[ip] * (1.0 / (1.0 + gamma) * mass * u2);
        ws += P.w[ip];
    }
    out[0] = e; out[1] = ws;
}

// Sum over the N^3 cells of |cell-centred average| -- what Regression/Checksum/checksum.py:110-116
// computes from a plotfile whose fields were averaged to cell centres by
// ablastr/coarsen/sample.H:69-103 (cr = 1: for each nodal direction the two neighbouring nodes
// are averaged; the loop nest there is ii outer .. kk inner with weight 1/(npx*npy*npz)).
inline double checksum_cell_centered(const pic_fab& f, const int box_lo[3], const int box_hi[3]) {
    W v(f);
    const int np0 = 1 + f.stag[0], np1 = 1 + f.stag[1], np2 = 1 + f.stag[2];
    const double wx = 1.0 / double(np0), wy = 1.0 / double(np1), wz = 1.0 / double(np2);
    double s = 0.0;
    for (int k = box_lo[2]; k <= box_hi[2]; ++k)
        for (int j = box_lo[1]; j <= box_hi[1]; ++j)
            for (int i = box_lo[0]; i <= box_hi[0]; ++i) {
                double c = 0.0;
                for (int kk = 0; kk < np2; ++kk)
                    for (int jj = 0; jj < np1; ++jj)
                        for (int ii = 0; ii < np0; ++ii) c += wx * wy * wz * v(i + ii, j + jj, k + kk);
                s += std::fabs(c);
            }
    return s;
}

}  // namespace orc
#endif
