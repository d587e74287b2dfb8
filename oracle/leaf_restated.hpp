// TEST INFRASTRUCTURE -- CPU oracle, leaf arithmetic restated by hand.
//
// Each function restates one leaf routine of the reference (paths relative to
// Source/ of ECP-WarpX/WarpX) with the SAME floating-point evaluation order, so that a build with
// -ffp-contract=off is bit-identical to the reference headers compiled verbatim through
// oracle/amrex_shim (see leaf_reference.hpp and tests/test_oracle_vs_reference_leaves.py).
// Nothing outside tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs may use this.
#ifndef PIC_ORACLE_LEAF_RESTATED_HPP_
#define PIC_ORACLE_LEAF_RESTATED_HPP_

#include <algorithm>
#include <cmath>
#include "../include/pic_b200.h"

namespace orc {

// CODATA-2018 values, ablastr/constant.H:44-54.
namespace si {
constexpr double c = 299792458.0;
constexpr double ep0 = 8.8541878128e-12;
constexpr double mu0 = 1.25663706212e-06;
constexpr double q_e = 1.602176634e-19;
constexpr double m_e = 9.1093837015e-31;
constexpr double m_p = 1.67262192369e-27;
}

// Fortran-ordered view with arbitrary lower bound == amrex::Array4 indexing.
struct View {
    double* p; int lo0, lo1, lo2; long sj, sk;
    View() : p(nullptr), lo0(0), lo1(0), lo2(0), sj(0), sk(0) {}
    explicit View(const pic_fab& f)
        : p(f.p), lo0(f.lo[0]), lo1(f.lo[1]), lo2(f.lo[2]),
          sj(f.hi[0] - f.lo[0] + 1), sk(sj * (long)(f.hi[1] - f.lo[1] + 1)) {}
    double& operator()(int i, int j, int k) const {
        return p[(i - lo0) + (j - lo1) * sj + (k - lo2) * sk];
    }
};

struct LeafRestated {
    static constexpr const char* name = "restated";
    using Arr = View;
    static Arr arr(const pic_fab& f) { return View(f); }

    // ---- Particles/ShapeFactors.H:27-84 (Compute_shape_factor), orders 0..4 -------------
    // B-spline weights around xmid (grid units); returns leftmost index touched.
    template <int N> static int shape(double* s, double xmid) {
        if constexpr (N == 0) {
            const int j = static_cast<int>(xmid + 0.5);
            s[0] = 1.0;
            return j;
        } else if constexpr (N == 1) {
            const int j = static_cast<int>(xmid);          // truncation, as the reference
            const double d = xmid - double(j);
            s[0] = 1.0 - d;
            s[1] = d;
            return j;
        } else if constexpr (N == 2) {
            const int j = static_cast<int>(xmid + 0.5);
            const double d = xmid - double(j);
            const double a = 0.5 - d, b = 0.5 + d;
            s[0] = 0.5 * a * a;
            s[1] = 0.75 - d * d;
            s[2] = 0.5 * b * b;
            return j - 1;
        } else if constexpr (N == 3) {
            const int j = static_cast<int>(xmid);
            const double d = xmid - double(j);
            const double e = 1.0 - d;
            const double sixth = 1.0 / 6.0, twothird = 2.0 / 3.0;
            s[0] = sixth * e * e * e;
            s[1] = twothird - d * d * (1.0 - d / 2.0);
            s[2] = twothird - e * e * (1.0 - 0.5 * e);
            s[3] = sixth * d * d * d;
            return j - 1;
        } else {
            static_assert(N == 4, "orders 0..4");
            const int j = static_cast<int>(xmid + 0.5);
            const double d = xmid - double(j);
            const double a = 0.5 - d, b = 0.5 + d;
            const double t = 1.0 / 24.0;
            s[0] = t * a * a * a * a;
            s[1] = t * (4.75 - 11.0 * d + 4.0 * d * d * (1.5 + d - d * d));
            s[2] = t * (14.375 + 6.0 * d * d * (d * d - 2.5));
            s[3] = t * (4.75 + 11.0 * d + 4.0 * d * d * (1.5 - d - d * d));
            s[4] = t * b * b * b * b;
            return j - 2;
        }
    }

    // ---- Particles/ShapeFactors.H:93-156 (Compute_shifted_shape_factor) -----------------
    // Weights of the OLD position written into an (N+3)-slot array whose slot 1 is the leftmost
    // point of the NEW position's stencil.  Orders 0/1 use floor, 2..4 use truncation (:104,110).
    template <int N> static int shifted_shape(double* s, double x_old, int i_new) {
        if constexpr (N == 0) {
            const int i = static_cast<int>(std::floor(x_old + 0.5));
            s[1 + (i - i_new)] = 1.0;
            return i;
        } else if constexpr (N == 1) {
            const int i = static_cast<int>(std::floor(x_old));
            const int sh = i - i_new;
            const double d = x_old - double(i);
            s[1 + sh] = 1.0 - d;
            s[2 + sh] = d;
            return i;
        } else if constexpr (N == 2) {
            const int i = static_cast<int>(x_old + 0.5);
            const int sh = i - (i_new + 1);
            const double d = x_old - double(i);
            const double a = 0.5 - d, b = 0.5 + d;
            s[1 + sh] = 0.5 * a * a;
            s[2 + sh] = 0.75 - d * d;
            s[3 + sh] = 0.5 * b * b;
            return i - 1;
        } else if constexpr (N == 3) {
            const int i = static_cast<int>(x_old);
            const int sh = i - (i_new + 1);
            const double d = x_old - double(i);
            const double e = 1.0 - d;
            const double sixth = 1.0 / 6.0, twothird = 2.0 / 3.0;
            s[1 + sh] = sixth * e * e * e;
            s[2 + sh] = twothird - d * d * (1.0 - d / 2.0);
            s[3 + sh] = twothird - e * e * (1.0 - 0.5 * e);
            s[4 + sh] = sixth * d * d * d;
            return i - 1;
        } else {
            static_assert(N == 4, "orders 0..4");
            const int i = static_cast<int>(x_old + 0.5);
            const int sh = i - (i_new + 2);
            const double d = x_old - double(i);
            const double a = 0.5 - d, b = 0.5 + d;
            const double t = 1.0 / 24.0;
            s[1 + sh] = t * a * a * a * a;
            s[2 + sh] = t * (4.75 - 11.0 * d + 4.0 * d * d * (1.5 + d - d * d));
            s[3 + sh] = t * (14.375 + 6.0 * d * d * (d * d - 2.5));
            s[4 + sh] = t * (4.75 + 11.0 * d + 4.0 * d * d * (1.5 - d - d * d));
            s[5 + sh] = t * b * b * b * b;
            return i - 2;
        }
    }

    // ---- Particles/Pusher/UpdateMomentumBoris.H:15-53 -----------------------------------
    static void boris(double& ux, double& uy, double& uz, double Ex, double Ey, double Ez,
                      double Bx, double By, double Bz, double q, double m, double dt) {
        const double ec = 0.5 * q * dt / m;
        ux += ec * Ex; uy += ec * Ey; uz += ec * Ez;                       // half E kick
        constexpr double ic2 = 1.0 / (si::c * si::c);
        const double ig = 1.0 / std::sqrt(1.0 + (ux * ux + uy * uy + uz * uz) * ic2);
        const double tx = ec * ig * Bx, ty = ec * ig * By, tz = ec * ig * Bz;  // rotation vector
        const double tsqi = 2.0 / (1.0 + tx * tx + ty * ty + tz * tz);
        const double sx = tx * tsqi, sy = ty * tsqi, sz = tz * tsqi;
        const double px = ux + uy * tz - uz * ty;
        const double py = uy + uz * tx - ux * tz;
        const double pz = uz + ux * ty - uy * tx;
        ux += py * sz - pz * sy;
        uy += pz * sx - px * sz;
        uz += px * sy - py * sx;
        ux += ec * Ex; uy += ec * Ey; uz += ec * Ez;                       // half E kick
    }

    // ---- Particles/Pusher/UpdateMomentumVay.H:19-62 -------------------------------------
    static void vay(double& ux, double& uy, double& uz, double Ex, double Ey, double Ez,
                    double Bx, double By, double Bz, double q, double m, double dt) {
        const double ec = q * dt / m;
        const double bc = 0.5 * q * dt / m;
        constexpr double ic = 1.0 / si::c;
        constexpr double ic2 = 1.0 / (si::c * si::c);
        const double ig = 1.0 / std::sqrt(1.0 + (ux * ux + uy * uy + uz * uz) * ic2);
        const double ax = bc * Bx, ay = bc * By, az = bc * Bz;             // tau
        const double a2 = ax * ax + ay * ay + az * az;
        const double px = ux + ec * Ex + (uy * az - uz * ay) * ig;         // u'
        const double py = uy + ec * Ey + (uz * ax - ux * az) * ig;
        const double pz = uz + ec * Ez + (ux * ay - uy * ax) * ig;
        const double gp2 = (1.0 + (px * px + py * py + pz * pz) * ic2);
        const double ust = (px * ax + py * ay + pz * az) * ic;
        const double sig = gp2 - a2;
        const double gi2 = 2.0 / (sig + std::sqrt(sig * sig + 4.0 * (a2 + ust * ust)));
        const double bg = bc * std::sqrt(gi2);
        const double tx = bg * Bx, ty = bg * By, tz = bg * Bz;
        const double s = 1.0 / (1.0 + a2 * gi2);
        const double tu = tx * px + ty * py + tz * pz;
        ux = s * (px + tx * tu + py * tz - pz * ty);
        uy = s * (py + ty * tu + pz * tx - px * tz);
        uz = s * (pz + tz * tu + px * ty - py * tx);
    }

    // ---- Particles/Pusher/UpdateMomentumHigueraCary.H:20-67 -----------------------------
    static void higuera_cary(double& ux, double& uy, double& uz, double Ex, double Ey, double Ez,
                             double Bx, double By, double Bz, double q, double m, double dt) {
        const double h = 0.5 * q * dt / m;
        constexpr double ic = 1.0 / si::c;
        constexpr double ic2 = 1.0 / (si::c * si::c);
        const double mx = ux + h * Ex, my = uy + h * Ey, mz = uz + h * Ez;  // u-
        double g = 1.0 + (mx * mx + my * my + mz * mz) * ic2;
        const double bx = h * Bx, by = h * By, bz = h * Bz;
        const double b2 = bx * bx + by * by + bz * bz;
        const double sig = g - b2;
        const double ust = (mx * bx + my * by + mz * bz) * ic;
        g = 1.0 / std::sqrt(0.5 * (sig + std::sqrt(sig * sig + 4.0 * (b2 + ust * ust))));
        const double tx = g * bx, ty = g * by, tz = g * bz;
        const double s = 1.0 / (1.0 + (tx * tx + ty * ty + tz * tz));
        const double mt = mx * tx + my * ty + mz * tz;
        const double px = s * (mx + mt * tx + my * tz - mz * ty);          // u+
        const double py = s * (my + mt * ty + mz * tx - mx * tz);
        const double pz = s * (mz + mt * tz + mx * ty - my * tx);
        ux = px + h * Ex + py * tz - pz * ty;
        uy = py + h * Ey + pz * tx - px * tz;
        uz = pz + h * Ez + px * ty - py * tx;
    }

    // ---- Particles/Pusher/UpdatePosition.H:24-45 ----------------------------------------
    static void update_position(double& x, double& y, double& z, double ux, double uy, double uz,
                                double dt) {
        constexpr double ic2 = 1.0 / (si::c * si::c);
        const double ig = 1.0 / std::sqrt(1.0 + (ux * ux + uy * uy + uz * uz) * ic2);
        x += ux * ig * dt;
        y += uy * ig * dt;
        z += uz * ig * dt;
    }

    // ---- FDTD stencil policies ----------------------------------------------------------
    // Yee : CartesianYeeAlgorithm.H:69-101 (Upward) / :88-101 (Downward), coefs = {1/d}.
    // CKC : CartesianCKCAlgorithm.H:130-299; Upward uses {alpha, beta1, beta2, gamma}
    //       ([1],[2],[3],[4] with the x/y/z specific meaning of :84-101), Downward is Yee-like.
    // d = 0,1,2 selects the derivative direction; (a,b) are the two transverse directions in
    // the order the reference stores their beta coefficients.
    template <int D> static double upward(int algo, const Arr& F, const double* c, int i, int j,
                                          int k) {
        constexpr int di = (D == 0), dj = (D == 1), dk = (D == 2);
        if (algo == PIC_SOLVER_YEE) {
            return c[0] * (F(i + di, j + dj, k + dk) - F(i, j, k));
        }
        // meaning of the beta slots (CartesianCKCAlgorithm.H:84-101):
        //   x: c[2]=beta_xy (y neighbours), c[3]=beta_xz (z)
        //   y: c[2]=beta_yz (z neighbours), c[3]=beta_yx (x)
        //   z: c[2]=beta_zx (x neighbours), c[3]=beta_zy (y)
        const double alpha = c[1], beta1 = c[2], beta2 = c[3], gamma = c[4];
        auto df = [&](int oi, int oj, int ok) {
            return F(i + di + oi, j + dj + oj, k + dk + ok) - F(i + oi, j + oj, k + ok);
        };
        double r;
        if constexpr (D == 0) {
            // x: beta_xy first (+y,-y), then beta_xz (+z,-z); gamma order (+y+z)(-y+z)(+y-z)(-y-z)
            r = alpha * df(0, 0, 0)
              + beta1 * (F(i+1,j+1,k) - F(i,j+1,k) + F(i+1,j-1,k) - F(i,j-1,k))
              + beta2 * (F(i+1,j,k+1) - F(i,j,k+1) + F(i+1,j,k-1) - F(i,j,k-1))
              + gamma * (F(i+1,j+1,k+1) - F(i,j+1,k+1) + F(i+1,j-1,k+1) - F(i,j-1,k+1)
                       + F(i+1,j+1,k-1) - F(i,j+1,k-1) + F(i+1,j-1,k-1) - F(i,j-1,k-1));
        } else if constexpr (D == 1) {
            // y: betayx (= c[3]) term first, then betayz (= c[2])  (:201-208)
            r = alpha * df(0, 0, 0)
              + beta2 * (F(i+1,j+1,k) - F(i+1,j,k) + F(i-1,j+1,k) - F(i-1,j,k))
              + beta1 * (F(i,j+1,k+1) - F(i,j,k+1) + F(i,j+1,k-1) - F(i,j,k-1))
              + gamma * (F(i+1,j+1,k+1) - F(i+1,j,k+1) + F(i-1,j+1,k+1) - F(i-1,j,k+1)
                       + F(i+1,j+1,k-1) - F(i+1,j,k-1) + F(i-1,j+1,k-1) - F(i-1,j,k-1));
        } else {
            // z: betazx (= c[2]) first, then betazy (= c[3])  (:267-275)
            r = alpha * df(0, 0, 0)
              + beta1 * (F(i+1,j,k+1) - F(i+1,j,k) + F(i-1,j,k+1) - F(i-1,j,k))
              + beta2 * (F(i,j+1,k+1) - F(i,j+1,k) + F(i,j-1,k+1) - F(i,j-1,k))
              + gamma * (F(i+1,j+1,k+1) - F(i+1,j+1,k) + F(i-1,j+1,k+1) - F(i-1,j+1,k)
                       + F(i+1,j-1,k+1) - F(i+1,j-1,k) + F(i-1,j-1,k+1) - F(i-1,j-1,k));
        }
        return r;
    }
    template <int D> static double downward(int /*algo*/, const Arr& F, const double* c, int i,
                                            int j, int k) {
        constexpr int di = (D == 0), dj = (D == 1), dk = (D == 2);
        return c[0] * (F(i, j, k) - F(i - di, j - dj, k - dk));
    }

    // ---- stencil coefficients / CFL time step -------------------------------------------
    // Yee: CartesianYeeAlgorithm.H:30-42 and :48-56.  CKC (Cowan 2013): CartesianCKCAlgorithm.H:31-101
    // and :107-118.
    static void stencil_coefs(int algo, const double dx[3], pic_stencil* st) {
        st->algo = algo;
        for (int n = 0; n < 5; ++n) { st->cx[n] = st->cy[n] = st->cz[n] = 0.0; }
        const double idx = 1.0 / dx[0], idy = 1.0 / dx[1], idz = 1.0 / dx[2];
        st->cx[0] = idx; st->cy[0] = idy; st->cz[0] = idz;
        if (algo == PIC_SOLVER_YEE) return;
        const double delta = std::max(idx, std::max(idy, idz));
        const double rx = (idx / delta) * (idx / delta);
        const double ry = (idy / delta) * (idy / delta);
        const double rz = (idz / delta) * (idz / delta);
        const double beta = 0.125 * (1.0 - rx * ry * rz / (ry * rz + rz * rx + rx * ry));
        const double irf = (1.0 / (ry * rz + rz * rx + rx * ry));
        const double gx = ry * rz * (0.0625 - 0.125 * ry * rz * irf);
        const double gy = rx * rz * (0.0625 - 0.125 * rx * rz * irf);
        const double gz = rx * ry * (0.0625 - 0.125 * rx * ry * irf);
        st->cx[1] = (1.0 - 2.0 * ry * beta - 2.0 * rz * beta - 4.0 * gx) * idx;
        st->cy[1] = (1.0 - 2.0 * rx * beta - 2.0 * rz * beta - 4.0 * gy) * idy;
        st->cz[1] = (1.0 - 2.0 * rx * beta - 2.0 * ry * beta - 4.0 * gz) * idz;
        st->cx[2] = ry * beta * idx;  st->cx[3] = rz * beta * idx;  st->cx[4] = gx * idx;
        st->cy[2] = rz * beta * idy;  st->cy[3] = rx * beta * idy;  st->cy[4] = gy * idy;
        st->cz[2] = rx * beta * idz;  st->cz[3] = ry * beta * idz;  st->cz[4] = gz * idz;
    }
    static double max_dt(int algo, const double dx[3]) {
        if (algo == PIC_SOLVER_YEE) {
            return 1.0 / (std::sqrt(1.0 / (dx[0] * dx[0]) + 1.0 / (dx[1] * dx[1])
                                    + 1.0 / (dx[2] * dx[2])) * si::c);
        }
        return std::min(dx[0], std::min(dx[1], dx[2])) / si::c;
    }
};

}  // namespace orc
#endif
