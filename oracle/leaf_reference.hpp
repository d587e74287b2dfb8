// TEST INFRASTRUCTURE -- the same Leaf interface as leaf_restated.hpp, but every routine
// forwards to the REFERENCE's own header, compiled verbatim from a WarpX source tree's Source/ through
// the minimal AMReX stand-in in oracle/amrex_shim.  Only built on request
// (make -C oracle ref REF=<WarpX tree> -> oracle/_ref/libpic_oracle_ref.so); no reference source is
// copied into this repository.
#ifndef PIC_ORACLE_LEAF_REFERENCE_HPP_
#define PIC_ORACLE_LEAF_REFERENCE_HPP_

#include <AMReX.H>
#include <AMReX_Array4.H>
#include "Utils/WarpXConst.H"
#include "Particles/ShapeFactors.H"
#include "Particles/Pusher/UpdateMomentumBoris.H"
#include "Particles/Pusher/UpdateMomentumVay.H"
#include "Particles/Pusher/UpdateMomentumHigueraCary.H"
#include "Particles/Pusher/UpdatePosition.H"
#include "FieldSolver/FiniteDifferenceSolver/FiniteDifferenceAlgorithms/CartesianYeeAlgorithm.H"
#include "FieldSolver/FiniteDifferenceSolver/FiniteDifferenceAlgorithms/CartesianCKCAlgorithm.H"

#include "../include/pic_b200.h"

namespace orc {

struct LeafReference {
    static constexpr const char* name = "reference";
    using Arr = amrex::Array4<amrex::Real const>;
    static Arr arr(const pic_fab& f) { return Arr(f.p, f.lo, f.hi); }

    template <int N> static int shape(double* s, double xmid) {
        return Compute_shape_factor<N>()(s, xmid);
    }
    template <int N> static int shifted_shape(double* s, double x_old, int i_new) {
        return Compute_shifted_shape_factor<N>()(s, x_old, i_new);
    }
    static void boris(double& ux, double& uy, double& uz, double Ex, double Ey, double Ez,
                      double Bx, double By, double Bz, double q, double m, double dt) {
        UpdateMomentumBoris(ux, uy, uz, Ex, Ey, Ez, Bx, By, Bz, q, m, dt);
    }
    static void vay(double& ux, double& uy, double& uz, double Ex, double Ey, double Ez,
                    double Bx, double By, double Bz, double q, double m, double dt) {
        UpdateMomentumVay(ux, uy, uz, Ex, Ey, Ez, Bx, By, Bz, q, m, dt);
    }
    static void higuera_cary(double& ux, double& uy, double& uz, double Ex, double Ey, double Ez,
                             double Bx, double By, double Bz, double q, double m, double dt) {
        UpdateMomentumHigueraCary<double>(ux, uy, uz, Ex, Ey, Ez, Bx, By, Bz, q, m, dt);
    }
    static void update_position(double& x, double& y, double& z, double ux, double uy, double uz,
                                double dt) {
        UpdatePosition(x, y, z, ux, uy, uz, dt);
    }
    template <int D> static double upward(int algo, const Arr& F, const double* c, int i, int j,
                                          int k) {
        if (algo == PIC_SOLVER_YEE) {
            if constexpr (D == 0) return CartesianYeeAlgorithm::UpwardDx(F, c, 1, i, j, k);
            else if constexpr (D == 1) return CartesianYeeAlgorithm::UpwardDy(F, c, 1, i, j, k);
            else return CartesianYeeAlgorithm::UpwardDz(F, c, 1, i, j, k);
        } else {
            if constexpr (D == 0) return CartesianCKCAlgorithm::UpwardDx(F, c, 5, i, j, k);
            else if constexpr (D == 1) return CartesianCKCAlgorithm::UpwardDy(F, c, 5, i, j, k);
            else return CartesianCKCAlgorithm::UpwardDz(F, c, 5, i, j, k);
        }
    }
    template <int D> static double downward(int algo, const Arr& F, const double* c, int i, int j,
                                            int k) {
        if (algo == PIC_SOLVER_YEE) {
            if constexpr (D == 0) return CartesianYeeAlgorithm::DownwardDx(F, c, 1, i, j, k);
            else if constexpr (D == 1) return CartesianYeeAlgorithm::DownwardDy(F, c, 1, i, j, k);
            else return CartesianYeeAlgorithm::DownwardDz(F, c, 1, i, j, k);
        } else {
            if constexpr (D == 0) return CartesianCKCAlgorithm::DownwardDx(F, c, 5, i, j, k);
            else if constexpr (D == 1) return CartesianCKCAlgorithm::DownwardDy(F, c, 5, i, j, k);
            else return CartesianCKCAlgorithm::DownwardDz(F, c, 5, i, j, k);
        }
    }
    // stencil coefficients and max dt straight from the reference policies
    static void stencil_coefs(int algo, const double dx[3], pic_stencil* st) {
        std::array<amrex::Real, 3> cs{dx[0], dx[1], dx[2]};
        amrex::Vector<amrex::Real> cx, cy, cz;
        if (algo == PIC_SOLVER_YEE) CartesianYeeAlgorithm::InitializeStencilCoefficients(cs, cx, cy, cz);
        else CartesianCKCAlgorithm::InitializeStencilCoefficients(cs, cx, cy, cz);
        st->algo = algo;
        for (int n = 0; n < 5; ++n) {
            st->cx[n] = n < (int)cx.size() ? cx[n] : 0.0;
            st->cy[n] = n < (int)cy.size() ? cy[n] : 0.0;
            st->cz[n] = n < (int)cz.size() ? cz[n] : 0.0;
        }
    }
    static double max_dt(int algo, const double dx[3]) {
        return algo == PIC_SOLVER_YEE ? CartesianYeeAlgorithm::ComputeMaxDt(dx)
                                      : CartesianCKCAlgorithm::ComputeMaxDt(dx);
    }
};

}  // namespace orc
#endif
