// TEST INFRASTRUCTURE -- CPU oracle of the stages that the laser-wakefield decks add to the
// periodic EM-PIC step (SURVEY.md 8f rank 3): PEC field / current boundaries, the moving window,
// the laser antenna and continuous plasma injection.  fp64, single box covering the domain.
// Every routine cites the reference lines it follows (paths relative to Source/ of ECP-WarpX/WarpX).
//
// Only tests/, __graft_entry__.smoke() and the cpu_baseline / --impl reference legs of bench.py
// may use this; the product (warpx_b200/) never links, imports or executes anything in oracle/.
#ifndef PIC_ORACLE_LWFA_HPP_
#define PIC_ORACLE_LWFA_HPP_

#include <complex>
#include <limits>

#include "pic_oracle_core.hpp"

namespace orc {

constexpr double PI = 3.14159265358979323846;   // ablastr/constant.H:37 (MathConst::pi)

// ============================================================================================
// PEC on E and B.  PEC::ApplyPECtoEfield / ApplyPECtoBfield (BoundaryConditions/WarpX_PEC.cpp:
// 456-612) with ::SetEfieldOnPEC (:120-190) and ::SetBfieldOnPEC (:252-318), called after every
// EvolveE / EvolveB (FieldSolver/WarpXPushFieldsEM.cpp:926,990 -> BoundaryConditions/
// WarpXFieldBoundaries.cpp:51-159).  Region: mfi.tilebox(nodal_flag, ng_fieldgather) = the valid
// points of the component grown by ng_FieldGather (:508-513).
//   is_E = true : tangential components vanish on the wall, are odd across it; normal are even.
//   is_E = false: normal component vanishes on the wall, is odd across it; tangential are even.
// ============================================================================================
inline void apply_pec_field(const pic_fab F[3], bool is_E, const pic_geom& g, const pic_boundaries& bnd,
                            const int ng_fg[3]) {
    for (int icomp = 0; icomp < 3; ++icomp) {
        const pic_fab& f = F[icomp];
        W A(f);
        const int lo[3] = {vlo(f, 0) - ng_fg[0], vlo(f, 1) - ng_fg[1], vlo(f, 2) - ng_fg[2]};
        const int hi[3] = {vhi(f, 0) + ng_fg[0], vhi(f, 1) + ng_fg[1], vhi(f, 2) + ng_fg[2]};
        for (int k = lo[2]; k <= hi[2]; ++k)
            for (int j = lo[1]; j <= hi[1]; ++j)
                for (int i = lo[0]; i <= hi[0]; ++i) {
                    const int ijk[3] = {i, j, k};
                    int mir[3] = {i, j, k};
                    bool on_pec = false, guard = false;
                    double sign = 1.0;
                    for (int idim = 0; idim < 3; ++idim)
                        for (int iside = 0; iside < 2; ++iside) {
                            const bool is_pec = (iside == 0 ? bnd.field_lo[idim] : bnd.field_hi[idim]) == PIC_FIELD_PEC;
                            if (!is_pec) continue;
                            // E: flips when tangential (icomp != idim); B: flips when normal (icomp == idim)
                            const bool flips = is_E ? (icomp != idim) : (icomp == idim);
                            const int dom_lo = 0, dom_hi = g.n_cell[idim] - 1;
                            // get_cell_count_to_boundary (:42-49)
                            const int ig = (iside == 0) ? (dom_lo - ijk[idim])
                                                        : (ijk[idim] - (dom_hi + f.stag[idim]));
                            if (ig == 0) {
                                if (flips && f.stag[idim] == 1) on_pec = true;
                            } else if (ig > 0) {
                                mir[idim] = (iside == 0) ? (dom_lo + ig - (1 - f.stag[idim]))
                                                         : (dom_hi + 1 - ig);
                                guard = true;
                                if (flips) sign *= -1.0;
                            }
                        }
                    if (on_pec) A(i, j, k) = 0.0;
                    else if (guard) A(i, j, k) = sign * A(mir[0], mir[1], mir[2]);
                }
    }
}

// ============================================================================================
// Reflective / PEC boundary on J.  PEC::ApplyReflectiveBoundarytoJfield (WarpX_PEC.cpp:702-880)
// with ::SetRhoOrJfieldFromPEC (:340-395), called at the end of WarpX::SyncCurrentAndRho
// (Evolve/WarpXEvolve.cpp:629-652).  Loop over the valid points of each component; the mirror
// guard point must exist in the fab.
// ============================================================================================
inline void apply_pec_current(const pic_fab J[3], const pic_geom& g, const pic_boundaries& bnd) {
    for (int icomp = 0; icomp < 3; ++icomp) {
        const pic_fab& f = J[icomp];
        W A(f);
        bool is_refl[3][2], tangent[3];
        double psign[3][2];
        int mirrorfac[3][2];
        bool any = false;
        for (int idim = 0; idim < 3; ++idim) {
            const bool plo = bnd.particle_lo[idim] == PIC_PARTICLE_REFLECTING;
            const bool phi = bnd.particle_hi[idim] == PIC_PARTICLE_REFLECTING;
            is_refl[idim][0] = plo || bnd.field_lo[idim] == PIC_FIELD_PEC;        // :735-740
            is_refl[idim][1] = phi || bnd.field_hi[idim] == PIC_FIELD_PEC;
            any = any || is_refl[idim][0] || is_refl[idim][1];
            tangent[idim] = (icomp != idim);                                       // :757
            if (tangent[idim]) { psign[idim][0] = plo ? 1.0 : -1.0; psign[idim][1] = phi ? 1.0 : -1.0; }   // :760-767
            else               { psign[idim][0] = plo ? -1.0 : 1.0; psign[idim][1] = phi ? -1.0 : 1.0; }   // :769-776
            // nodal domain box [0, n_cell] (:716-719); :783-788
            mirrorfac[idim][0] = 2 * 0 - (1 - f.stag[idim]);
            mirrorfac[idim][1] = 2 * g.n_cell[idim] - (1 - f.stag[idim]);
        }
        if (!any) continue;
        auto contains = [&](const int* iv) {
            return iv[0] >= f.lo[0] && iv[0] <= f.hi[0] && iv[1] >= f.lo[1] && iv[1] <= f.hi[1] &&
                   iv[2] >= f.lo[2] && iv[2] <= f.hi[2];
        };
        for (int k = vlo(f, 2); k <= vhi(f, 2); ++k)
            for (int j = vlo(f, 1); j <= vhi(f, 1); ++j)
                for (int i = vlo(f, 0); i <= vhi(f, 0); ++i) {
                    const int ijk[3] = {i, j, k};
                    // 1) interior points receive what was deposited in the mirror guard point (:354-374)
                    for (int idim = 0; idim < 3; ++idim)
                        for (int iside = 0; iside < 2; ++iside) {
                            if (!is_refl[idim][iside]) continue;
                            int mir[3] = {i, j, k};
                            mir[idim] = mirrorfac[idim][iside] - ijk[idim];
                            if (mir[idim] == ijk[idim]) A(i, j, k) = 0.0;
                            else if (contains(mir)) A(i, j, k) += psign[idim][iside] * A(mir[0], mir[1], mir[2]);
                        }
                    // 2) guard points get the image charge of the interior points (:377-394)
                    for (int idim = 0; idim < 3; ++idim)
                        for (int iside = 0; iside < 2; ++iside) {
                            if (!is_refl[idim][iside]) continue;
                            int mir[3] = {i, j, k};
                            mir[idim] = mirrorfac[idim][iside] - ijk[idim];
                            if (mir[idim] != ijk[idim] && contains(mir))
                                A(mir[0], mir[1], mir[2]) = tangent[idim] ? -A(i, j, k) : A(i, j, k);
                        }
                }
    }
}

// PEC::ApplyReflectiveBoundarytoRhofield (WarpX_PEC.cpp:624-699): like the tangential current --
// the wall value vanishes, the interior loses the image charge deposited beyond the wall (psign = -1
// unless the particles are reflected), the guards hold minus the interior.  mirrorfac: :679-680.
inline void apply_pec_rho(const pic_fab& f, const pic_geom& g, const pic_boundaries& bnd) {
    W A(f);
    bool is_refl[3][2];
    double psign[3][2];
    int mirrorfac[3][2];
    bool any = false;
    for (int idim = 0; idim < 3; ++idim) {
        const bool plo = bnd.particle_lo[idim] == PIC_PARTICLE_REFLECTING;
        const bool phi = bnd.particle_hi[idim] == PIC_PARTICLE_REFLECTING;
        is_refl[idim][0] = plo || bnd.field_lo[idim] == PIC_FIELD_PEC;
        is_refl[idim][1] = phi || bnd.field_hi[idim] == PIC_FIELD_PEC;
        any = any || is_refl[idim][0] || is_refl[idim][1];
        psign[idim][0] = plo ? 1.0 : -1.0;
        psign[idim][1] = phi ? 1.0 : -1.0;
        const int dom_lo = 0, dom_hi = g.n_cell[idim] - 1 + f.stag[idim];     // domain box converted to rho's type
        mirrorfac[idim][0] = 2 * dom_lo - (1 - f.stag[idim]);
        mirrorfac[idim][1] = 2 * dom_hi + (1 - f.stag[idim]);
    }
    if (!any) return;
    auto contains = [&](const int* iv) {
        return iv[0] >= f.lo[0] && iv[0] <= f.hi[0] && iv[1] >= f.lo[1] && iv[1] <= f.hi[1] &&
               iv[2] >= f.lo[2] && iv[2] <= f.hi[2];
    };
    for (int k = vlo(f, 2); k <= vhi(f, 2); ++k)
        for (int j = vlo(f, 1); j <= vhi(f, 1); ++j)
            for (int i = vlo(f, 0); i <= vhi(f, 0); ++i) {
                const int ijk[3] = {i, j, k};
                for (int idim = 0; idim < 3; ++idim)
                    for (int iside = 0; iside < 2; ++iside) {
                        if (!is_refl[idim][iside]) continue;
                        int mir[3] = {i, j, k};
                        mir[idim] = mirrorfac[idim][iside] - ijk[idim];
                        if (mir[idim] == ijk[idim]) A(i, j, k) = 0.0;
                        else if (contains(mir)) A(i, j, k) += psign[idim][iside] * A(mir[0], mir[1], mir[2]);
                    }
                for (int idim = 0; idim < 3; ++idim)
                    for (int iside = 0; iside < 2; ++iside) {
                        if (!is_refl[idim][iside]) continue;
                        int mir[3] = {i, j, k};
                        mir[idim] = mirrorfac[idim][iside] - ijk[idim];
                        if (mir[idim] != ijk[idim] && contains(mir)) A(mir[0], mir[1], mir[2]) = -A(i, j, k);
                    }
            }
}

// ============================================================================================
// Moving window: shift of one field component by num_shift cells along dir.
// WarpX::shiftMF (Utils/WarpXMovingWindow.cpp:478-604), single box:
//   tmp = copy incl. guards (:492-493); FillBoundary(tmp, ng_mw) with ng_mw = 1 everywhere and
//   num_shift along dir, capped by ng (:499-505); the allocated points beyond the domain face the
//   window moves into are set to external_field (:508-531,552-556); then
//   dst(i,j,k) = tmp(i,j,k + shift) over the fab box shortened by |num_shift| at the far end (:591-600).
// ============================================================================================
inline void shift_fab(const pic_fab& f, const pic_geom& g, int num_shift, int dir, double external_field) {
    if (num_shift == 0) return;
    std::vector<double> buf((size_t)fab_size(f));
    std::memcpy(buf.data(), f.p, buf.size() * sizeof(double));
    pic_fab t = f;
    t.p = buf.data();
    int ng_mw[3] = {1, 1, 1};
    ng_mw[dir] = std::abs(num_shift);
    for (int d = 0; d < 3; ++d) ng_mw[d] = std::min(ng_mw[d], f.ng[d]);
    fill_boundary(&t, 1, ng_mw, g);
    W S(t), D(f);
    int lo[3] = {f.lo[0], f.lo[1], f.lo[2]}, hi[3] = {f.hi[0], f.hi[1], f.hi[2]};
    // adjBox: adjCellHi/Lo(domain, dir, ng) converted to the component's index type, minus the
    // boundary node when nodal along dir, grown by ng in the other directions
    if (num_shift > 0) { lo[dir] = vhi(f, dir) + 1; hi[dir] = vhi(f, dir) + f.ng[dir]; }
    else               { lo[dir] = vlo(f, dir) - f.ng[dir]; hi[dir] = vlo(f, dir) - 1; }
    for (int k = lo[2]; k <= hi[2]; ++k)
        for (int j = lo[1]; j <= hi[1]; ++j)
            for (int i = lo[0]; i <= hi[0]; ++i) S(i, j, k) = external_field;
    int dlo[3] = {f.lo[0], f.lo[1], f.lo[2]}, dhi[3] = {f.hi[0], f.hi[1], f.hi[2]};
    if (num_shift > 0) dhi[dir] -= num_shift; else dlo[dir] -= num_shift;
    const int sh[3] = {dir == 0 ? num_shift : 0, dir == 1 ? num_shift : 0, dir == 2 ? num_shift : 0};
    for (int k = dlo[2]; k <= dhi[2]; ++k)
        for (int j = dlo[1]; j <= dhi[1]; ++j)
            for (int i = dlo[0]; i <= dhi[0]; ++i) D(i, j, k) = S(i + sh[0], j + sh[1], k + sh[2]);
}

// ============================================================================================
// Laser antenna.  LaserParticleContainer (Particles/LaserParticleContainer.cpp), 3D; lab frame or a
// frame boosted along the propagation direction (prm.gamma_boost > 1).
// ============================================================================================
struct Antenna {
    pic_laser_antenna prm;          // nvec, p_X normalised; position in the simulation frame
    double p_Y[3], u_X[3], u_Y[3];
    double S_X, S_Y, mobility, weight;
    double Z0_lab;                  // antenna plane along nvec in the lab frame (boosted runs)
    bool boosted;
};

// Constructor (:84-270, 3D: u_X = p_X, u_Y = p_Y = nvec x p_X) + ComputeSpacing (:727-761) +
// ComputeWeightMobility (:763-781).
inline Antenna antenna_setup(const pic_laser_antenna& in, const double dx[3]) {
    Antenna a;
    a.prm = in;
    double s = 1.0 / std::sqrt(in.nvec[0] * in.nvec[0] + in.nvec[1] * in.nvec[1] + in.nvec[2] * in.nvec[2]);   // :179-180
    for (int d = 0; d < 3; ++d) a.prm.nvec[d] = in.nvec[d] * s;
    a.boosted = in.gamma_boost > 1.;
    a.Z0_lab = 0.0;
    if (a.boosted) {                                                                                               // :183-197
        a.Z0_lab = a.prm.nvec[0] * a.prm.position[0] + a.prm.nvec[1] * a.prm.position[1] + a.prm.nvec[2] * a.prm.position[2];
        const double Z0_boost = a.Z0_lab / in.gamma_boost;
        for (int d = 0; d < 3; ++d) a.prm.position[d] += (Z0_boost - a.Z0_lab) * a.prm.nvec[d];
    }
    s = 1.0 / std::sqrt(in.p_X[0] * in.p_X[0] + in.p_X[1] * in.p_X[1] + in.p_X[2] * in.p_X[2]);                 // :199-200
    for (int d = 0; d < 3; ++d) a.prm.p_X[d] = in.p_X[d] * s;
    const double* n = a.prm.nvec; const double* p = a.prm.p_X;
    a.p_Y[0] = n[1] * p[2] - n[2] * p[1]; a.p_Y[1] = n[2] * p[0] - n[0] * p[2]; a.p_Y[2] = n[0] * p[1] - n[1] * p[0];   // :207
    for (int d = 0; d < 3; ++d) { a.u_X[d] = a.prm.p_X[d]; a.u_Y[d] = a.p_Y[d]; }                                 // :210-211
    const double eps = dx[0] * 1.e-50;                                                                             // :733-738
    a.S_X = std::min(std::min(dx[0] / (std::abs(a.u_X[0]) + eps), dx[1] / (std::abs(a.u_X[1]) + eps)),
                     dx[2] / (std::abs(a.u_X[2]) + eps));                                                          // :740-742
    a.S_Y = std::min(std::min(dx[0] / (std::abs(a.u_Y[0]) + eps), dx[1] / (std::abs(a.u_Y[1]) + eps)),
                     dx[2] / (std::abs(a.u_Y[2]) + eps));                                                          // :743-745
    a.mobility = 0.05 / a.prm.e_max;                                                                               // :770-771
    a.weight = EP0 / a.mobility;                                                                                   // :772
    a.weight *= 1.0 * a.S_X * a.S_Y;                                                                               // :774
    if (a.boosted) a.mobility = a.mobility / in.gamma_boost;                                                       // :775 (divides by 1 otherwise)
    return a;
}

// RealBox::contains(point): strictly inside (AMReX_RealBox.H, eps = 0).
inline bool realbox_contains(const double lo[3], const double hi[3], const double p[3]) {
    return lo[0] < p[0] && p[0] < hi[0] && lo[1] < p[1] && p[1] < hi[1] && lo[2] < p[2] && p[2] < hi[2];
}

// LaserParticleContainer::InitData(lev) (:369-560): one +w / -w pair per cell of the antenna plane
// grid that lies inside the injection box.  out[0..6] = x y z w ux uy uz (appended).
inline void antenna_init_particles(const Antenna& a, const double box_lo[3], const double box_hi[3],
                                   std::vector<double> out[7]) {
    const double* pos0 = a.prm.position;
    int plane_lo[2] = {std::numeric_limits<int>::max(), std::numeric_limits<int>::max()};
    int plane_hi[2] = {std::numeric_limits<int>::min(), std::numeric_limits<int>::min()};
    for (int c = 0; c < 8; ++c) {                                                                  // :436-443
        const double x = (c & 1) ? box_hi[0] : box_lo[0], y = (c & 2) ? box_hi[1] : box_lo[1],
                     z = (c & 4) ? box_hi[2] : box_lo[2];
        const double px = a.u_X[0] * (x - pos0[0]) + a.u_X[1] * (y - pos0[1]) + a.u_X[2] * (z - pos0[2]);   // :405-407
        const double py = a.u_Y[0] * (x - pos0[0]) + a.u_Y[1] * (y - pos0[1]) + a.u_Y[2] * (z - pos0[2]);
        const int i = static_cast<int>(px / a.S_X), j = static_cast<int>(py / a.S_Y);             // :424-425
        plane_lo[0] = std::min(plane_lo[0], i); plane_lo[1] = std::min(plane_lo[1], j);
        plane_hi[0] = std::max(plane_hi[0], i); plane_hi[1] = std::max(plane_hi[1], j);
    }
    for (int j = plane_lo[1]; j <= plane_hi[1]; ++j)            // Box::next: first index fastest (:497)
        for (int i = plane_lo[0]; i <= plane_hi[0]; ++i) {
            const double pos[3] = {                                                                 // :384-387
                pos0[0] + (a.S_X * (double(i) + 0.5)) * a.u_X[0] + (a.S_Y * (double(j) + 0.5)) * a.u_Y[0],
                pos0[1] + (a.S_X * (double(i) + 0.5)) * a.u_X[1] + (a.S_Y * (double(j) + 0.5)) * a.u_Y[1],
                pos0[2] + (a.S_X * (double(i) + 0.5)) * a.u_X[2] + (a.S_Y * (double(j) + 0.5)) * a.u_Y[2]};
            if (!realbox_contains(box_lo, box_hi, pos)) continue;                                  // :511
            for (int kk = 0; kk < 2; ++kk) {                                                       // :514-520
                out[0].push_back(pos[0]); out[1].push_back(pos[1]); out[2].push_back(pos[2]);
                out[4].push_back(0.0); out[5].push_back(0.0); out[6].push_back(0.0);
            }
            out[3].push_back(a.weight); out[3].push_back(-a.weight);
        }
}

// One step of the antenna particles (LaserParticleContainer::Evolve :614-626):
// calculate_laser_plane_coordinates (:800-848), GaussianLaserProfile::fill_amplitude
// (LaserProfileGaussian.cpp:100-162, zeta = beta = phi2 = 0 so stretch_factor = 1 and theta_stc
// drops out), update_laser_particle (:860-951, explicit push).  In a boosted frame the profile is
// evaluated at the lab time of the antenna plane (:573-579) and the antenna drifts with -beta c nvec.
inline void antenna_push(const Antenna& a, const pic_soa& P, double t_sim, double dt) {
    using cplx = std::complex<double>;
    const double gamma_boost = a.boosted ? a.prm.gamma_boost : 1.0, beta_boost = a.boosted ? a.prm.beta_boost : 0.0;
    const double t = a.boosted ? 1. / gamma_boost * t_sim + beta_boost * a.Z0_lab / C_LIGHT : t_sim;
    const cplx I(0.0, 1.0);
    const double k0 = 2.0 * PI / a.prm.wavelength;
    const double inv_tau2 = 1.0 / (a.prm.duration * a.prm.duration);
    const double oscillation_phase = k0 * C_LIGHT * (t - a.prm.t_peak) + a.prm.phi0;
    const cplx diffract_factor = 1.0 + I * a.prm.focal_distance * 2.0 / (k0 * a.prm.waist * a.prm.waist);
    const cplx inv_complex_waist_2 = 1.0 / (a.prm.waist * a.prm.waist * diffract_factor);
    const cplx stretch_factor = 1.0 + 4.0 * (0.0 + 0.0 * a.prm.focal_distance * inv_tau2)
                                          * (0.0 + 0.0 * a.prm.focal_distance * inv_complex_waist_2)
                              + 2.0 * I * (0.0 - 0.0 * 0.0 * k0 * a.prm.focal_distance) * inv_tau2;
    const cplx t_prefactor = a.prm.e_max * std::exp(I * oscillation_phase);
    const cplx prefactor = t_prefactor / diffract_factor;                                          // 3D (:134)
#pragma omp parallel for schedule(static)
    for (long ip = 0; ip < P.np; ++ip) {
        const double x = P.x[ip], y = P.y[ip], z = P.z[ip];
        const double Xp = a.u_X[0] * (x - a.prm.position[0]) + a.u_X[1] * (y - a.prm.position[1])
                        + a.u_X[2] * (z - a.prm.position[2]);
        const double Yp = a.u_Y[0] * (x - a.prm.position[0]) + a.u_Y[1] * (y - a.prm.position[1])
                        + a.u_Y[2] * (z - a.prm.position[2]);
        const cplx arg = (t - a.prm.t_peak) - 0.0 * k0 * (Xp * 1.0 + Yp * 0.0)
                         - 2.0 * I * (Xp * 1.0 + Yp * 0.0) * (0.0 - 0.0 * a.prm.focal_distance) * inv_complex_waist_2;
        const cplx stc_exponent = 1.0 / stretch_factor * inv_tau2 * (arg * arg);                   // amrex::pow(.,2)
        const cplx stcfactor = prefactor * std::exp(-stc_exponent);
        const cplx exp_argument = -(Xp * Xp + Yp * Yp) * inv_complex_waist_2;
        const double amplitude = (stcfactor * std::exp(exp_argument)).real();
        // update_laser_particle (:905-949)
        const double sign_charge = (P.w[ip] > 0) ? -1.0 : 1.0;
        const double v_over_c = sign_charge * a.mobility * amplitude;
        double vx = C_LIGHT * v_over_c * a.prm.p_X[0];
        double vy = C_LIGHT * v_over_c * a.prm.p_X[1];
        double vz = C_LIGHT * v_over_c * a.prm.p_X[2];
        if (gamma_boost > 1.) {                                                                    // :908-912
            vx -= C_LIGHT * beta_boost * a.prm.nvec[0];
            vy -= C_LIGHT * beta_boost * a.prm.nvec[1];
            vz -= C_LIGHT * beta_boost * a.prm.nvec[2];
        }
        const double gamma = gamma_boost / std::sqrt(1. - v_over_c * v_over_c);                  // :914-915
        P.ux[ip] = gamma * vx; P.uy[ip] = gamma * vy; P.uz[ip] = gamma * vz;
        P.x[ip] = x + vx * dt; P.y[ip] = y + vy * dt; P.z[ip] = z + vz * dt;
    }
}

// ============================================================================================
// Plasma injection.  PhysicalParticleContainer::AddPlasma (Particles/PhysicalParticleContainer.cpp:
// 924-1333) for injection_style = NUniformPerCell, profile = constant, momentum at rest (in the lab
// frame; inj.gamma_boost > 1: frame boosted along z, t = t_new), one tile = the whole box (tile decomposition only changes positions at the
// rounding level, see find_overlap).  part_lo/hi = the RealBox particles are requested in
// (whole domain at start-up, the freshly uncovered slab for continuous injection).
// Appends to out[0..6]; returns the number of particles added.
// ============================================================================================
inline long add_plasma(const pic_plasma_injector& inj, const pic_geom& g, const double dx[3],
                       const double part_lo[3], const double part_hi[3], std::vector<double> out[7],
                       double t = 0.0) {
    const bool boosted = inj.gamma_boost > 1.;
    const double gamma_boost = boosted ? inj.gamma_boost : 1.0, beta_boost = boosted ? inj.beta_boost : 0.0;
    // applyBallisticCorrection (:138-148) for a plasma at rest in the lab: betaz_bulk = 0
    auto z_lab = [&](double z) { return gamma_boost * (z * (1.0 - beta_boost * 0.0) - C_LIGHT * t * (0.0 - beta_boost)); };
    // tile_realbox = RealBox(box, dx, prob_lo) (WarpX::getRealBox, WarpX.cpp:2852-2857)
    double tile_lo[3], tile_hi[3], ov_lo[3], ov_hi[3];
    int nov[3];
    for (int d = 0; d < 3; ++d) {
        tile_lo[d] = g.prob_lo[d] + dx[d] * 0;
        tile_hi[d] = g.prob_lo[d] + dx[d] * (g.n_cell[d] - 1 + 1);
        // find_overlap (Particles/AddPlasmaUtilities.cpp:12-43)
        if (tile_lo[d] <= part_hi[d]) {
            const double adj = std::floor((tile_lo[d] - part_lo[d]) / dx[d]);
            ov_lo[d] = part_lo[d] + std::max(adj, 0.0) * dx[d];
        } else return 0;
        if (tile_hi[d] >= part_lo[d]) {
            const double adj = std::floor((part_hi[d] - tile_hi[d]) / dx[d]);
            ov_hi[d] = part_hi[d] - std::max(adj, 0.0) * dx[d];
        } else return 0;
        nov[d] = int(std::round((ov_hi[d] - ov_lo[d]) / dx[d]));       // overlap_box = [0, nov-1]
    }
    const int num_ppc = inj.ppc[0] * inj.ppc[1] * inj.ppc[2];
    auto inside = [&](double x, double y, double z) {                    // InjectorPosition::insideBounds (InjectorPosition.H:202-207)
        return x < inj.bound_hi[0] && x >= inj.bound_lo[0] && y < inj.bound_hi[1] && y >= inj.bound_lo[1] &&
               z < inj.bound_hi[2] && z >= inj.bound_lo[2];
    };
    long added = 0;
    // Box iteration order of ParallelFor on the host: i fastest
    for (int k = 0; k < nov[2]; ++k)
        for (int j = 0; j < nov[1]; ++j)
            for (int i = 0; i < nov[0]; ++i) {
                const int iv[3] = {i, j, k};
                double lo[3], hi[3];
                for (int d = 0; d < 3; ++d) {                            // getCellCoords (:151-175)
                    lo[d] = ov_lo[d] + (iv[d] + 0.0) * dx[d];
                    hi[d] = ov_lo[d] + (iv[d] + 1.0) * dx[d];
                }
                lo[2] = z_lab(lo[2]); hi[2] = z_lab(hi[2]);                 // :1021-1022 (identity in the lab frame)
                // overlapsWith (InjectorPosition.H:228-233)
                if (!((inj.bound_lo[0] <= hi[0]) && (inj.bound_hi[0] >= lo[0]) && (inj.bound_lo[1] <= hi[1]) &&
                      (inj.bound_hi[1] >= lo[1]) && (inj.bound_lo[2] <= hi[2]) && (inj.bound_hi[2] >= lo[2])))
                    continue;
                // corners / centre test (:1032-1049); constant density > 0
                bool any = false;
                const double xl[3] = {lo[0], (lo[0] + hi[0]) / 2.0, hi[0]}, yl[3] = {lo[1], (lo[1] + hi[1]) / 2.0, hi[1]},
                             zl[3] = {lo[2], (lo[2] + hi[2]) / 2.0, hi[2]};
                for (int a = 0; a < 3 && !any; ++a)
                    for (int b = 0; b < 3 && !any; ++b)
                        for (int c = 0; c < 3 && !any; ++c)
                            if (inside(xl[a], yl[b], zl[c]) && inj.density > 0) any = true;
                if (!any) continue;
                const long pcount = num_ppc;
                const double scale_fac = dx[0] * dx[1] * dx[2] / pcount;                   // compute_scale_fac_volume (AddPlasmaUtilities.H:73-77)
                for (int i_part = 0; i_part < pcount; ++i_part) {
                    // InjectorPositionRegular::getPositionUnitBox (InjectorPosition.H:78-108), ref_fac = 1
                    const int nx = inj.ppc[0], ny = inj.ppc[1], nz = inj.ppc[2];
                    const int ix_part = i_part / (ny * nz);
                    const int iz_part = (i_part - ix_part * (ny * nz)) / ny;
                    const int iy_part = (i_part - ix_part * (ny * nz)) - ny * iz_part;
                    const double r[3] = {(0.5 + ix_part) / nx, (0.5 + iy_part) / ny, (0.5 + iz_part) / nz};
                    double pos[3];
                    for (int d = 0; d < 3; ++d) pos[d] = ov_lo[d] + (iv[d] + r[d]) * dx[d];
                    if (!realbox_contains(tile_lo, tile_hi, pos)) continue;                // :1141-1156
                    if (!inside(pos[0], pos[1], z_lab(pos[2]))) continue;                  // :1184-1197 / :1211-1224
                    double dens = inj.density, uz = 0.0;
                    if (boosted) {                                                           // :1232-1246, u = 0 in the lab
                        const double gamma_lab = std::sqrt(1. + (0.0 * 0.0 + 0.0 * 0.0 + uz * uz));
                        const double betaz_lab = uz / (gamma_lab);
                        dens = gamma_boost * dens * (1.0 - beta_boost * betaz_lab);
                        uz = gamma_boost * (uz - beta_boost * gamma_lab);
                    }
                    uz *= C_LIGHT;                                                           // :1275-1277
                    double weight = dens;                                                    // :1282-1283
                    weight *= scale_fac;
                    out[0].push_back(pos[0]); out[1].push_back(pos[1]); out[2].push_back(pos[2]);
                    out[3].push_back(weight);
                    out[4].push_back(0.0); out[5].push_back(0.0); out[6].push_back(uz);
                    ++added;
                }
            }
    return added;
}

// ============================================================================================
// Particle boundaries.  WarpXParticleContainer::ApplyBoundaryConditions (Particles/
// WarpXParticleContainer.cpp:1574-1638) -> ApplyParticleBoundaries::apply_boundary
// (Particles/ParticleBoundaries_K.H:21-75): absorbing -> lost, reflecting -> mirrored with the
// normal momentum flipped; followed by the removal done by AMReX Redistribute.
// keep[ip] = 0 marks particles to delete.
// ============================================================================================
inline void apply_particle_boundaries(const pic_soa& P, const pic_geom& g, const pic_boundaries& bnd,
                                      std::vector<char>& keep) {
    keep.assign((size_t)P.np, 1);
    double* X[3] = {P.x, P.y, P.z};
    double* U[3] = {P.ux, P.uy, P.uz};
    for (int d = 0; d < 3; ++d) {
        if (bnd.particle_lo[d] == PIC_PARTICLE_PERIODIC && bnd.particle_hi[d] == PIC_PARTICLE_PERIODIC) continue;
        const double lo = g.prob_lo[d], hi = g.prob_hi[d];
        for (long ip = 0; ip < P.np; ++ip) {
            double& x = X[d][ip];
            if (x < lo) {
                if (bnd.particle_lo[d] == PIC_PARTICLE_ABSORBING) keep[ip] = 0;
                else if (bnd.particle_lo[d] == PIC_PARTICLE_REFLECTING) { x = 2 * lo - x; U[d][ip] = -U[d][ip]; }
            } else if (x > hi) {
                if (bnd.particle_hi[d] == PIC_PARTICLE_ABSORBING) keep[ip] = 0;
                else if (bnd.particle_hi[d] == PIC_PARTICLE_REFLECTING) { x = 2 * hi - x; U[d][ip] = -U[d][ip]; }
            }
        }
    }
}

}  // namespace orc
#endif
