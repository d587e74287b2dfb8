// Stages that the laser-wakefield decks add to the periodic PIC step (SURVEY.md 8f rank 3; config 4
// of BASELINE.json needs all of them): PEC walls on E, B and J, the moving-window shift, the laser
// antenna, continuous plasma injection, absorbing / reflecting particle boundaries.
//
// Replaces (paths relative to Source/ of ECP-WarpX/WarpX):
//   pic_apply_pec_field          <- PEC::ApplyPECtoEfield / ApplyPECtoBfield   BoundaryConditions/WarpX_PEC.cpp:456-612
//   pic_apply_pec_current        <- PEC::ApplyReflectiveBoundarytoJfield       BoundaryConditions/WarpX_PEC.cpp:702-880
//   pic_shift_fab                <- WarpX::shiftMF                             Utils/WarpXMovingWindow.cpp:478-604
//   pic_laser_antenna_*          <- LaserParticleContainer                     Particles/LaserParticleContainer.cpp
//                                   GaussianLaserProfile::fill_amplitude       Laser/LaserProfilesImpl/LaserProfileGaussian.cpp:100-162
//   pic_add_plasma               <- PhysicalParticleContainer::AddPlasma       Particles/PhysicalParticleContainer.cpp:924-1333
//   pic_particles_boundary_*     <- WarpXParticleContainer::ApplyBoundaryConditions  Particles/WarpXParticleContainer.cpp:1574-1638
//                                   + the removal done by AMReX Redistribute
// All of them are thin HBM streams or O(surface) kernels; none is on the 256^3 benchmark path.
//
// The per-thread bodies are in lwfa_body.cuh.  With -DPIC_HOST_HARNESS (tests/host_harness only) the
// launches below become host loops over the same thread ids, so the CPU test-suite can compare the
// bodies and the host-side argument builders with the oracle where no GPU exists; the product library
// is never built that way.
#include "lwfa_body.cuh"
#include "harness_launch.cuh"
#include <cmath>
#include <complex>
#include <cstring>
#include <limits>
#include <vector>

namespace pic {

__global__ void pec_field_kernel(PecFieldArgs a) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.total) pec_field_body(t, a);
}
__global__ void pec_current_kernel(PecCurrentArgs a) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.total) pec_current_body(t, a);
}
__global__ void shift_kernel(ShiftArgs a) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.total) shift_body(t, a);
}
__global__ void laser_kernel(LaserArgs a) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.np) laser_body(t, a);
}
__global__ void inject_kernel(InjectArgs a) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.total) inject_body(t, a);
}

PIC_HD void boundary_mark_body(long ip, const BoundaryArgs& a) {
    if (boundary_body(ip, a)) { const int n = slot_add(a.count); if (n < a.cap) a.list[n] = (int)ip; }
}
__global__ void boundary_mark_kernel(BoundaryArgs a) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.np) boundary_mark_body(t, a);
}

// Removal of the listed particles: the survivors of the tail [m, n) move into the holes below m.
struct CompactArgs {
    SoaView P;
    uint64_t* id;
    const int* list;    // n_lost indices
    int* holes; int* srcs; int* tailflag;      // each n_lost ints
    int* nh; int* ns;
    long m;             // new particle count
    int n_lost;
};
PIC_HD void compact_split_body(long t, const CompactArgs& a) {      // t < n_lost
    const int idx = a.list[t];
    if (idx >= a.m) a.tailflag[idx - a.m] = 1;
    else a.holes[slot_add(a.nh)] = idx;
}
PIC_HD void compact_tail_body(long t, const CompactArgs& a) {       // t < n_lost (tail length)
    if (!a.tailflag[t]) a.srcs[slot_add(a.ns)] = (int)(a.m + t);
}
PIC_HD void compact_move_body(long t, const CompactArgs& a) {       // t < *nh (== *ns)
    if (t >= *a.nh) return;
    const int dst = a.holes[t], src = a.srcs[t];
    a.P.x[dst] = a.P.x[src]; a.P.y[dst] = a.P.y[src]; a.P.z[dst] = a.P.z[src]; a.P.w[dst] = a.P.w[src];
    a.P.ux[dst] = a.P.ux[src]; a.P.uy[dst] = a.P.uy[src]; a.P.uz[dst] = a.P.uz[src];
    if (a.id) a.id[dst] = a.id[src];
}
__global__ void compact_split_kernel(CompactArgs a) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.n_lost) compact_split_body(t, a);
}
__global__ void compact_tail_kernel(CompactArgs a) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.n_lost) compact_tail_body(t, a);
}
__global__ void compact_move_kernel(CompactArgs a) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.n_lost) compact_move_body(t, a);
}

// ---- host-side pieces -----------------------------------------------------------------------
struct AntennaSetup {
    double nvec[3], p_X[3], p_Y[3], u_X[3], u_Y[3];
    double S_X, S_Y, mobility, weight;
    double position[3];              // in the simulation frame
    double Z0_lab, gamma_boost, beta_boost;
};

// LaserParticleContainer ctor (:179-211, 3D: u_X = p_X, u_Y = p_Y = nvec x p_X), ComputeSpacing
// (:727-761), ComputeWeightMobility (:763-781); in a frame boosted along nvec the plane moves to
// Z0 / gamma_boost (:183-197) and the mobility is divided by gamma_boost (:775).
static AntennaSetup antenna_setup(const pic_laser_antenna& in, const double dx[3]) {
    AntennaSetup a;
    double s = 1.0 / std::sqrt(in.nvec[0] * in.nvec[0] + in.nvec[1] * in.nvec[1] + in.nvec[2] * in.nvec[2]);
    for (int d = 0; d < 3; ++d) { a.nvec[d] = in.nvec[d] * s; a.position[d] = in.position[d]; }
    const bool boosted = in.gamma_boost > 1.;
    a.gamma_boost = boosted ? in.gamma_boost : 1.0;
    a.beta_boost = boosted ? in.beta_boost : 0.0;
    a.Z0_lab = 0.0;
    if (boosted) {
        a.Z0_lab = a.nvec[0] * a.position[0] + a.nvec[1] * a.position[1] + a.nvec[2] * a.position[2];
        const double Z0_boost = a.Z0_lab / in.gamma_boost;
        for (int d = 0; d < 3; ++d) a.position[d] += (Z0_boost - a.Z0_lab) * a.nvec[d];
    }
    s = 1.0 / std::sqrt(in.p_X[0] * in.p_X[0] + in.p_X[1] * in.p_X[1] + in.p_X[2] * in.p_X[2]);
    for (int d = 0; d < 3; ++d) a.p_X[d] = in.p_X[d] * s;
    const double* n = a.nvec; const double* p = a.p_X;
    a.p_Y[0] = n[1] * p[2] - n[2] * p[1]; a.p_Y[1] = n[2] * p[0] - n[0] * p[2]; a.p_Y[2] = n[0] * p[1] - n[1] * p[0];
    for (int d = 0; d < 3; ++d) { a.u_X[d] = a.p_X[d]; a.u_Y[d] = a.p_Y[d]; }
    const double eps = dx[0] * 1.e-50;
    a.S_X = std::min(std::min(dx[0] / (std::abs(a.u_X[0]) + eps), dx[1] / (std::abs(a.u_X[1]) + eps)),
                     dx[2] / (std::abs(a.u_X[2]) + eps));
    a.S_Y = std::min(std::min(dx[0] / (std::abs(a.u_Y[0]) + eps), dx[1] / (std::abs(a.u_Y[1]) + eps)),
                     dx[2] / (std::abs(a.u_Y[2]) + eps));
    a.mobility = 0.05 / in.e_max;
    a.weight = EP0 / a.mobility;
    a.weight *= 1.0 * a.S_X * a.S_Y;
    if (boosted) a.mobility = a.mobility / in.gamma_boost;
    return a;
}

static bool strictly_inside(const double lo[3], const double hi[3], const double p[3]) {   // RealBox::contains
    return lo[0] < p[0] && p[0] < hi[0] && lo[1] < p[1] && p[1] < hi[1] && lo[2] < p[2] && p[2] < hi[2];
}

}  // namespace pic

using namespace pic;

// ---------------------------------------------------------------------------------------------
extern "C" int pic_apply_pec_field(const pic_fab F[3], int is_E, const pic_geom* g, const pic_boundaries* b,
                                   const int ng_fieldgather[3], void* stream) {
    bool any = false;
    for (int d = 0; d < 3; ++d) any = any || b->field_lo[d] == PIC_FIELD_PEC || b->field_hi[d] == PIC_FIELD_PEC;
    if (!any) return 0;
    for (int c = 0; c < 3; ++c) {
        PecFieldArgs a;
        a.F = make_view(F[c]);
        a.icomp = c; a.is_E = is_E ? 1 : 0;
        a.total = 1;
        for (int d = 0; d < 3; ++d) {
            PIC_REQUIRE(ng_fieldgather[d] <= F[c].ng[d], "pic_apply_pec_field: ng_fieldgather exceeds the allocated guard cells");
            a.stag[d] = F[c].stag[d];
            a.lo[d] = vlo(F[c], d) - ng_fieldgather[d];
            a.n[d] = vhi(F[c], d) + ng_fieldgather[d] - a.lo[d] + 1;
            a.ncell[d] = g->n_cell[d];
            a.pec_lo[d] = b->field_lo[d] == PIC_FIELD_PEC;
            a.pec_hi[d] = b->field_hi[d] == PIC_FIELD_PEC;
            a.total *= a.n[d];
        }
        PIC_LAUNCH(pec_field_kernel, pec_field_body, a, a.total, stream);
    }
    return launched_ok("pic_apply_pec_field") ? 0 : 1;
}

extern "C" int pic_apply_pec_current(const pic_fab J[3], const pic_geom* g, const pic_boundaries* b, void* stream) {
    for (int c = 0; c < 3; ++c) {
        PecCurrentArgs a;
        a.F = make_view(J[c]);
        a.icomp = c;
        a.total = 1;
        bool any = false;
        for (int d = 0; d < 3; ++d) {
            const bool plo = b->particle_lo[d] == PIC_PARTICLE_REFLECTING, phi = b->particle_hi[d] == PIC_PARTICLE_REFLECTING;
            a.refl[d][0] = plo || b->field_lo[d] == PIC_FIELD_PEC;
            a.refl[d][1] = phi || b->field_hi[d] == PIC_FIELD_PEC;
            any = any || a.refl[d][0] || a.refl[d][1];
            const bool tangent = (c != d);
            a.psign[d][0] = tangent ? (plo ? 1.0 : -1.0) : (plo ? -1.0 : 1.0);
            a.psign[d][1] = tangent ? (phi ? 1.0 : -1.0) : (phi ? -1.0 : 1.0);
            a.stag[d] = J[c].stag[d];
            a.mirrorfac[d][0] = 2 * 0 - (1 - J[c].stag[d]);
            a.mirrorfac[d][1] = 2 * g->n_cell[d] - (1 - J[c].stag[d]);
            a.lo[d] = vlo(J[c], d);
            a.n[d] = vhi(J[c], d) - a.lo[d] + 1;
            a.alo[d] = J[c].lo[d]; a.ahi[d] = J[c].hi[d];
            a.total *= a.n[d];
        }
        if (!any) return 0;
        PIC_LAUNCH(pec_current_kernel, pec_current_body, a, a.total, stream);
    }
    return launched_ok("pic_apply_pec_current") ? 0 : 1;
}

// tmp: scratch of the size of the fab (borrowed); the periodic refresh shiftMF does on its temporary
// is folded into the read (lwfa_body.cuh, shift_body).
extern "C" int pic_shift_fab(const pic_fab* f, double* tmp, const pic_geom* g, int num_shift, int dir,
                             double external_field, void* stream) {
    if (num_shift == 0) return 0;
    PIC_REQUIRE(dir >= 0 && dir < 3 && !g->periodic[dir], "pic_shift_fab: the moving-window direction must be non-periodic");
    const int mag = num_shift > 0 ? num_shift : -num_shift;
    PIC_REQUIRE(f->ng[dir] >= mag, "pic_shift_fab: %d guard cells < shift %d (shiftMF asserts the same)", f->ng[dir], mag);
    PIC_REQUIRE(tmp && tmp != f->p, "pic_shift_fab: needs a scratch array");
    dev_copy(tmp, f->p, sizeof(double) * (size_t)fab_size(*f), stream);
    pic_fab t = *f;
    t.p = tmp;
    ShiftArgs a;
    a.D = make_view(*f); a.S = make_view(t);
    a.dir = dir; a.shift = num_shift; a.ext = external_field;
    a.total = 1;
    for (int d = 0; d < 3; ++d) {
        a.lo[d] = f->lo[d]; a.n[d] = f->hi[d] - f->lo[d] + 1;
        a.per[d] = g->periodic[d]; a.vlo[d] = vlo(*f, d); a.vhi[d] = vhi(*f, d); a.ncell[d] = g->n_cell[d];
    }
    // adjBox = the allocated points beyond the DOMAIN face the window moves into: only a box that touches
    // that face has them; elsewhere those guard planes hold the neighbour's data (exchanged by the caller
    // with ng = |num_shift|, the FillBoundary of shiftMF's temporary, :499-505)
    const bool top = vhi(*f, dir) == g->n_cell[dir] - 1 + f->stag[dir], bottom = vlo(*f, dir) == 0;
    if (num_shift > 0) { a.n[dir] -= mag; a.adj_lo = vhi(*f, dir) + 1; a.adj_hi = top ? vhi(*f, dir) + f->ng[dir] : vhi(*f, dir); }
    else { a.lo[dir] += mag; a.n[dir] -= mag; a.adj_lo = bottom ? vlo(*f, dir) - f->ng[dir] : vlo(*f, dir); a.adj_hi = vlo(*f, dir) - 1; }
    // the planes just exchanged with the next slab count as valid for the folded periodic refresh
    // (FillBoundary reaches them: their periodic image is a valid point of the neighbour)
    if (num_shift > 0 && !top) a.vhi[dir] += mag;
    if (num_shift < 0 && !bottom) a.vlo[dir] -= mag;
    for (int d = 0; d < 3; ++d)
        PIC_REQUIRE(d == dir || !g->periodic[d] || vhi(*f, d) - vlo(*f, d) + 1 - f->stag[d] == g->n_cell[d],
                    "pic_shift_fab: the box must span the periodic direction %d (slabs along the moving direction)", d);
    for (int d = 0; d < 3; ++d) a.total *= a.n[d];
    PIC_LAUNCH(shift_kernel, shift_body, a, a.total, stream);
    return launched_ok("pic_shift_fab") ? 0 : 1;
}

// ---------------------------------------------------------------------------------------------
extern "C" int pic_laser_antenna_info(const pic_laser_antenna* prm, const double dx[3], double out[4]) {
    PIC_REQUIRE(prm->e_max > 0 && prm->wavelength > 0, "pic_laser_antenna: e_max and wavelength must be > 0");
    PIC_REQUIRE(!(prm->gamma_boost > 1.) || (prm->beta_boost > 0. && prm->beta_boost < 1.),
                "pic_laser_antenna: gamma_boost > 1 needs 0 < beta_boost < 1");
    const AntennaSetup a = antenna_setup(*prm, dx);
    const double dp = a.nvec[0] * a.p_X[0] + a.nvec[1] * a.p_X[1] + a.nvec[2] * a.p_X[2];
    PIC_REQUIRE(std::abs(dp) < 1.0e-14, "Laser plane vector is not perpendicular to the main polarization vector");
    out[0] = a.S_X; out[1] = a.S_Y; out[2] = a.mobility; out[3] = a.weight;
    return 0;
}

// LaserParticleContainer::InitData(lev) (:369-560): HOST arrays (the reference builds host vectors and
// hands them to AddNParticles).  Returns the number of particles, or -1 when capacity is too small.
extern "C" long pic_laser_antenna_particles(const pic_laser_antenna* prm, const double dx[3], const double box_lo[3],
                                            const double box_hi[3], double* x, double* y, double* z, double* w,
                                            long capacity) {
    const AntennaSetup a = antenna_setup(*prm, dx);
    const double* pos0 = a.position;
    int plane_lo[2] = {std::numeric_limits<int>::max(), std::numeric_limits<int>::max()};
    int plane_hi[2] = {std::numeric_limits<int>::min(), std::numeric_limits<int>::min()};
    for (int c = 0; c < 8; ++c) {
        const double cx = (c & 1) ? box_hi[0] : box_lo[0], cy = (c & 2) ? box_hi[1] : box_lo[1],
                     cz = (c & 4) ? box_hi[2] : box_lo[2];
        const double px = a.u_X[0] * (cx - pos0[0]) + a.u_X[1] * (cy - pos0[1]) + a.u_X[2] * (cz - pos0[2]);
        const double py = a.u_Y[0] * (cx - pos0[0]) + a.u_Y[1] * (cy - pos0[1]) + a.u_Y[2] * (cz - pos0[2]);
        const int i = static_cast<int>(px / a.S_X), j = static_cast<int>(py / a.S_Y);
        plane_lo[0] = std::min(plane_lo[0], i); plane_lo[1] = std::min(plane_lo[1], j);
        plane_hi[0] = std::max(plane_hi[0], i); plane_hi[1] = std::max(plane_hi[1], j);
    }
    long n = 0;
    for (int j = plane_lo[1]; j <= plane_hi[1]; ++j)
        for (int i = plane_lo[0]; i <= plane_hi[0]; ++i) {
            const double pos[3] = {
                pos0[0] + (a.S_X * (double(i) + 0.5)) * a.u_X[0] + (a.S_Y * (double(j) + 0.5)) * a.u_Y[0],
                pos0[1] + (a.S_X * (double(i) + 0.5)) * a.u_X[1] + (a.S_Y * (double(j) + 0.5)) * a.u_Y[1],
                pos0[2] + (a.S_X * (double(i) + 0.5)) * a.u_X[2] + (a.S_Y * (double(j) + 0.5)) * a.u_Y[2]};
            if (!strictly_inside(box_lo, box_hi, pos)) continue;
            if (x) {
                if (n + 2 > capacity) return -1;
                for (int k = 0; k < 2; ++k) { x[n + k] = pos[0]; y[n + k] = pos[1]; z[n + k] = pos[2]; }
                w[n] = a.weight; w[n + 1] = -a.weight;
            }
            n += 2;
        }
    return n;
}

// One step of the antenna particles at time t (beginning of the step), LaserParticleContainer::Evolve
// :614-626: plane coordinates, Gaussian amplitude, u and x update.
extern "C" int pic_laser_antenna_push(const pic_laser_antenna* prm, const double dx[3], const pic_soa* p,
                                      double t_sim, double dt, void* stream) {
    if (p->np == 0) return 0;
    using cplx = std::complex<double>;
    const AntennaSetup s = antenna_setup(*prm, dx);
    // boosted frame: the profile is evaluated at the lab time of the antenna plane (:573-579)
    const double t = s.gamma_boost > 1. ? 1. / s.gamma_boost * t_sim + s.beta_boost * s.Z0_lab / C_LIGHT : t_sim;
    const cplx I(0.0, 1.0);
    constexpr double pi = 3.14159265358979323846;
    const double k0 = 2.0 * pi / prm->wavelength;
    const double inv_tau2 = 1.0 / (prm->duration * prm->duration);
    const double oscillation_phase = k0 * C_LIGHT * (t - prm->t_peak) + prm->phi0;
    const cplx diffract_factor = 1.0 + I * prm->focal_distance * 2.0 / (k0 * prm->waist * prm->waist);
    const cplx inv_complex_waist_2 = 1.0 / (prm->waist * prm->waist * diffract_factor);
    const cplx t_prefactor = prm->e_max * std::exp(I * oscillation_phase);
    const cplx prefactor = t_prefactor / diffract_factor;
    // zeta = beta = phi2 = 0: stretch_factor = 1 and the exponent does not depend on the particle
    const cplx arg = (t - prm->t_peak);
    const cplx stc_exponent = inv_tau2 * (arg * arg);
    const cplx stc = prefactor * std::exp(-stc_exponent);
    LaserArgs a;
    a.P = make_soa(*p, 0);
    a.np = p->np;
    for (int d = 0; d < 3; ++d) { a.pos[d] = s.position[d]; a.uX[d] = s.u_X[d]; a.uY[d] = s.u_Y[d]; a.pX[d] = s.p_X[d]; a.nvec[d] = s.nvec[d]; }
    a.gamma_boost = s.gamma_boost; a.beta_boost = s.beta_boost;
    a.stc_re = stc.real(); a.stc_im = stc.imag();
    a.icw_re = inv_complex_waist_2.real(); a.icw_im = inv_complex_waist_2.imag();
    a.mobility = s.mobility; a.dt = dt;
    PIC_LAUNCH(laser_kernel, laser_body, a, a.np, stream);
    return launched_ok("pic_laser_antenna_push") ? 0 : 1;
}

// Multi-rank antennas are replicated on every rank (a few thousand particles); each rank deposits
// only the particles inside its own box: w_out = w inside [own_lo, own_hi), 0 elsewhere.
namespace pic {
struct OwnedArgs { const double* x; const double* y; const double* z; const double* w; double* w_out; long np; double lo[3], hi[3]; };
PIC_HD void owned_body(long ip, const OwnedArgs& a) {
    const bool in = a.x[ip] >= a.lo[0] && a.x[ip] < a.hi[0] && a.y[ip] >= a.lo[1] && a.y[ip] < a.hi[1] &&
                    a.z[ip] >= a.lo[2] && a.z[ip] < a.hi[2];
    a.w_out[ip] = in ? a.w[ip] : 0.0;
}
__global__ void owned_kernel(OwnedArgs a) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.np) owned_body(t, a);
}
}  // namespace pic
extern "C" int pic_particles_owned_weights(const pic_soa* p, const double own_lo[3], const double own_hi[3],
                                           double* w_out, void* stream) {
    if (p->np == 0) return 0;
    OwnedArgs a;
    a.x = p->x; a.y = p->y; a.z = p->z; a.w = p->w; a.w_out = w_out; a.np = p->np;
    for (int d = 0; d < 3; ++d) { a.lo[d] = own_lo[d]; a.hi[d] = own_hi[d]; }
    PIC_LAUNCH(owned_kernel, owned_body, a, a.np, stream);
    return launched_ok("pic_particles_owned_weights") ? 0 : 1;
}

// ---------------------------------------------------------------------------------------------
// AddPlasma for NUniformPerCell / constant density / at rest, one tile = the rank's whole domain box.
// Particles are appended after p->np (ids first_id, first_id+1, ... in creation order).
// Returns the number of particles added (>= 0) or -1 on error.
extern "C" long pic_add_plasma(const pic_plasma_injector* inj, const pic_geom* g, const double cell_size[3],
                               const int box_lo[3], const int box_hi[3], const double part_lo[3],
                               const double part_hi[3], const pic_soa* p, long capacity, uint64_t first_id,
                               double t, void* stream) {
    const bool boosted = inj->gamma_boost > 1.;
    if (boosted && !(inj->beta_boost > 0. && inj->beta_boost < 1.)) { fail("pic_add_plasma: gamma_boost > 1 needs 0 < beta_boost < 1"); return -1; }
    const double gamma_boost = boosted ? inj->gamma_boost : 1.0, beta_boost = boosted ? inj->beta_boost : 0.0;
    // applyBallisticCorrection (:138-148) for a plasma at rest in the lab (betaz_bulk = 0): the lab-frame z
    // the bounds are tested at; the identity in the lab frame
    auto lab = [&](int d, double z) {
        return d == 2 ? gamma_boost * (z * (1.0 - beta_boost * 0.0) - C_LIGHT * t * (0.0 - beta_boost)) : z;
    };
    double dx[3], tile_lo[3], tile_hi[3], ov_lo[3], ov_hi[3];
    int nov[3];
    for (int d = 0; d < 3; ++d) {
        // geom.CellSize(): fixed at start-up; the moving window only translates prob_lo / prob_hi
        dx[d] = cell_size ? cell_size[d] : (g->prob_hi[d] - g->prob_lo[d]) / g->n_cell[d];
        // tile_realbox = RealBox(tile_box, dx, prob_lo) (WarpX::getRealBox, Source/WarpX.cpp:2852-2857)
        tile_lo[d] = g->prob_lo[d] + dx[d] * (box_lo ? box_lo[d] : 0);
        tile_hi[d] = g->prob_lo[d] + dx[d] * ((box_hi ? box_hi[d] : g->n_cell[d] - 1) + 1);
        // find_overlap (Particles/AddPlasmaUtilities.cpp:12-43)
        if (tile_lo[d] <= part_hi[d]) {
            const double adj = std::floor((tile_lo[d] - part_lo[d]) / dx[d]);
            ov_lo[d] = part_lo[d] + std::max(adj, 0.0) * dx[d];
        } else return 0;
        if (tile_hi[d] >= part_lo[d]) {
            const double adj = std::floor((part_hi[d] - tile_hi[d]) / dx[d]);
            ov_hi[d] = part_hi[d] - std::max(adj, 0.0) * dx[d];
        } else return 0;
        nov[d] = int(std::round((ov_hi[d] - ov_lo[d]) / dx[d]));
        if (nov[d] <= 0) return 0;
    }
    if (inj->density <= 0) return 0;
    InjectArgs a;
    long count = 1;
    a.total = (long)inj->ppc[0] * inj->ppc[1] * inj->ppc[2];
    for (int d = 0; d < 3; ++d) {
        // Along d, which lattice points m = cell*ppc + in-cell index survive every test of AddPlasma:
        // the cell overlaps the plasma bounds (InjectorPosition.H:228-233) and one of its three test
        // abscissae lies inside them (:1032-1049), the position lies inside the tile's RealBox
        // (:1141-1156) and inside the bounds (:1189-1197).  All tests are separable per direction.
        const int ppc = inj->ppc[d];
        if (ppc < 1) { fail("pic_add_plasma: num_particles_per_cell_each_dim must be >= 1"); return -1; }
        int m_lo = -1, m_hi = -2;
        bool closed = false;
        for (int cell = 0; cell < nov[d]; ++cell) {
            const double lo = lab(d, ov_lo[d] + (cell + 0.0) * dx[d]), hi = lab(d, ov_lo[d] + (cell + 1.0) * dx[d]);   // :1017-1022
            const bool overlaps = inj->bound_lo[d] <= hi && inj->bound_hi[d] >= lo;
            const double tp[3] = {lo, (lo + hi) / 2.0, hi};
            bool any = false;
            for (int q = 0; q < 3; ++q) any = any || (tp[q] < inj->bound_hi[d] && tp[q] >= inj->bound_lo[d]);
            for (int ip = 0; ip < ppc; ++ip) {
                const double r = (0.5 + ip) / ppc;
                const double pos = ov_lo[d] + (cell + r) * dx[d];
                const double pos_lab = lab(d, pos);                                 // z0 / z0_lab (:1184,1211)
                const bool ok = overlaps && any && tile_lo[d] < pos && pos < tile_hi[d] &&
                                pos_lab < inj->bound_hi[d] && pos_lab >= inj->bound_lo[d];
                const int m = cell * ppc + ip;
                if (ok) {
                    if (closed) { fail("pic_add_plasma: the admitted lattice points along %d are not contiguous", d); return -1; }
                    if (m_lo < 0) m_lo = m;
                    m_hi = m;
                } else if (m_lo >= 0) closed = true;
            }
        }
        if (m_lo < 0) return 0;
        a.m_lo[d] = m_lo; a.m_hi[d] = m_hi;
        a.ppc[d] = ppc;
        a.c0[d] = m_lo / ppc;
        a.nc[d] = m_hi / ppc - a.c0[d] + 1;
        a.ov_lo[d] = ov_lo[d]; a.dx[d] = dx[d];
        count *= (m_hi - m_lo + 1);
        a.total *= a.nc[d];
    }
    if (p == nullptr) return count;                      // count only (ranks that do not own the slab keep the id counter in step)
    if (p->np + count > capacity) { fail("pic_add_plasma: %ld + %ld particles exceed the capacity %ld", (long)p->np, count, capacity); return -1; }
    a.P = make_soa(*p, p->np);
    a.id = p->idcpu ? p->idcpu + p->np : nullptr;
    a.id0 = first_id;
    const long pcount = (long)inj->ppc[0] * inj->ppc[1] * inj->ppc[2];
    double dens = inj->density, uz = 0.0;
    if (boosted) {                                        // Lorentz transform of a plasma at rest (:1232-1246)
        const double gamma_lab = std::sqrt(1. + (0.0 * 0.0 + 0.0 * 0.0 + uz * uz));
        const double betaz_lab = uz / (gamma_lab);
        dens = gamma_boost * dens * (1.0 - beta_boost * betaz_lab);
        uz = gamma_boost * (uz - beta_boost * gamma_lab);
    }
    a.uz = uz * C_LIGHT;                                  // :1275-1277
    a.weight = dens;
    a.weight *= dx[0] * dx[1] * dx[2] / pcount;           // compute_scale_fac_volume (AddPlasmaUtilities.H:73-77)
    PIC_LAUNCH(inject_kernel, inject_body, a, a.total, stream);
    return launched_ok("pic_add_plasma") ? count : -1;
}

// ---------------------------------------------------------------------------------------------
// Particle boundaries, step 1: reflect at reflecting faces, list the particles lost at absorbing
// faces.  work = 4 + 4*cap ints (device): work[0] = number lost (keeps counting beyond cap),
// work[1..3] = scratch, then list[cap], holes[cap], srcs[cap], tailflag[cap].
extern "C" long pic_particles_boundary_workspace_ints(int cap) { return 4 + 4 * (long)cap; }

extern "C" int pic_particles_boundary_mark(const pic_soa* p, const pic_geom* g, const pic_boundaries* b,
                                           int* work, int cap, void* stream) {
    dev_zero(work, 4 * sizeof(int), stream);
    if (p->np == 0) return 0;
    BoundaryArgs a;
    a.P = make_soa(*p, 0);
    a.np = p->np;
    bool any = false;
    for (int d = 0; d < 3; ++d) {
        a.lo[d] = g->prob_lo[d]; a.hi[d] = g->prob_hi[d];
        a.bc_lo[d] = b->particle_lo[d]; a.bc_hi[d] = b->particle_hi[d];
        any = any || a.bc_lo[d] != PIC_PARTICLE_PERIODIC || a.bc_hi[d] != PIC_PARTICLE_PERIODIC;
    }
    if (!any) return 0;
    a.count = work; a.list = work + 4; a.cap = cap;
    PIC_LAUNCH(boundary_mark_kernel, boundary_mark_body, a, a.np, stream);
    return launched_ok("pic_particles_boundary_mark") ? 0 : 1;
}

// Step 2, after the host has read n_lost = work[0]: drop the listed particles; the new count is
// p->np - n_lost (what AMReX Redistribute leaves after ApplyBoundaryConditions invalidated them).
extern "C" int pic_particles_boundary_compact(const pic_soa* p, int* work, int cap, int n_lost, void* stream) {
    if (n_lost == 0) return 0;
    PIC_REQUIRE(n_lost <= cap, "pic_particles_boundary_compact: %d particles lost in one step exceed the list capacity %d", n_lost, cap);
    PIC_REQUIRE(n_lost <= p->np, "pic_particles_boundary_compact: inconsistent count");
    CompactArgs a;
    a.P = make_soa(*p, 0);
    a.id = p->idcpu;
    a.list = work + 4; a.holes = work + 4 + cap; a.srcs = work + 4 + 2 * (long)cap; a.tailflag = work + 4 + 3 * (long)cap;
    a.nh = work + 1; a.ns = work + 2;
    a.m = p->np - n_lost;
    a.n_lost = n_lost;
    dev_zero(a.tailflag, sizeof(int) * (size_t)n_lost, stream);
    PIC_LAUNCH(compact_split_kernel, compact_split_body, a, (long)n_lost, stream);
    PIC_LAUNCH(compact_tail_kernel, compact_tail_body, a, (long)n_lost, stream);
    PIC_LAUNCH(compact_move_kernel, compact_move_body, a, (long)n_lost, stream);
    return launched_ok("pic_particles_boundary_compact") ? 0 : 1;
}
