// Per-thread bodies of the kernels that the laser-wakefield decks add to the periodic PIC step
// (SURVEY.md 8f rank 3): PEC walls, moving-window shift, laser antenna, continuous plasma injection,
// absorbing / reflecting particle boundaries.  Each body takes the linear thread id and a POD
// argument block; the __global__ wrappers live in lwfa.cu.  The bodies are __host__ __device__ so
// that tests/host_harness can run the SAME code over the same index space on the host (a check of
// the per-thread logic where no GPU is available; never part of the product path).
//
// Reference (paths relative to Source/ of ECP-WarpX/WarpX):
//   pec_field_body        <- ::SetEfieldOnPEC / ::SetBfieldOnPEC     BoundaryConditions/WarpX_PEC.cpp:120-190,252-318
//   pec_current_body      <- ::SetRhoOrJfieldFromPEC                 BoundaryConditions/WarpX_PEC.cpp:340-395
//   shift_body            <- WarpX::shiftMF                          Utils/WarpXMovingWindow.cpp:508-600
//   laser_body            <- GaussianLaserProfile::fill_amplitude    Laser/LaserProfilesImpl/LaserProfileGaussian.cpp:145-160
//                            LaserParticleContainer::update_laser_particle  Particles/LaserParticleContainer.cpp:905-949
//   inject_body           <- PhysicalParticleContainer::AddPlasma    Particles/PhysicalParticleContainer.cpp:1120-1300
//   boundary_mark_body    <- ApplyParticleBoundaries::apply_boundary Particles/ParticleBoundaries_K.H:21-75
#ifndef PIC_LWFA_BODY_CUH_
#define PIC_LWFA_BODY_CUH_

#include "pic_common.cuh"

namespace pic {

#define PIC_HD __host__ __device__ __forceinline__
#define PIC_AT(F, i, j, k) (F).p[(F).off((i), (j), (k))]

PIC_HD void decode3(long t, const int n[3], const int lo[3], int idx[3]) {
    idx[0] = lo[0] + (int)(t % n[0]);
    idx[1] = lo[1] + (int)((t / n[0]) % n[1]);
    idx[2] = lo[2] + (int)(t / ((long)n[0] * n[1]));
}

// ---------------------------------------------------------------------------------------------
// PEC on one component of E (is_E) or B: region = valid points grown by ng_FieldGather.
struct PecFieldArgs {
    FabView F;
    int stag[3], icomp, is_E;
    int lo[3], n[3];                 // region
    int ncell[3], pec_lo[3], pec_hi[3];
    long total;
};

PIC_HD void pec_field_body(long t, const PecFieldArgs& a) {
    int ijk[3];
    decode3(t, a.n, a.lo, ijk);
    int mir[3] = {ijk[0], ijk[1], ijk[2]};
    bool on_pec = false, guard = false;
    double sign = 1.0;
    for (int idim = 0; idim < 3; ++idim)
        for (int iside = 0; iside < 2; ++iside) {
            if (!(iside == 0 ? a.pec_lo[idim] : a.pec_hi[idim])) continue;
            // E: tangential components flip; B: the normal component flips
            const bool flips = a.is_E ? (a.icomp != idim) : (a.icomp == idim);
            const int dom_hi = a.ncell[idim] - 1;
            const int ig = (iside == 0) ? (0 - ijk[idim]) : (ijk[idim] - (dom_hi + a.stag[idim]));
            if (ig == 0) {
                if (flips && a.stag[idim] == 1) on_pec = true;
            } else if (ig > 0) {
                mir[idim] = (iside == 0) ? (0 + ig - (1 - a.stag[idim])) : (dom_hi + 1 - ig);
                guard = true;
                if (flips) sign *= -1.0;
            }
        }
    if (on_pec) PIC_AT(a.F, ijk[0], ijk[1], ijk[2]) = 0.0;
    else if (guard) PIC_AT(a.F, ijk[0], ijk[1], ijk[2]) = sign * PIC_AT(a.F, mir[0], mir[1], mir[2]);
}

// ---------------------------------------------------------------------------------------------
// Reflective / PEC boundary on one component of J: loop over the valid points.
struct PecCurrentArgs {
    FabView F;
    int stag[3], icomp;
    int lo[3], n[3];                 // valid points
    int alo[3], ahi[3];              // allocated bounds (fabbox)
    int refl[3][2], mirrorfac[3][2];
    double psign[3][2];
    long total;
};

PIC_HD void pec_current_body(long t, const PecCurrentArgs& a) {
    int ijk[3];
    decode3(t, a.n, a.lo, ijk);
    double* self = &PIC_AT(a.F, ijk[0], ijk[1], ijk[2]);
    // 1) the point receives what was deposited in its mirror guard point
    for (int idim = 0; idim < 3; ++idim)
        for (int iside = 0; iside < 2; ++iside) {
            if (!a.refl[idim][iside]) continue;
            int mir[3] = {ijk[0], ijk[1], ijk[2]};
            mir[idim] = a.mirrorfac[idim][iside] - ijk[idim];
            if (mir[idim] == ijk[idim]) *self = 0.0;
            else if (mir[idim] >= a.alo[idim] && mir[idim] <= a.ahi[idim])
                *self += a.psign[idim][iside] * PIC_AT(a.F, mir[0], mir[1], mir[2]);
        }
    // 2) the guard point gets the image of the interior value
    for (int idim = 0; idim < 3; ++idim)
        for (int iside = 0; iside < 2; ++iside) {
            if (!a.refl[idim][iside]) continue;
            int mir[3] = {ijk[0], ijk[1], ijk[2]};
            mir[idim] = a.mirrorfac[idim][iside] - ijk[idim];
            if (mir[idim] != ijk[idim] && mir[idim] >= a.alo[idim] && mir[idim] <= a.ahi[idim])
                PIC_AT(a.F, mir[0], mir[1], mir[2]) = (a.icomp != idim) ? -*self : *self;
        }
}

// ---------------------------------------------------------------------------------------------
// Moving-window shift: D(i,j,k) = S(i,j,k + shift) over the fab box shortened at the far end; S is a
// copy of the array before the shift.  The allocated points of S beyond the domain face the window
// moves into count as `ext` (:508-556).  shiftMF refreshes its temporary with FillBoundary(ng = 1 off
// the moving direction, :499-505) before shifting; here that refresh is folded into the read: a
// source point in the first guard layer of a periodic direction whose periodic image is a valid
// point reads the image.
struct ShiftArgs {
    FabView D, S;
    int lo[3], n[3];                 // destination box
    int dir, shift;
    int adj_lo, adj_hi;              // index range along dir that holds `ext`
    int per[3], vlo[3], vhi[3], ncell[3];
    double ext;
    long total;
};

PIC_HD void shift_body(long t, const ShiftArgs& a) {
    int ijk[3];
    decode3(t, a.n, a.lo, ijk);
    int src[3] = {ijk[0], ijk[1], ijk[2]};
    src[a.dir] += a.shift;
    if (src[a.dir] >= a.adj_lo && src[a.dir] <= a.adj_hi) { PIC_AT(a.D, ijk[0], ijk[1], ijk[2]) = a.ext; return; }
    // FillBoundary(ng_mw) touches a point when it lies within one layer of the valid points along
    // the periodic directions and on a valid index along the others
    bool fillable = true, in_guard = false;
    int img[3] = {src[0], src[1], src[2]};
    for (int d = 0; d < 3; ++d) {
        if (src[d] >= a.vlo[d] && src[d] <= a.vhi[d]) continue;
        if (a.per[d] && d != a.dir && (src[d] == a.vlo[d] - 1 || src[d] == a.vhi[d] + 1)) {
            in_guard = true;
            img[d] = src[d] < a.vlo[d] ? src[d] + a.ncell[d] : src[d] - a.ncell[d];
        } else fillable = false;
    }
    if (fillable && in_guard) { src[0] = img[0]; src[1] = img[1]; src[2] = img[2]; }
    PIC_AT(a.D, ijk[0], ijk[1], ijk[2]) = PIC_AT(a.S, src[0], src[1], src[2]);
}

// ---------------------------------------------------------------------------------------------
// Laser antenna particles: amplitude at the particle, velocity along the polarisation, position push.
// stc = prefactor * exp(-stc_exponent) (the same for every particle when zeta = beta = phi2 = 0) and
// icw = 1 / (w0^2 * diffract_factor) are evaluated on the host like the reference does (:104-140).
struct LaserArgs {
    SoaView P;
    long np;
    double pos[3], uX[3], uY[3], pX[3];
    double stc_re, stc_im, icw_re, icw_im;
    double mobility, dt;
    double nvec[3], gamma_boost, beta_boost;     // boosted frame (gamma_boost = 1, beta_boost = 0 in the lab)
};

PIC_HD void laser_body(long ip, const LaserArgs& a) {
    const double x = a.P.x[ip], y = a.P.y[ip], z = a.P.z[ip];
    const double Xp = a.uX[0] * (x - a.pos[0]) + a.uX[1] * (y - a.pos[1]) + a.uX[2] * (z - a.pos[2]);
    const double Yp = a.uY[0] * (x - a.pos[0]) + a.uY[1] * (y - a.pos[1]) + a.uY[2] * (z - a.pos[2]);
    // exp_argument = -(Xp^2 + Yp^2) * icw ; amplitude = Re(stc * exp(exp_argument))
    const double r2 = -(Xp * Xp + Yp * Yp);
    const double er = r2 * a.icw_re, ei = r2 * a.icw_im;
    const double mag = exp(er);
    const double cr = mag * cos(ei), ci = mag * sin(ei);
    const double amplitude = a.stc_re * cr - a.stc_im * ci;
    const double sign_charge = (a.P.w[ip] > 0) ? -1.0 : 1.0;
    const double v_over_c = sign_charge * a.mobility * amplitude;
    double vx = C_LIGHT * v_over_c * a.pX[0];
    double vy = C_LIGHT * v_over_c * a.pX[1];
    double vz = C_LIGHT * v_over_c * a.pX[2];
    if (a.gamma_boost > 1.) {                    // the antenna drifts with the lab (LaserParticleContainer.cpp:908-912)
        vx -= C_LIGHT * a.beta_boost * a.nvec[0];
        vy -= C_LIGHT * a.beta_boost * a.nvec[1];
        vz -= C_LIGHT * a.beta_boost * a.nvec[2];
    }
    const double gamma = a.gamma_boost / sqrt(1. - v_over_c * v_over_c);    // :914-915
    a.P.ux[ip] = gamma * vx; a.P.uy[ip] = gamma * vy; a.P.uz[ip] = gamma * vz;
    a.P.x[ip] = x + vx * a.dt; a.P.y[ip] = y + vy * a.dt; a.P.z[ip] = z + vz * a.dt;
}

// ---------------------------------------------------------------------------------------------
// Plasma injection on the NUniformPerCell lattice.  Candidates = cells [c0, c0+nc) of the overlap
// box x in-cell index; along each direction the lattice points m = cell*ppc + in-cell index that
// pass every test of the reference form one interval [m_lo, m_hi] (found on the host), so the
// output slot of a particle has a closed form: cells i-fastest, in-cell index ascending -- the
// order in which the reference's loops create them.
struct InjectArgs {
    SoaView P;                       // already offset to the first free slot
    uint64_t* id;                    // idem (may be null)
    uint64_t id0;
    double ov_lo[3], dx[3];
    int ppc[3], c0[3], nc[3], m_lo[3], m_hi[3];
    double weight, uz;               // uz = -gamma_boost beta_boost c in a boosted frame, 0 in the lab
    long total;
};

// lo + (cell + r) * dx exactly as the reference's host/CPU build evaluates getCellCoords: a product
// rounded to double, then a sum (no fused multiply-add), so that the particle positions a moving
// window injects are bit-identical to the CPU reference's.
PIC_HD double cell_coord(double lo, double cr, double dx) {
#ifdef __CUDA_ARCH__
    return __dadd_rn(lo, __dmul_rn(cr, dx));
#else
    return lo + cr * dx;
#endif
}

PIC_HD int inject_prefix(int cell, int ppc, int m_lo, int m_hi) {   // valid lattice points below `cell`
    const int v = cell * ppc - m_lo, M = m_hi - m_lo + 1;
    return v < 0 ? 0 : (v > M ? M : v);
}

PIC_HD void inject_body(long t, const InjectArgs& a) {
    const int nppc = a.ppc[0] * a.ppc[1] * a.ppc[2];
    const int i_part = (int)(t % nppc);
    const long cell = t / nppc;
    const int iv[3] = {a.c0[0] + (int)(cell % a.nc[0]), a.c0[1] + (int)((cell / a.nc[0]) % a.nc[1]),
                       a.c0[2] + (int)(cell / ((long)a.nc[0] * a.nc[1]))};
    // InjectorPositionRegular::getPositionUnitBox (Initialization/InjectorPosition.H:99-107)
    const int ny = a.ppc[1], nz = a.ppc[2];
    const int ixp = i_part / (ny * nz);
    const int izp = (i_part - ixp * (ny * nz)) / ny;
    const int iyp = (i_part - ixp * (ny * nz)) - ny * izp;
    const int ip3[3] = {ixp, iyp, izp};
    int rank[3], cnt[3], pre[3], M[3];
    for (int d = 0; d < 3; ++d) {
        const int m = iv[d] * a.ppc[d] + ip3[d];
        if (m < a.m_lo[d] || m > a.m_hi[d]) return;
        pre[d] = inject_prefix(iv[d], a.ppc[d], a.m_lo[d], a.m_hi[d]);
        cnt[d] = inject_prefix(iv[d] + 1, a.ppc[d], a.m_lo[d], a.m_hi[d]) - pre[d];
        const int first = iv[d] * a.ppc[d] > a.m_lo[d] ? iv[d] * a.ppc[d] : a.m_lo[d];
        rank[d] = m - first;
        M[d] = a.m_hi[d] - a.m_lo[d] + 1;
    }
    const long cell_off = (long)pre[2] * M[1] * M[0] + (long)cnt[2] * ((long)pre[1] * M[0] + (long)cnt[1] * pre[0]);
    const long slot = cell_off + ((long)rank[0] * cnt[2] + rank[2]) * cnt[1] + rank[1];
    const double r[3] = {(0.5 + ixp) / a.ppc[0], (0.5 + iyp) / a.ppc[1], (0.5 + izp) / a.ppc[2]};
    a.P.x[slot] = cell_coord(a.ov_lo[0], iv[0] + r[0], a.dx[0]);    // getCellCoords (:151-175)
    a.P.y[slot] = cell_coord(a.ov_lo[1], iv[1] + r[1], a.dx[1]);
    a.P.z[slot] = cell_coord(a.ov_lo[2], iv[2] + r[2], a.dx[2]);
    a.P.w[slot] = a.weight;
    a.P.ux[slot] = 0.0; a.P.uy[slot] = 0.0; a.P.uz[slot] = a.uz;
    if (a.id) a.id[slot] = a.id0 + (uint64_t)slot;
}

// ---------------------------------------------------------------------------------------------
// Particle boundaries on the non-periodic faces: reflecting -> mirrored, normal momentum flipped;
// absorbing -> the index is appended to `list` (count[0] keeps counting beyond cap).
struct BoundaryArgs {
    SoaView P;
    long np;
    double lo[3], hi[3];
    int bc_lo[3], bc_hi[3];          // PIC_PARTICLE_*
    int* count;
    int* list;
    int cap;
};

PIC_HD bool boundary_body(long ip, const BoundaryArgs& a) {          // returns "lost"
    double* X[3] = {a.P.x, a.P.y, a.P.z};
    double* U[3] = {a.P.ux, a.P.uy, a.P.uz};
    bool lost = false;
    for (int d = 0; d < 3; ++d) {
        if (a.bc_lo[d] == PIC_PARTICLE_PERIODIC && a.bc_hi[d] == PIC_PARTICLE_PERIODIC) continue;
        const double x = X[d][ip];
        if (x < a.lo[d]) {
            if (a.bc_lo[d] == PIC_PARTICLE_ABSORBING) lost = true;
            else if (a.bc_lo[d] == PIC_PARTICLE_REFLECTING) { X[d][ip] = 2 * a.lo[d] - x; U[d][ip] = -U[d][ip]; }
        } else if (x > a.hi[d]) {
            if (a.bc_hi[d] == PIC_PARTICLE_ABSORBING) lost = true;
            else if (a.bc_hi[d] == PIC_PARTICLE_REFLECTING) { X[d][ip] = 2 * a.hi[d] - x; U[d][ip] = -U[d][ip]; }
        }
    }
    return lost;
}

}  // namespace pic
#endif
