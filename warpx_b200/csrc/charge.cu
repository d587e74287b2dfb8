// Charge deposition and the PEC / reflecting boundary of rho -- the `rho` diagnostic of a plotfile
// (outside the per-step path of the explicit FDTD loop: WarpX deposits rho only for diagnostics there).
//
// Replaces (paths relative to Source/ of ECP-WarpX/WarpX):
//   pic_deposit_charge  <- WarpXParticleContainer::DepositCharge (Particles/WarpXParticleContainer.cpp:890-1216)
//                          -> doChargeDepositionShapeN<N> (Particles/Deposition/ChargeDeposition.H:37-157)
//   pic_apply_pec_rho   <- PEC::ApplyReflectiveBoundarytoRhofield (BoundaryConditions/WarpX_PEC.cpp:624-699)
// Order-agnostic: one thread per particle, fp64 red.global per grid point (the reference's GPU strategy).
// Bodies are __host__ __device__ (see harness_launch.cuh).
#include "pic_common.cuh"
#include "harness_launch.cuh"

namespace pic {

struct ChargeArgs {
    const double* x; const double* y; const double* z; const double* w;
    long np;
    FabView R;
    int stag[3], lo[3];
    double dinv[3], xyzmin[3];
    double q_invvol;
};

template <int N>
PIC_HD void charge_body(long ip, const ChargeArgs& a) {
    const double wq = a.q_invvol * a.w[ip];                       // q * w * invvol (:66)
    double s[3][N + 1];
    int j0[3];
    const double pos[3] = {(a.x[ip] - a.xyzmin[0]) * a.dinv[0], (a.y[ip] - a.xyzmin[1]) * a.dinv[1],
                           (a.z[ip] - a.xyzmin[2]) * a.dinv[2]};
    for (int d = 0; d < 3; ++d) j0[d] = shape_factor<N>(s[d], a.stag[d] ? pos[d] : pos[d] - 0.5);   // :91-127
    for (int iz = 0; iz <= N; ++iz)                                // :146-155
        for (int iy = 0; iy <= N; ++iy)
            for (int ix = 0; ix <= N; ++ix)
                real_add(&a.R.p[a.R.off(a.lo[0] + j0[0] + ix, a.lo[1] + j0[1] + iy, a.lo[2] + j0[2] + iz)],
                         s[0][ix] * s[1][iy] * s[2][iz] * wq);
}
template <int N>
__global__ void charge_kernel(ChargeArgs a) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.np) charge_body<N>(t, a);
}

struct PecRhoArgs {
    FabView F;
    int lo[3], n[3], alo[3], ahi[3];
    int refl[3][2], mirrorfac[3][2];
    double psign[3][2];
    long total;
};
PIC_HD void pec_rho_body(long t, const PecRhoArgs& a) {
    int ijk[3];
    ijk[0] = a.lo[0] + (int)(t % a.n[0]);
    ijk[1] = a.lo[1] + (int)((t / a.n[0]) % a.n[1]);
    ijk[2] = a.lo[2] + (int)(t / ((long)a.n[0] * a.n[1]));
    double* self = &a.F.p[a.F.off(ijk[0], ijk[1], ijk[2])];
    for (int idim = 0; idim < 3; ++idim)                           // ::SetRhoOrJfieldFromPEC, WarpX_PEC.cpp:354-374
        for (int iside = 0; iside < 2; ++iside) {
            if (!a.refl[idim][iside]) continue;
            int mir[3] = {ijk[0], ijk[1], ijk[2]};
            mir[idim] = a.mirrorfac[idim][iside] - ijk[idim];
            if (mir[idim] == ijk[idim]) *self = 0.0;
            else if (mir[idim] >= a.alo[idim] && mir[idim] <= a.ahi[idim])
                *self += a.psign[idim][iside] * a.F.p[a.F.off(mir[0], mir[1], mir[2])];
        }
    for (int idim = 0; idim < 3; ++idim)                           // :377-394, rho counts as tangential (:666)
        for (int iside = 0; iside < 2; ++iside) {
            if (!a.refl[idim][iside]) continue;
            int mir[3] = {ijk[0], ijk[1], ijk[2]};
            mir[idim] = a.mirrorfac[idim][iside] - ijk[idim];
            if (mir[idim] != ijk[idim] && mir[idim] >= a.alo[idim] && mir[idim] <= a.ahi[idim])
                a.F.p[a.F.off(mir[0], mir[1], mir[2])] = -*self;
        }
}
__global__ void pec_rho_kernel(PecRhoArgs a) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.total) pec_rho_body(t, a);
}

}  // namespace pic

using namespace pic;

// rho is ADDED to (the caller zeroes it); xyzmin / lo describe the tile box grown by rho's guard cells
// (WarpXParticleContainer.cpp:952-975).
extern "C" int pic_deposit_charge(const pic_soa* p, long offset, long np, const pic_fab* rho, const double dinv[3],
                                  const double xyzmin[3], const int lo[3], double q, int nox, void* stream) {
    if (np == 0 || q == 0.0) return 0;
    PIC_REQUIRE(nox >= 1 && nox <= 4, "pic_deposit_charge: particle shape order %d not in 1..4", nox);
    PIC_REQUIRE(offset >= 0 && offset + np <= p->np, "pic_deposit_charge: range outside the tile");
    ChargeArgs a;
    a.x = p->x + offset; a.y = p->y + offset; a.z = p->z + offset; a.w = p->w + offset;
    a.np = np;
    a.R = make_view(*rho);
    for (int d = 0; d < 3; ++d) {
        PIC_REQUIRE(rho->ng[d] >= nox, "pic_deposit_charge: rho needs more guard cells");
        a.stag[d] = rho->stag[d]; a.lo[d] = lo[d]; a.dinv[d] = dinv[d]; a.xyzmin[d] = xyzmin[d];
    }
    a.q_invvol = q * (dinv[0] * dinv[1] * dinv[2]);
    if (nox == 1) PIC_LAUNCH(charge_kernel<1>, charge_body<1>, a, a.np, stream);
    else if (nox == 2) PIC_LAUNCH(charge_kernel<2>, charge_body<2>, a, a.np, stream);
    else if (nox == 3) PIC_LAUNCH(charge_kernel<3>, charge_body<3>, a, a.np, stream);
    else PIC_LAUNCH(charge_kernel<4>, charge_body<4>, a, a.np, stream);
    return launched_ok("pic_deposit_charge") ? 0 : 1;
}

extern "C" int pic_apply_pec_rho(const pic_fab* rho, const pic_geom* g, const pic_boundaries* b, void* stream) {
    PecRhoArgs a;
    a.F = make_view(*rho);
    a.total = 1;
    bool any = false;
    for (int d = 0; d < 3; ++d) {
        const bool plo = b->particle_lo[d] == PIC_PARTICLE_REFLECTING, phi = b->particle_hi[d] == PIC_PARTICLE_REFLECTING;
        a.refl[d][0] = plo || b->field_lo[d] == PIC_FIELD_PEC;
        a.refl[d][1] = phi || b->field_hi[d] == PIC_FIELD_PEC;
        any = any || a.refl[d][0] || a.refl[d][1];
        a.psign[d][0] = plo ? 1.0 : -1.0;
        a.psign[d][1] = phi ? 1.0 : -1.0;
        const int dom_hi = g->n_cell[d] - 1 + rho->stag[d];            // the domain box in rho's index type (:640)
        a.mirrorfac[d][0] = 2 * 0 - (1 - rho->stag[d]);                // :679-680
        a.mirrorfac[d][1] = 2 * dom_hi + (1 - rho->stag[d]);
        a.lo[d] = vlo(*rho, d); a.n[d] = vhi(*rho, d) - a.lo[d] + 1;
        a.alo[d] = rho->lo[d]; a.ahi[d] = rho->hi[d];
        a.total *= a.n[d];
    }
    if (!any) return 0;
    PIC_LAUNCH(pec_rho_kernel, pec_rho_body, a, a.total, stream);
    return launched_ok("pic_apply_pec_rho") ? 0 : 1;
}
