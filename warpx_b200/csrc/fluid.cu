// Cold relativistic fluid species (3D Cartesian, periodic domains): the four kernels of
// WarpXFluidContainer::Evolve (paths relative to Source/ of ECP-WarpX/WarpX):
//   pic_fluid_gather_push     <- WarpXFluidContainer::GatherAndPush        Fluids/WarpXFluidContainer.cpp:967-1238
//   pic_fluid_advect          <- WarpXFluidContainer::AdvectivePush_Muscl  :421-893 (leaves Fluids/MusclHancockUtils.H)
//   pic_fluid_deposit_current <- WarpXFluidContainer::DepositCurrent       :1276-1398
//   pic_fluid_deposit_charge  <- WarpXFluidContainer::DepositCharge        :1240-1273
// State: four all-nodal components N, NUx, NUy, NUz with 2 guard nodes (AllocateLevelMFs :142-164).
//
// Every expression is evaluated in the reference's order with products and sums rounded separately: build.py
// compiles this file with -fmad=false (the host harness compiles with -ffp-contract=off), so a stage gives the
// bits of the reference's CPU build, and the fusion below changes where intermediates live, not what they are.
//
// The advection is one kernel.  The reference predicts six 4-component edge arrays in HBM (the MUSCL-Hancock
// half step, :538-755) and differences their Rusanov fluxes in a second pass (:786-891).  Here a block stages
// N and U = NU/N of its 8x8x4 nodes plus a 2-node halo in shared memory; each thread predicts the edge states
// of its node and of its six neighbours (the edges its two fluxes per direction need) in registers and writes
// N and NU of its node to the output state.  HBM traffic: 64 B per node plus the halo re-reads.  Output goes to
// a second state (the update reads the neighbours' old values, which another block may already have replaced).
#include <math.h>

#include "pic_common.cuh"
#include "harness_launch.cuh"

namespace pic {

struct FluidView { FabView N, U[3]; };

static inline FluidView make_fluid(const pic_fab f[4]) {
    FluidView v;
    v.N = make_view(f[0]);
    for (int c = 0; c < 3; ++c) v.U[c] = make_view(f[1 + c]);
    return v;
}

// ---- leaves of MusclHancockUtils.H ------------------------------------------------------------------------
PIC_HD double fl_min(double a, double b) { return (b < a) ? b : a; }       // std::min
PIC_HD double fl_max(double a, double b) { return (a < b) ? b : a; }       // std::max
PIC_HD double fl_minmod3(double a, double b, double c) {                    // :69-79
    if (a > 0.0 && b > 0.0 && c > 0.0) return fl_min(a, fl_min(b, c));
    if (a < 0.0 && b < 0.0 && c < 0.0) return fl_max(a, fl_max(b, c));
    return 0.0;
}
PIC_HD double fl_ave(double a, double b) {                                  // :145-154
    return (a * b > 0.0) ? fl_minmod3((a + b) / 2.0, 2.0 * a, 2.0 * b) : 0.0;
}

struct Edge { double q[4]; };   // N, Ux, Uy, Uz at one side of an edge

// V_calc (:34-41): velocity component d of an edge state
PIC_HD double fl_v(const Edge& e, int d, double c_sq) {
    const double gamma = sqrt(1.0 + (e.q[1] * e.q[1] + e.q[2] * e.q[2] + e.q[3] * e.q[3]) / c_sq);
    return e.q[1 + d] / gamma;
}
// Rusanov fluxes flux_N / flux_NUx,y,z (:94-131) of component k at an edge: m = U_minus (left), p = U_plus (right)
PIC_HD double fl_flux(const Edge& m, const Edge& p, int k, double vm, double vp) {
    const double c = fl_max(fabs(vm), fabs(vp));
    if (k == 0) return 0.5 * (vm * m.q[0] + vp * p.q[0]) - (0.5 * c) * (p.q[0] - m.q[0]);
    return 0.5 * (vm * m.q[0] * m.q[k] + vp * p.q[0] * p.q[k]) - (0.5 * c) * (p.q[0] * p.q[k] - m.q[0] * m.q[k]);
}

struct AdvectConsts {
    double c_sq;
    double dt_over_dx[3], dt_over_dx_half[3];
};

// Tile of the fused advection: TX x TY x TZ output nodes, staged with a 2-node halo.
constexpr int FL_TX = 8, FL_TY = 8, FL_TZ = 4, FL_H = 2;
constexpr int FL_SX = FL_TX + 2 * FL_H, FL_SY = FL_TY + 2 * FL_H, FL_SZ = FL_TZ + 2 * FL_H;
constexpr int FL_S = FL_SX * FL_SY * FL_SZ;

// The half-step prediction of one node (:543-656): edge states hi[d] (U_minus at the node's own index, the left
// state of the edge to its +d side) and lo[d] (U_plus at index - 1, the right state of the edge to its -d side),
// before the positivity limiter.  Returns false where N <= 0: the edges are zero (set_U_edges_to_zero, :741-751).
PIC_HD bool fl_predict(const double* sN, const double* const sU[3], int s, const int st[3], const AdvectConsts& k,
                       Edge hi[3], Edge lo[3]) {
    const double N = sN[s];
    if (!(N > 0.0)) {
        for (int d = 0; d < 3; ++d)
            for (int c = 0; c < 4; ++c) hi[d].q[c] = lo[d].q[c] = 0.0;
        return false;
    }
    const double U[3] = {sU[0][s], sU[1][s], sU[2][s]};
    const double gamma = sqrt(1.0 + (U[0] * U[0] + U[1] * U[1] + U[2] * U[2]) / (k.c_sq));
    const double inv_c2_gamma3 = 1.0 / (k.c_sq * gamma * gamma * gamma);
    double dU[3][4], JdU[3][4];
    for (int d = 0; d < 3; ++d) {
        const int m = s - st[d], p = s + st[d];
        dU[d][0] = fl_ave(N - sN[m], sN[p] - N);                                      // DownD*_N, UpD*_N
        for (int c = 0; c < 3; ++c) dU[d][1 + c] = fl_ave(U[c] - sU[c][m], sU[c][p] - U[c]);   // DownD*_U, UpD*_U
        const double V = U[d] / gamma;
        double J0[3];                                                                 // row 0 of J_d (:560-606)
        for (int c = 0; c < 3; ++c)
            J0[c] = (c == d) ? N * (1 / gamma) * (1 - V * V / k.c_sq) : -N * U[c] * U[d] * inv_c2_gamma3;
        JdU[d][0] = V * dU[d][0] + J0[0] * dU[d][1] + J0[1] * dU[d][2] + J0[2] * dU[d][3];   // :619-630
        for (int c = 1; c < 4; ++c) JdU[d][c] = V * dU[d][c];
    }
    const double base[4] = {N, U[0], U[1], U[2]};
    for (int c = 0; c < 4; ++c) {
        const double ut = base[c] - k.dt_over_dx_half[0] * JdU[0][c] - k.dt_over_dx_half[1] * JdU[1][c]
                          - k.dt_over_dx_half[2] * JdU[2][c];                          // U_tilde, :631-634
        for (int d = 0; d < 3; ++d) {                                                 // compute_U_edges, :203-226
            hi[d].q[c] = ut + dU[d][c] / 2.0;
            lo[d].q[c] = ut - dU[d][c] / 2.0;
        }
    }
    return true;
}

// positivity_limiter (:253-294) in direction d.  have_hi / have_lo: whether the edge lies in the box the
// reference predicts over (the valid box grown by 1, converted to the edge's index type): for a node on the
// outer layer of that box only its inner edge exists, and only that edge's own density decides.
PIC_HD int fl_limit(Edge& hi, Edge& lo, const double* sN, const double* const sU[3], int s, bool have_hi,
                    bool have_lo) {
    const bool reset_hi = have_hi && (hi.q[0] < 0.0 || (have_lo && lo.q[0] < 0.0));
    const bool reset_lo = have_lo && (lo.q[0] < 0.0 || (have_hi && hi.q[0] < 0.0));
    const double r[4] = {sN[s], sU[0][s], sU[1][s], sU[2][s]};
    for (int c = 0; c < 4; ++c) {
        if (reset_hi) hi.q[c] = r[c];
        if (reset_lo) lo.q[c] = r[c];
    }
    return (reset_hi || reset_lo) ? 1 : 0;
}

struct AdvectArgs {
    FluidView in, out;
    int vlo[3], vhi[3];      // valid nodes (inclusive)
    int alo[3], ahi[3];      // allocated range of the input
    AdvectConsts k;
    unsigned long long* counters;   // optional (tests): [0] nodes with zero edges, [1] directions the limiter reset
};

__global__ void __launch_bounds__(FL_TX * FL_TY * FL_TZ)
fluid_advect_kernel(AdvectArgs a) {
    PIC_STATIC_SMEM(double, sN, FL_S);
    PIC_STATIC_SMEM(double, sUx, FL_S);
    PIC_STATIC_SMEM(double, sUy, FL_S);
    PIC_STATIC_SMEM(double, sUz, FL_S);
    double* const sU[3] = {sUx, sUy, sUz};
    const int o[3] = {a.vlo[0] + (int)blockIdx.x * FL_TX - FL_H, a.vlo[1] + (int)blockIdx.y * FL_TY - FL_H,
                      a.vlo[2] + (int)blockIdx.z * FL_TZ - FL_H};
    const int tid = threadIdx.x + FL_TX * (threadIdx.y + FL_TY * threadIdx.z);
    for (int t = tid; t < FL_S; t += FL_TX * FL_TY * FL_TZ) {
        const int g[3] = {o[0] + t % FL_SX, o[1] + (t / FL_SX) % FL_SY, o[2] + t / (FL_SX * FL_SY)};
        double n = 0.0, u[3] = {0.0, 0.0, 0.0};
        if (g[0] >= a.alo[0] && g[0] <= a.ahi[0] && g[1] >= a.alo[1] && g[1] <= a.ahi[1] && g[2] >= a.alo[2] &&
            g[2] <= a.ahi[2]) {
            const long off = a.in.N.off(g[0], g[1], g[2]);
            n = a.in.N.p[off];
            // U = NU / N where N > 0, else 0: the reference's U of the node (:547-549) and of its neighbours
            // (DownD*_U / UpD*_U) are this same quotient
            if (n > 0.0)
                for (int c = 0; c < 3; ++c) u[c] = a.in.U[c].p[off] / n;
        }
        sN[t] = n;
        for (int c = 0; c < 3; ++c) sU[c][t] = u[c];
    }
    __syncthreads();
    const int l[3] = {(int)threadIdx.x + FL_H, (int)threadIdx.y + FL_H, (int)threadIdx.z + FL_H};
    const int g[3] = {o[0] + l[0], o[1] + l[1], o[2] + l[2]};
    if (g[0] > a.vhi[0] || g[1] > a.vhi[1] || g[2] > a.vhi[2]) return;
    const int st[3] = {1, FL_SX, FL_SX * FL_SY};
    const int s = l[0] + FL_SX * (l[1] + FL_SY * l[2]);
    Edge hi[3], lo[3], nb_hi[3], nb_lo[3];
    int limited = 0;
    const bool self_pos = fl_predict(sN, sU, s, st, a.k, hi, lo);
    if (self_pos)
        for (int d = 0; d < 3; ++d) limited += fl_limit(hi[d], lo[d], sN, sU, s, true, true);
    if (a.counters) {
        if (!self_pos) atomicAdd(&a.counters[0], 1ull);
        if (limited) atomicAdd(&a.counters[1], (unsigned long long)limited);
    }
    double dF[3][4];
    for (int d = 0; d < 3; ++d) {
        // left neighbour: its hi edge is the left state of this node's -d edge
        Edge L, R;
        {
            const int sm = s - st[d];
            if (fl_predict(sN, sU, sm, st, a.k, nb_hi, nb_lo))
                fl_limit(nb_hi[d], nb_lo[d], sN, sU, sm, true, g[d] - 1 >= a.vlo[d]);
            L = nb_hi[d];
        }
        {
            const int sp = s + st[d];
            if (fl_predict(sN, sU, sp, st, a.k, nb_hi, nb_lo))
                fl_limit(nb_hi[d], nb_lo[d], sN, sU, sp, g[d] + 1 <= a.vhi[d], true);
            R = nb_lo[d];
        }
        // dF (:493-517): flux at the +d edge (this node's hi, right neighbour's lo) minus flux at the -d edge
        const double vm_i = fl_v(hi[d], d, a.k.c_sq), vp_i = fl_v(R, d, a.k.c_sq);
        const double vm_l = fl_v(L, d, a.k.c_sq), vp_l = fl_v(lo[d], d, a.k.c_sq);
        for (int c = 0; c < 4; ++c) dF[d][c] = fl_flux(hi[d], R, c, vm_i, vp_i) - fl_flux(L, lo[d], c, vm_l, vp_l);
    }
    const long off = a.in.N.off(g[0], g[1], g[2]);
    const double q0[4] = {sN[s], a.in.U[0].p[off], a.in.U[1].p[off], a.in.U[2].p[off]};
    double* const dst[4] = {a.out.N.p, a.out.U[0].p, a.out.U[1].p, a.out.U[2].p};
    for (int c = 0; c < 4; ++c)                                                       // :794-805
        dst[c][off] = q0[c] - a.k.dt_over_dx[0] * dF[0][c] - a.k.dt_over_dx[1] * dF[1][c] - a.k.dt_over_dx[2] * dF[2][c];
}

// ---- GatherAndPush (:967-1238, no external fields, no boost) ------------------------------------------------
// ablastr::coarsen::sample::Interp (ablastr/coarsen/sample.H:47-104) with cr = 1 onto the nodal index type
template <typename Src>
PIC_HD double fl_interp(const Src& F, const int sf[3], const int sc[3], int i, int j, int k) {
    int np[3], imin[3];
    const int ic[3] = {i, j, k};
    for (int l = 0; l < 3; ++l) {
        np[l] = 1 + (sf[l] > sc[l] ? sf[l] - sc[l] : sc[l] - sf[l]);
        imin[l] = ic[l] - sc[l] * (1 - sf[l]);
    }
    const double wx = 1.0 / (double)np[0], wy = 1.0 / (double)np[1], wz = 1.0 / (double)np[2];
    double c = 0.0;
    for (int kr = 0; kr < np[2]; ++kr)
        for (int jr = 0; jr < np[1]; ++jr)
            for (int ir = 0; ir < np[0]; ++ir) c += wx * wy * wz * F.p[F.off(imin[0] + ir, imin[1] + jr, imin[2] + kr)];
    return c;
}

// UpdateMomentumHigueraCary (Particles/Pusher/UpdateMomentumHigueraCary.H:21-64)
PIC_HD void fl_push_hc(double& ux, double& uy, double& uz, double Ex, double Ey, double Ez, double Bx, double By,
                       double Bz, double q, double m, double dt) {
    const double qmt = 0.5 * q * dt / m;
    constexpr double invclight = 1.0 / C_LIGHT;
    constexpr double invclightsq = 1.0 / (C_LIGHT * C_LIGHT);
    const double umx = ux + qmt * Ex, umy = uy + qmt * Ey, umz = uz + qmt * Ez;
    double gamma = 1.0 + (umx * umx + umy * umy + umz * umz) * invclightsq;
    const double betax = qmt * Bx, betay = qmt * By, betaz = qmt * Bz;
    const double betam = betax * betax + betay * betay + betaz * betaz;
    const double sigma = gamma - betam;
    const double ust = (umx * betax + umy * betay + umz * betaz) * invclight;
    gamma = 1.0 / sqrt(0.5 * (sigma + sqrt(sigma * sigma + 4.0 * (betam + ust * ust))));
    const double tx = gamma * betax, ty = gamma * betay, tz = gamma * betaz;
    const double s = 1.0 / (1.0 + (tx * tx + ty * ty + tz * tz));
    const double umt = umx * tx + umy * ty + umz * tz;
    const double upx = s * (umx + umt * tx + umy * tz - umz * ty);
    const double upy = s * (umy + umt * ty + umz * tx - umx * tz);
    const double upz = s * (umz + umt * tz + umx * ty - umy * tx);
    ux = upx + qmt * Ex + upy * tz - upz * ty;
    uy = upy + qmt * Ey + upz * tx - upx * tz;
    uz = upz + qmt * Ez + upx * ty - upy * tx;
}

struct GatherPushArgs {
    FluidView U;
    FabView E[3], B[3];
    int se[3][3], sb[3][3];
    int lo[3], n[3];
    double q, m, dt;
    long total;
};
PIC_HD void fluid_gather_push_body(long t, const GatherPushArgs& a) {
    const int i = a.lo[0] + (int)(t % a.n[0]);
    const int j = a.lo[1] + (int)((t / a.n[0]) % a.n[1]);
    const int k = a.lo[2] + (int)(t / ((long)a.n[0] * a.n[1]));
    const long off = a.U.N.off(i, j, k);
    const double N = a.U.N.p[off];
    if (!(N > 0.0)) return;
    const int nodal[3] = {1, 1, 1};
    double F[6];
    for (int c = 0; c < 3; ++c) {
        F[c] = fl_interp(a.E[c], a.se[c], nodal, i, j, k);
        F[3 + c] = fl_interp(a.B[c], a.sb[c], nodal, i, j, k);
    }
    double ux = a.U.U[0].p[off] / N, uy = a.U.U[1].p[off] / N, uz = a.U.U[2].p[off] / N;
    fl_push_hc(ux, uy, uz, F[0], F[1], F[2], F[3], F[4], F[5], a.q, a.m, a.dt);
    a.U.U[0].p[off] = N * ux;
    a.U.U[1].p[off] = N * uy;
    a.U.U[2].p[off] = N * uz;
}
__global__ void fluid_gather_push_kernel(GatherPushArgs a) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.total) fluid_gather_push_body(t, a);
}

// ---- DepositCurrent (:1276-1398) / DepositCharge (:1240-1273) ---------------------------------------------
// OwnerMask of a brick grid: a node shared by several bricks (or by periodic images of one) is added by exactly
// one of them.  Here that is the brick whose cells start at the node: the owned points of a component are its
// points with every index in [box_lo, box_hi].  J's SumBoundary afterwards gives every copy the one value.
struct FluidCurrentArgs {
    FluidView U;
    FabView J;
    int stag[3];
    int lo[3], n[3];
    double q, inv_clight_sq;
    long total;
    int comp;
};
// q * NU_c / gamma at a node, the reference's tmp_j*_fluid (:1333-1348)
PIC_HD double fl_nodal_current(const FluidView& U, int comp, double q, double inv_clight_sq, int i, int j, int k) {
    const long off = U.N.off(i, j, k);
    const double N = U.N.p[off];
    double gamma = 1.0;
    if (N > 0.0) {
        const double ux = U.U[0].p[off] / N, uy = U.U[1].p[off] / N, uz = U.U[2].p[off] / N;
        gamma = sqrt(1.0 + (ux * ux + uy * uy + uz * uz) * inv_clight_sq);
    }
    return q * (U.U[comp].p[off] / gamma);
}
PIC_HD void fluid_current_body(long t, const FluidCurrentArgs& a) {
    const int i = a.lo[0] + (int)(t % a.n[0]);
    const int j = a.lo[1] + (int)((t / a.n[0]) % a.n[1]);
    const int k = a.lo[2] + (int)(t / ((long)a.n[0] * a.n[1]));
    // Interp from the nodal temporary to the component's index type (:1380-1395): the nodes ic .. ic + 1 - stag
    int np[3];
    for (int l = 0; l < 3; ++l) np[l] = 2 - a.stag[l];
    const double w = (1.0 / (double)np[0]) * (1.0 / (double)np[1]) * (1.0 / (double)np[2]);
    double c = 0.0;
    for (int kr = 0; kr < np[2]; ++kr)
        for (int jr = 0; jr < np[1]; ++jr)
            for (int ir = 0; ir < np[0]; ++ir) c += w * fl_nodal_current(a.U, a.comp, a.q, a.inv_clight_sq, i + ir, j + jr, k + kr);
    a.J.p[a.J.off(i, j, k)] += c;
}
__global__ void fluid_current_kernel(FluidCurrentArgs a) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.total) fluid_current_body(t, a);
}

struct FluidChargeArgs {
    FabView N, R;
    int lo[3], n[3];
    double q;
    long total;
};
PIC_HD void fluid_charge_body(long t, const FluidChargeArgs& a) {
    const int i = a.lo[0] + (int)(t % a.n[0]);
    const int j = a.lo[1] + (int)((t / a.n[0]) % a.n[1]);
    const int k = a.lo[2] + (int)(t / ((long)a.n[0] * a.n[1]));
    a.R.p[a.R.off(i, j, k)] += a.q * a.N.p[a.N.off(i, j, k)];
}
__global__ void fluid_charge_kernel(FluidChargeArgs a) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.total) fluid_charge_body(t, a);
}

static int check_fluid(const pic_fab f[4], int min_ng, const char* who) {
    PIC_REQUIRE(f != nullptr, "%s: null fluid state", who);
    for (int c = 0; c < 4; ++c) {
        PIC_REQUIRE(f[c].p != nullptr, "%s: component %d has no data", who, c);
        for (int d = 0; d < 3; ++d) {
            PIC_REQUIRE(f[c].stag[d] == 1, "%s: the fluid state is all-nodal", who);
            PIC_REQUIRE(f[c].ng[d] >= min_ng, "%s: the fluid state needs %d guard nodes", who, min_ng);
            PIC_REQUIRE(f[c].lo[d] == f[0].lo[d] && f[c].hi[d] == f[0].hi[d] && f[c].ng[d] == f[0].ng[d],
                        "%s: the four components must have one shape", who);
        }
    }
    return 0;
}

}  // namespace pic

using namespace pic;

extern "C" int pic_fluid_gather_push(const pic_fab U[4], const pic_fab E[3], const pic_fab B[3], double q, double m,
                                     double dt, void* stream) {
    if (int rc = check_fluid(U, 1, "pic_fluid_gather_push")) return rc;
    PIC_REQUIRE(E && B && is_yee(E, B), "pic_fluid_gather_push: E and B must be on the Yee grid");
    PIC_REQUIRE(m > 0.0, "pic_fluid_gather_push: mass must be positive");
    GatherPushArgs a;
    a.U = make_fluid(U);
    a.total = 1;
    for (int d = 0; d < 3; ++d) {
        a.lo[d] = vlo(U[0], d);
        a.n[d] = vhi(U[0], d) - a.lo[d] + 1;
        a.total *= a.n[d];
    }
    for (int c = 0; c < 3; ++c) {
        a.E[c] = make_view(E[c]);
        a.B[c] = make_view(B[c]);
        for (int d = 0; d < 3; ++d) {
            a.se[c][d] = E[c].stag[d];
            a.sb[c][d] = B[c].stag[d];
            // the interpolation reads index - 1 along every staggered direction of the valid nodes
            PIC_REQUIRE(E[c].lo[d] <= a.lo[d] - 1 + E[c].stag[d] && E[c].hi[d] >= a.lo[d] + a.n[d] - 1 &&
                        B[c].lo[d] <= a.lo[d] - 1 + B[c].stag[d] && B[c].hi[d] >= a.lo[d] + a.n[d] - 1,
                        "pic_fluid_gather_push: E / B do not cover the fluid's valid nodes and one guard");
        }
    }
    a.q = q; a.m = m; a.dt = dt;
    PIC_LAUNCH(fluid_gather_push_kernel, fluid_gather_push_body, a, a.total, stream);
    return launched_ok("pic_fluid_gather_push") ? 0 : 1;
}

extern "C" int pic_fluid_advect(const pic_fab U_in[4], const pic_fab U_out[4], const double dx[3], double dt,
                                unsigned long long* counters, void* stream) {
    if (int rc = check_fluid(U_in, 2, "pic_fluid_advect")) return rc;
    if (int rc = check_fluid(U_out, 0, "pic_fluid_advect")) return rc;
    AdvectArgs a;
    a.in = make_fluid(U_in);
    a.out = make_fluid(U_out);
    for (int c = 0; c < 4; ++c) {
        PIC_REQUIRE(U_in[c].p != U_out[c].p, "pic_fluid_advect: input and output must be different arrays");
        for (int d = 0; d < 3; ++d)
            PIC_REQUIRE(U_out[c].lo[d] == U_in[c].lo[d] && U_out[c].hi[d] == U_in[c].hi[d],
                        "pic_fluid_advect: input and output must have one shape");
    }
    a.k.c_sq = C_LIGHT * C_LIGHT;
    unsigned grid[3];
    for (int d = 0; d < 3; ++d) {
        PIC_REQUIRE(dx[d] > 0.0, "pic_fluid_advect: cell size must be positive");
        a.vlo[d] = vlo(U_in[0], d);
        a.vhi[d] = vhi(U_in[0], d);
        a.alo[d] = U_in[0].lo[d];
        a.ahi[d] = U_in[0].hi[d];
        a.k.dt_over_dx[d] = (dt / dx[d]);                                               // :433-438
        a.k.dt_over_dx_half[d] = 0.5 * (dt / dx[d]);
    }
    grid[0] = (unsigned)((a.vhi[0] - a.vlo[0] + FL_TX) / FL_TX);
    grid[1] = (unsigned)((a.vhi[1] - a.vlo[1] + FL_TY) / FL_TY);
    grid[2] = (unsigned)((a.vhi[2] - a.vlo[2] + FL_TZ) / FL_TZ);
    a.counters = counters;
    fluid_advect_kernel<<<dim3(grid[0], grid[1], grid[2]), dim3(FL_TX, FL_TY, FL_TZ), 0, (cudaStream_t)stream>>>(a);
    count_launch();
    return check_launch("pic_fluid_advect") ? 0 : 1;
}

extern "C" int pic_fluid_deposit_current(const pic_fab U[4], const pic_fab J[3], double q, void* stream) {
    if (int rc = check_fluid(U, 0, "pic_fluid_deposit_current")) return rc;
    PIC_REQUIRE(J != nullptr, "pic_fluid_deposit_current: null J");
    static const int yee[3][3] = {{0, 1, 1}, {1, 0, 1}, {1, 1, 0}};
    for (int c = 0; c < 3; ++c) {
        for (int d = 0; d < 3; ++d) {
            PIC_REQUIRE(J[c].stag[d] == yee[c][d], "pic_fluid_deposit_current: J must be on the Yee grid");
            PIC_REQUIRE(vlo(J[c], d) == vlo(U[0], d) && vhi(J[c], d) + 1 - J[c].stag[d] == vhi(U[0], d),
                        "pic_fluid_deposit_current: J and the fluid must be on one box");
        }
    }
    for (int c = 0; c < 3; ++c) {
        FluidCurrentArgs a;
        a.U = make_fluid(U);
        a.J = make_view(J[c]);
        a.comp = c;
        a.q = q;
        a.inv_clight_sq = 1.0 / C_LIGHT / C_LIGHT;                                      // :1318
        a.total = 1;
        for (int d = 0; d < 3; ++d) {
            a.stag[d] = J[c].stag[d];
            a.lo[d] = vlo(U[0], d);
            a.n[d] = vhi(U[0], d) - a.lo[d];                                           // owned: [box_lo, box_hi]
            a.total *= a.n[d];
        }
        PIC_LAUNCH(fluid_current_kernel, fluid_current_body, a, a.total, stream);
        if (!launched_ok("pic_fluid_deposit_current")) return 1;
    }
    return 0;
}

extern "C" int pic_fluid_deposit_charge(const pic_fab* N, const pic_fab* rho, double q, void* stream) {
    PIC_REQUIRE(N && rho && N->p && rho->p, "pic_fluid_deposit_charge: null array");
    FluidChargeArgs a;
    a.N = make_view(*N);
    a.R = make_view(*rho);
    a.q = q;
    a.total = 1;
    for (int d = 0; d < 3; ++d) {
        PIC_REQUIRE(N->stag[d] == 1 && rho->stag[d] == 1, "pic_fluid_deposit_charge: N and rho are nodal");
        PIC_REQUIRE(vlo(*rho, d) == vlo(*N, d) && vhi(*rho, d) == vhi(*N, d),
                    "pic_fluid_deposit_charge: N and rho must be on one box");
        a.lo[d] = vlo(*N, d);
        a.n[d] = vhi(*N, d) - a.lo[d];                                                  // owned: [box_lo, box_hi]
        a.total *= a.n[d];
    }
    PIC_LAUNCH(fluid_charge_kernel, fluid_charge_body, a, a.total, stream);
    return launched_ok("pic_fluid_deposit_charge") ? 0 : 1;
}
