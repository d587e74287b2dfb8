// TEST INFRASTRUCTURE -- C API of the CPU oracle (see pic_oracle_core.hpp) plus a whole-loop
// driver that restates WarpX::Evolve / OneStep_nosub for a single-level, periodic, explicit
// FDTD run (Evolve/WarpXEvolve.cpp:93-347, 353-455, 473-531, 64-91).
//
// Built twice by oracle/Makefile:
//   libpic_oracle.so           leaf arithmetic = hand restatement   (always)
//   _ref/libpic_oracle_ref.so  leaf arithmetic = reference headers compiled verbatim from a
//                              WarpX source tree through oracle/amrex_shim (on request:
//                              make ref REF=<tree>; tests/golden/reference_leaves.json records it)
#ifdef ORC_LEAF_REFERENCE
#include "leaf_reference.hpp"
using Leaf = orc::LeafReference;
#else
#include "leaf_restated.hpp"
using Leaf = orc::LeafRestated;
#endif
#include "pic_oracle_core.hpp"
#include "pic_oracle_lwfa.hpp"

#include <array>
#include <chrono>
#include <memory>
#include <string>

using namespace orc;

namespace {

struct Species {
    double q, m;
    std::vector<double> a[7];           // x y z w ux uy uz  (PIdx order)
    // plasma injector (continuous injection with the moving window); z_inj = z at creation, the
    // input of user attributes such as regionofinterest(x,y,z,...) of the laser_acceleration deck
    bool has_injector = false;
    pic_plasma_injector inj{};
    double current_injection_position = 0.0;      // WarpXParticleContainer::m_current_injection_position
    std::vector<double> z_inj;
    pic_soa soa() {
        pic_soa s;
        s.x = a[0].data(); s.y = a[1].data(); s.z = a[2].data(); s.w = a[3].data();
        s.ux = a[4].data(); s.uy = a[5].data(); s.uz = a[6].data();
        s.idcpu = nullptr; s.np = (long)a[0].size();
        return s;
    }
};

// One box == the whole periodic domain, or a brick decomposition nb[0] x nb[1] x nb[2]
// (used as the oracle of the multi-GPU path).  All boxes live in this process.
struct Sim {
    pic_geom geom;
    int nox, galerkin, pusher, solver;
    int use_filter = 0, npass[3] = {1, 1, 1};      // warpx.use_filter / filter_npass_each_dir (WarpX.cpp:158,189)
    double dx[3], dinv[3], dt, cfl;
    int ng_EB[3], ng_J[3], ng_FG[3], ng_FS[3], ng_depos_J[3];
    pic_stencil st;
    int nb[3];
    struct Box {
        int lo[3], hi[3];                // cells
        std::vector<double> data[9];     // Ex Ey Ez Bx By Bz jx jy jz
        pic_fab fab[9];
        std::vector<Species> sp;
    };
    std::vector<Box> boxes;
    int nspecies = 0;
    bool is_synchronized = true;
    int istep = 0;
    double cur_time = 0.0;                         // t_new[0]
    // laser-wakefield additions (single box): boundaries, moving window, antennas
    pic_boundaries bnd{};
    bool any_pec = false;
    bool do_moving_window = false;
    int mw_dir = 2;
    double mw_v = 0.0, mw_x = 0.0;                 // moving_window_v [m/s], moving_window_x
    double gamma_boost = 1.0, beta_boost = 0.0;    // warpx.gamma_boost, boost_direction = z (WarpXUtil.cpp:114-121)
    bool use_nci = false;                          // particles.use_fdtd_nci_corr
    double nci_stencil[2][5];                      // [0] Ex Ey Bz, [1] Bx By Ez (m_stencil_2 of the two NCIGodfreyFilter)
    struct Laser { Antenna ant; std::vector<double> a[7]; };
    std::vector<Laser> lasers;
    double t_push = 0, t_dep = 0, t_fdtd = 0, t_halo = 0, t_other = 0;
};

double now() {
    return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// Staggering, Source/WarpX.cpp:2117-2125 (Yee grid): 1 = nodal.
const int STAG[9][3] = {{0, 1, 1}, {1, 0, 1}, {1, 1, 0},   // Ex Ey Ez
                        {1, 0, 0}, {0, 1, 0}, {0, 0, 1},   // Bx By Bz
                        {0, 1, 1}, {1, 0, 1}, {1, 1, 0}};  // jx jy jz (= E)

// guardCellManager::Init, Parallelization/GuardCellManager.cpp:62-161,310-343 (no MR, no NCI,
// not safe_guard_cells, FDTD).
void guard_cells(Sim& s) {
    for (int d = 0; d < 3; ++d) {
        const int ngt = s.nox;                                   // :62-64
        int ng = (ngt % 2) ? ngt + 1 : ngt;                      // :83-85 (even)
        int ngJ = ngt;                                           // :96-98
        if (s.use_nci && d == 2) { const int n4 = ngt + 4; ng = (n4 % 2) ? n4 + 1 : n4; }   // :87-90, nci_corr_stencil = m_stencil_width = 4
        if (s.do_moving_window) { ng = std::max(ng, 2); ngJ = std::max(ngJ, 2); }   // :103-115 (max_r = 2 on one level)
        s.ng_EB[d] = ng;
        s.ng_J[d] = ngJ + (int)std::ceil(C_LIGHT * 0.5 * s.dt / s.dx[d]);   // :147,161
        s.ng_depos_J[d] = s.ng_J[d];                             // :165
        if (s.use_filter) s.ng_J[d] += s.npass[d];               // + stencil_length - 1, :169-172
        s.ng_FS[d] = 1;                                          // Yee/CKC GetMaxGuardCell
        s.ng_EB[d] = std::max(s.ng_EB[d], s.ng_FS[d]);           // :297
        int fg = std::min((s.nox + 1) / 2, s.ng_EB[d]);          // :314-316
        fg = std::min(fg, s.ng_EB[d]);
        if (s.use_nci && d == 2) fg = std::min(fg + 4, s.ng_EB[d]);   // :319-330
        s.ng_FG[d] = std::max(fg, s.ng_FS[d]);                   // :338
    }
}

void alloc_box(Sim& s, Sim::Box& b) {
    for (int c = 0; c < 9; ++c) {
        pic_fab& f = b.fab[c];
        const int* ng = (c < 6) ? s.ng_EB : s.ng_J;
        for (int d = 0; d < 3; ++d) {
            f.stag[d] = STAG[c][d];
            f.ng[d] = ng[d];
            f.lo[d] = b.lo[d] - ng[d];
            f.hi[d] = b.hi[d] + STAG[c][d] + ng[d];
        }
        b.data[c].assign((size_t)fab_size(f), 0.0);
        f.p = b.data[c].data();
    }
}

void fill_EB(Sim& s, int c0, const int ng[3]) {  // FillBoundaryE (c0=0) / FillBoundaryB (c0=3)
    const double t0 = now();
    std::vector<pic_fab> fabs(s.boxes.size());
    for (int c = c0; c < c0 + 3; ++c) {
        for (size_t b = 0; b < s.boxes.size(); ++b) fabs[b] = s.boxes[b].fab[c];
        fill_boundary(fabs.data(), (int)fabs.size(), ng, s.geom);
    }
    s.t_halo += now() - t0;
}

// xyzmin of a box grown by ng: RealBox(bx, dx, prob_lo).lo = prob_lo + lo_index*dx
// (WarpX::getRealBox / LowerCorner, Source/WarpX.cpp:2851-2874; AMReX RealBox ctor).
void lower_corner(const Sim& s, const Sim::Box& b, const int ng[3], double xyzmin[3], int lo[3]) {
    for (int d = 0; d < 3; ++d) {
        lo[d] = b.lo[d] - ng[d];
        xyzmin[d] = s.geom.prob_lo[d] + s.dx[d] * lo[d];
    }
}

void push_p(Sim& s, double dtp) {  // mypc->PushP(lev, dt, E_aux, B_aux): box grown by Ex.nGrowVect (:2384-2385)
    const double t0 = now();
    for (auto& b : s.boxes) {
        double xyzmin[3]; int lo[3];
        lower_corner(s, b, s.ng_EB, xyzmin, lo);
        for (auto& sp : b.sp) {
            pic_soa P = sp.soa();
            gather_push<Leaf>(P, 0, P.np, b.fab, b.fab + 3, s.dinv, xyzmin, lo, sp.q, sp.m, dtp,
                              s.nox, s.galerkin, s.pusher, 0);
        }
    }
    s.t_push += now() - t0;
}

// Move particles that left their box to the owning box after the periodic wrap
// (ParticleContainer::Redistribute semantics; locate by cell index).
void erase_marked(std::vector<double>* a, int na, const std::vector<char>& keep) {
    for (int c = 0; c < na; ++c) {
        if (a[c].empty()) continue;
        size_t o = 0;
        for (size_t ip = 0; ip < keep.size(); ++ip) if (keep[ip]) a[c][o++] = a[c][ip];
        a[c].resize(o);
    }
}

void redistribute(Sim& s) {
    const double t0 = now();
    const bool all_periodic = s.geom.periodic[0] && s.geom.periodic[1] && s.geom.periodic[2];
    if (!all_periodic) {
        // mypc->ApplyBoundaryConditions() over all containers (species and lasers,
        // MultiParticleContainer.cpp:659-664), then Redistribute drops the lost particles
        std::vector<char> keep;
        for (auto& b : s.boxes)
            for (auto& sp : b.sp) {
                pic_soa P = sp.soa();
                apply_particle_boundaries(P, s.geom, s.bnd, keep);
                erase_marked(sp.a, 7, keep);
                erase_marked(&sp.z_inj, 1, keep);
            }
        for (auto& L : s.lasers) {
            pic_soa P; P.x = L.a[0].data(); P.y = L.a[1].data(); P.z = L.a[2].data(); P.w = L.a[3].data();
            P.ux = L.a[4].data(); P.uy = L.a[5].data(); P.uz = L.a[6].data(); P.idcpu = nullptr; P.np = (long)L.a[0].size();
            apply_particle_boundaries(P, s.geom, s.bnd, keep);
            erase_marked(L.a, 7, keep);
        }
    }
    for (auto& b : s.boxes)
        for (auto& sp : b.sp) { pic_soa P = sp.soa(); wrap_periodic(P, s.geom); }
    for (auto& L : s.lasers) {
        pic_soa P; P.x = L.a[0].data(); P.y = L.a[1].data(); P.z = L.a[2].data(); P.w = nullptr;
        P.ux = P.uy = P.uz = nullptr; P.idcpu = nullptr; P.np = (long)L.a[0].size();
        wrap_periodic(P, s.geom);
    }
    if (s.boxes.size() > 1) {
        for (int isp = 0; isp < s.nspecies; ++isp) {
            std::vector<std::array<std::vector<double>, 7>> in(s.boxes.size());
            for (size_t ib = 0; ib < s.boxes.size(); ++ib) {
                Species& sp = s.boxes[ib].sp[isp];
                std::array<std::vector<double>, 7> keep;
                const long np = (long)sp.a[0].size();
                for (long ip = 0; ip < np; ++ip) {
                    int cell[3], owner[3];
                    for (int d = 0; d < 3; ++d) {
                        cell[d] = (int)std::floor((sp.a[d][ip] - s.geom.prob_lo[d]) * s.dinv[d]);
                        cell[d] = std::min(std::max(cell[d], 0), s.geom.n_cell[d] - 1);
                        owner[d] = cell[d] / (s.geom.n_cell[d] / s.nb[d]);
                    }
                    const size_t ob = owner[0] + (size_t)s.nb[0] * (owner[1] + (size_t)s.nb[1] * owner[2]);
                    auto& dst = (ob == ib) ? keep : in[ob];
                    for (int a = 0; a < 7; ++a) dst[a].push_back(sp.a[a][ip]);
                }
                for (int a = 0; a < 7; ++a) sp.a[a].swap(keep[a]);
            }
            for (size_t ib = 0; ib < s.boxes.size(); ++ib)
                for (int a = 0; a < 7; ++a) {
                    auto& v = s.boxes[ib].sp[isp].a[a];
                    v.insert(v.end(), in[ib][a].begin(), in[ib][a].end());
                }
        }
    }
    s.t_other += now() - t0;
}

pic_soa laser_soa(Sim::Laser& L) {
    pic_soa P;
    P.x = L.a[0].data(); P.y = L.a[1].data(); P.z = L.a[2].data(); P.w = L.a[3].data();
    P.ux = L.a[4].data(); P.uy = L.a[5].data(); P.uz = L.a[6].data(); P.idcpu = nullptr;
    P.np = (long)L.a[0].size();
    return P;
}

// WarpX::MoveWindow (Utils/WarpXMovingWindow.cpp:139-476), one level, no PML, lab frame:
// advance moving_window_x, shift E, B (and J when move_j) by the whole number of cells the window
// has covered, move the domain, continuously inject plasma into the uncovered slab.
int move_window(Sim& s, int step, bool move_j) {
    (void)step;                                          // start_moving_window_step = 0, no end step
    if (!s.do_moving_window) return 0;
    const int dir = s.mw_dir;
    s.mw_x += (s.mw_v - s.beta_boost * C_LIGHT) / (1 - s.mw_v * s.beta_boost / C_LIGHT) * s.dt;  // :156
    // UpdateInjectionPosition (:59-136): plasma at rest in the lab -> v_shift = 0, transformed to the
    // boosted frame (:108-133; boost_direction[dir] = 1, the boost is along the window)
    for (auto& b : s.boxes)
        for (auto& sp : b.sp) {
            if (!sp.has_injector || !sp.inj.do_continuous_injection) continue;
            double v_shift = C_LIGHT * 0.0 / std::sqrt(1. + 0.0 * 0.0);
            if (s.gamma_boost > 1.) {
                v_shift = (v_shift - C_LIGHT * s.beta_boost) / (1. - v_shift * s.beta_boost / C_LIGHT);
                v_shift *= (dir == 2) ? 1 : 0;
            }
            sp.current_injection_position += v_shift * s.dt;
        }
    const double cdx = s.dx[dir];
    const int num_shift_base = static_cast<int>((s.mw_x - s.geom.prob_lo[dir]) / cdx);            // :171
    if (num_shift_base == 0) return 0;
    s.geom.prob_lo[dir] = s.geom.prob_lo[dir] + num_shift_base * cdx;                              // :181-184
    s.geom.prob_hi[dir] = s.geom.prob_hi[dir] + num_shift_base * cdx;
    for (auto& b : s.boxes)
        for (int dim = 0; dim < 3; ++dim) {                                                        // :226-266
            shift_fab(b.fab[3 + dim], s.geom, num_shift_base, dir, 0.0);
            shift_fab(b.fab[dim], s.geom, num_shift_base, dir, 0.0);
            if (move_j) shift_fab(b.fab[6 + dim], s.geom, num_shift_base, dir, 0.0);
        }
    // continuous injection (:388-438)
    for (auto& b : s.boxes)
        for (auto& sp : b.sp) {
            if (!sp.has_injector || !sp.inj.do_continuous_injection) continue;
            double new_pos = sp.current_injection_position;
            if (s.mw_v > 0.0)
                new_pos = sp.current_injection_position +
                          std::floor((s.geom.prob_hi[dir] - sp.current_injection_position) / cdx) * cdx;
            else if (s.mw_v < 0.0)
                new_pos = sp.current_injection_position -
                          std::floor((sp.current_injection_position - s.geom.prob_lo[dir]) / cdx) * cdx;
            double plo[3], phi[3];
            for (int d = 0; d < 3; ++d) { plo[d] = s.geom.prob_lo[d]; phi[d] = s.geom.prob_hi[d]; }
            if (s.mw_v > 0.0) { plo[dir] = sp.current_injection_position; phi[dir] = new_pos; }
            else if (s.mw_v < 0.0) { plo[dir] = new_pos; phi[dir] = sp.current_injection_position; }
            const bool ok = plo[0] < phi[0] && plo[1] < phi[1] && plo[2] < phi[2];               // RealBox::ok
            if (ok && sp.current_injection_position != new_pos) {
                const size_t n0 = sp.a[2].size();
                add_plasma(sp.inj, s.geom, s.dx, plo, phi, sp.a, s.cur_time);   // t = t_new (WarpXEvolve.cpp:232-246)
                for (size_t ip = n0; ip < sp.a[2].size(); ++ip) sp.z_inj.push_back(sp.a[2][ip]);
                sp.current_injection_position = new_pos;
            }
        }
    return num_shift_base;
}

// WarpX::OneStep_nosub (WarpXEvolve.cpp:353-455) preceded by ExplicitFillBoundaryEBUpdateAux
// (:473-531) and followed by the end-of-step bookkeeping of WarpX::Evolve (:221-256).
void one_step(Sim& s, bool last_step) {
    // ---- ExplicitFillBoundaryEBUpdateAux ----
    if (s.is_synchronized) {
        fill_EB(s, 0, s.ng_EB); fill_EB(s, 3, s.ng_EB);          // :487-488 (ng_alloc_EB)
        push_p(s, -0.5 * s.dt);                                    // :492-504
        s.is_synchronized = false;
    } else {
        fill_EB(s, 0, s.ng_FG); fill_EB(s, 3, s.ng_FG);          // :515-516
    }
    // ---- PushParticlesandDeposit (:366 -> MultiParticleContainer::Evolve) ----
    double t0 = now();
    for (auto& b : s.boxes)
        for (int c = 6; c < 9; ++c) {                                                   // J.setVal(0)
            double* p = b.data[c].data();
            const long n = (long)b.data[c].size();
#pragma omp parallel for schedule(static)
            for (long i = 0; i < n; ++i) p[i] = 0.0;
        }
    s.t_other += now() - t0;
    for (auto& b : s.boxes) {
        double xyzmin[3], xyzminJ[3]; int lo[3], loJ[3];
        lower_corner(s, b, s.ng_EB, xyzmin, lo);                   // PushPX: box.grow(ngEB), :2583
        lower_corner(s, b, s.ng_J, xyzminJ, loJ);                  // DepositCurrent: tilebox.grow(ng_J)
        // applyNCIFilter (PhysicalParticleContainer.cpp:1900-1911,2097-2169): E and B are filtered along z
        // into temporaries over the tile box grown by the shape order; the gather reads those
        const pic_fab* EB = b.fab;
        std::vector<double> nci_data[6];
        pic_fab nci_fab[6];
        if (s.use_nci) {
            t0 = now();
            for (int c = 0; c < 6; ++c) {
                nci_fab[c] = b.fab[c];
                nci_data[c].assign((size_t)fab_size(b.fab[c]), 0.0);
                nci_fab[c].p = nci_data[c].data();
                int tlo[3], thi[3];
                for (int d = 0; d < 3; ++d) { tlo[d] = b.lo[d] - s.nox; thi[d] = b.hi[d] + s.nox + STAG[c][d]; }
                const bool exeybz = (c == 0 || c == 1 || c == 5);                      // :2132-2163
                apply_nci_filter(b.fab[c], nci_fab[c], s.nci_stencil[exeybz ? 0 : 1], tlo, thi);
            }
            EB = nci_fab;
            s.t_other += now() - t0;
        }
        for (auto& sp : b.sp) {
            pic_soa P = sp.soa();
            t0 = now();
            gather_push<Leaf>(P, 0, P.np, EB, EB + 3, s.dinv, xyzmin, lo, sp.q, sp.m, s.dt,
                              s.nox, s.galerkin, s.pusher, 1);
            s.t_push += now() - t0;
            t0 = now();
            deposit<Leaf>(P, 0, P.np, b.fab + 6, s.dinv, xyzminJ, loJ, sp.q, s.dt,
                          -0.5 * s.dt /* relative_time, PhysicalParticleContainer.cpp:2029 */, s.nox);
            s.t_dep += now() - t0;
        }
        // laser antennas come after the species in allcontainers (MultiParticleContainer.cpp:60-75);
        // LaserParticleContainer::Evolve (LaserParticleContainer.cpp:563-700): charge = 1 (:88)
        for (auto& L : s.lasers) {
            pic_soa P = laser_soa(L);
            antenna_push(L.ant, P, s.cur_time, s.dt);
            deposit<Leaf>(P, 0, P.np, b.fab + 6, s.dinv, xyzminJ, loJ, 1.0, s.dt, -0.5 * s.dt, s.nox);
        }
    }
    // ---- SyncCurrentAndRho -> [ApplyFilterJ, WarpXComm.cpp:1233-1237,1357-1374] -> SumBoundaryJ
    //      (:1386-1424): src = ng_depos_J (+ stencil_length-1 with the filter, :1413-1416),
    //      dst = all guards of J (WarpXSumGuardCells.cpp:22-23) ----
    t0 = now();
    {
        int src_ng[3];
        for (int d = 0; d < 3; ++d) src_ng[d] = std::min(s.ng_depos_J[d] + (s.use_filter ? s.npass[d] : 0), s.ng_J[d]);
        if (s.use_filter)
            for (auto& b : s.boxes)
                for (int c = 6; c < 9; ++c) {
                    std::vector<double> tmp(b.data[c].size());
                    pic_fab dst = b.fab[c];
                    dst.p = tmp.data();
                    apply_filter(b.fab[c], dst, s.npass);
                    b.data[c].swap(tmp);                         // MultiFab::Copy(J, Jf)
                    b.fab[c].p = b.data[c].data();
                }
        std::vector<pic_fab> fabs(s.boxes.size());
        for (int c = 6; c < 9; ++c) {
            for (size_t b = 0; b < s.boxes.size(); ++b) fabs[b] = s.boxes[b].fab[c];
            sum_boundary(fabs.data(), (int)fabs.size(), src_ng, s.ng_J, s.geom);
        }
        // reflect J over PEC / reflecting boundaries (WarpXEvolve.cpp:629-640)
        if (s.any_pec) for (auto& b : s.boxes) apply_pec_current(b.fab + 6, s.geom, s.bnd);
    }
    s.t_halo += now() - t0;
    // ---- field solve (:421-437); WarpX::EvolveB / EvolveE end with ApplyB/EfieldBoundary
    //      (FieldSolver/WarpXPushFieldsEM.cpp:926,990) ----
    auto evolveB = [&](double dtb) {
        const double t1 = now();
        for (auto& b : s.boxes) {
            evolve_b<Leaf>(b.fab + 3, b.fab, s.st, dtb);
            if (s.any_pec) apply_pec_field(b.fab + 3, false, s.geom, s.bnd, s.ng_FG);
        }
        s.t_fdtd += now() - t1;
    };
    evolveB(0.5 * s.dt);
    fill_EB(s, 3, s.ng_FS);
    t0 = now();
    for (auto& b : s.boxes) {
        evolve_e<Leaf>(b.fab, b.fab + 3, b.fab + 6, s.st, s.dt);
        if (s.any_pec) apply_pec_field(b.fab, true, s.geom, s.bnd, s.ng_FG);
    }
    s.t_fdtd += now() - t0;
    fill_EB(s, 0, s.ng_FS);
    evolveB(0.5 * s.dt);
    // ---- end of step (WarpX::Evolve :219-256) ----
    if (last_step) {  // Synchronize() (:64-91)
        fill_EB(s, 0, s.ng_FG); fill_EB(s, 3, s.ng_FG);
        push_p(s, 0.5 * s.dt);
        s.is_synchronized = true;
    }
    ++s.istep;
    s.cur_time += s.dt;                                           // :232
    move_window(s, s.istep, s.is_synchronized);                   // :247 (move_j = is_synchronized)
    redistribute(s);   // HandleParticlesAtBoundaries -> ApplyBoundaryConditions, RedistributeLocal
}

}  // namespace

extern "C" {

const char* orc_leaf_name() { return Leaf::name; }

// ---- leaf probes (used to compare restated vs reference leaves bit for bit) -----------------
int orc_shape(int order, double x, double* s) {
    switch (order) {
        case 0: return Leaf::shape<0>(s, x);
        case 1: return Leaf::shape<1>(s, x);
        case 2: return Leaf::shape<2>(s, x);
        case 3: return Leaf::shape<3>(s, x);
        case 4: return Leaf::shape<4>(s, x);
    }
    return -999;
}
int orc_shifted_shape(int order, double x_old, int i_new, double* s /* order+3, pre-zeroed */) {
    switch (order) {
        case 0: return Leaf::shifted_shape<0>(s, x_old, i_new);
        case 1: return Leaf::shifted_shape<1>(s, x_old, i_new);
        case 2: return Leaf::shifted_shape<2>(s, x_old, i_new);
        case 3: return Leaf::shifted_shape<3>(s, x_old, i_new);
        case 4: return Leaf::shifted_shape<4>(s, x_old, i_new);
    }
    return -999;
}
void orc_push_momentum(int pusher, double* u /*3*/, const double* EB /*6*/, double q, double m,
                       double dt) {
    if (pusher == PIC_PUSHER_BORIS) Leaf::boris(u[0], u[1], u[2], EB[0], EB[1], EB[2], EB[3], EB[4], EB[5], q, m, dt);
    else if (pusher == PIC_PUSHER_VAY) Leaf::vay(u[0], u[1], u[2], EB[0], EB[1], EB[2], EB[3], EB[4], EB[5], q, m, dt);
    else Leaf::higuera_cary(u[0], u[1], u[2], EB[0], EB[1], EB[2], EB[3], EB[4], EB[5], q, m, dt);
}
void orc_update_position(double* x /*3*/, const double* u /*3*/, double dt) {
    Leaf::update_position(x[0], x[1], x[2], u[0], u[1], u[2], dt);
}
void orc_stencil_coefs(int algo, const double* dx, pic_stencil* st) { Leaf::stencil_coefs(algo, dx, st); }
double orc_max_dt(int algo, const double* dx) { return Leaf::max_dt(algo, dx); }

// ---- stage-level entry points: same argument sets as include/pic_b200.h, host pointers -----
int orc_evolve_b(const pic_fab* B, const pic_fab* E, const pic_stencil* st, double dt) {
    evolve_b<Leaf>(B, E, *st, dt); return 0;
}
int orc_evolve_e(const pic_fab* E, const pic_fab* B, const pic_fab* J, const pic_stencil* st, double dt) {
    evolve_e<Leaf>(E, B, J, *st, dt); return 0;
}
int orc_gather_push(const pic_soa* p, long offset, long np, const pic_fab* E, const pic_fab* B,
                    const double* dinv, const double* xyzmin, const int* lo, double q, double m,
                    double dt, int nox, int galerkin, int pusher, int push_position) {
    return gather_push<Leaf>(*p, offset, np, E, B, dinv, xyzmin, lo, q, m, dt, nox, galerkin, pusher,
                             push_position);
}
int orc_deposit_esirkepov(const pic_soa* p, long offset, long np, const pic_fab* J,
                          const double* dinv, const double* xyzmin, const int* lo, double q,
                          double dt, double relative_time, int nox) {
    return deposit<Leaf>(*p, offset, np, J, dinv, xyzmin, lo, q, dt, relative_time, nox);
}
void orc_fill_boundary(const pic_fab* fabs, int nfab, const int* ng, const pic_geom* g) {
    fill_boundary(fabs, nfab, ng, *g);
}
void orc_sum_boundary(const pic_fab* fabs, int nfab, const int* src_ng, const int* dst_ng,
                      const pic_geom* g) {
    sum_boundary(fabs, nfab, src_ng, dst_ng, *g);
}
void orc_wrap_periodic(const pic_soa* p, const pic_geom* g) { wrap_periodic(*p, *g); }
double orc_sum_squares_unique(const pic_fab* fabs, int nfab, const pic_geom* g) {
    return sum_squares_unique(fabs, nfab, *g);
}
void orc_apply_filter(const pic_fab* src, const pic_fab* dst, const int* npass) { apply_filter(*src, *dst, npass); }
void orc_filter_stencil(int npass, double* out /* npass+1 */) {
    const std::vector<double> st = filter_stencil(npass);
    for (size_t n = 0; n < st.size(); ++n) out[n] = st[n];
}
double orc_checksum_cell_centered(const pic_fab* f, const int* box_lo, const int* box_hi) {
    return checksum_cell_centered(*f, box_lo, box_hi);
}

// ---- whole-loop driver --------------------------------------------------------------------
// dt <= 0: dt = cfl * max_dt (WarpXComputeDt.cpp:56-95).
void* orc_sim_create(const int* n_cell, const double* prob_lo, const double* prob_hi, int nox,
                     int galerkin, int pusher, int solver, double cfl, double dt, const int* nb,
                     int use_filter, const int* npass) {
    auto* s = new Sim();
    s->use_filter = use_filter;
    for (int d = 0; d < 3; ++d) s->npass[d] = npass ? npass[d] : 1;
    for (int d = 0; d < 3; ++d) {
        s->geom.n_cell[d] = n_cell[d]; s->geom.prob_lo[d] = prob_lo[d]; s->geom.prob_hi[d] = prob_hi[d];
        s->geom.periodic[d] = 1;
        s->dx[d] = (prob_hi[d] - prob_lo[d]) / n_cell[d];       // amrex::Geometry cell size
        s->dinv[d] = 1.0 / s->dx[d];                             // WarpX::InvCellSize
        s->nb[d] = nb ? nb[d] : 1;
        if (n_cell[d] % s->nb[d]) { delete s; return nullptr; }
    }
    s->nox = nox; s->galerkin = galerkin; s->pusher = pusher; s->solver = solver; s->cfl = cfl;
    s->dt = dt > 0 ? dt : cfl * Leaf::max_dt(solver, s->dx);
    Leaf::stencil_coefs(solver, s->dx, &s->st);
    guard_cells(*s);
    for (int bz = 0; bz < s->nb[2]; ++bz)
        for (int by = 0; by < s->nb[1]; ++by)
            for (int bx = 0; bx < s->nb[0]; ++bx) {
                s->boxes.emplace_back();
                Sim::Box& b = s->boxes.back();
                const int bi[3] = {bx, by, bz};
                for (int d = 0; d < 3; ++d) {
                    const int w = n_cell[d] / s->nb[d];
                    b.lo[d] = bi[d] * w; b.hi[d] = b.lo[d] + w - 1;
                }
                alloc_box(*s, b);
            }
    return s;
}
// ---- laser-wakefield configuration (single box; call before adding particles) ----------------
// boundary.field_lo/hi, boundary.particle_lo/hi (Utils/WarpXUtil.cpp:470-540)
int orc_sim_set_boundaries(void* h, const pic_boundaries* b) {
    Sim* s = static_cast<Sim*>(h);
    if (s->nspecies) return 1;             // (several boxes are fine here; the moving window and the antennas need one)
    s->bnd = *b;
    s->any_pec = false;
    for (int d = 0; d < 3; ++d) {
        const bool per = b->field_lo[d] == PIC_FIELD_PERIODIC;
        if (per != (b->field_hi[d] == PIC_FIELD_PERIODIC)) return 2;
        s->geom.periodic[d] = per ? 1 : 0;
        if (per) s->bnd.particle_lo[d] = s->bnd.particle_hi[d] = PIC_PARTICLE_PERIODIC;
        else if (b->particle_lo[d] == PIC_PARTICLE_PERIODIC || b->particle_hi[d] == PIC_PARTICLE_PERIODIC) return 3;
        s->any_pec = s->any_pec || b->field_lo[d] == PIC_FIELD_PEC || b->field_hi[d] == PIC_FIELD_PEC;
    }
    return 0;
}
// warpx.do_moving_window / moving_window_dir / moving_window_v (in units of c; WarpX.cpp:619-650)
int orc_sim_set_moving_window(void* h, int dir, double v_over_c) {
    Sim* s = static_cast<Sim*>(h);
    if (s->boxes.size() != 1 || s->nspecies || s->geom.periodic[dir]) return 1;
    s->do_moving_window = true; s->mw_dir = dir; s->mw_v = v_over_c * C_LIGHT;
    s->mw_x = s->geom.prob_lo[dir];
    guard_cells(*s);
    alloc_box(*s, s->boxes[0]);
    return 0;
}
// particles.use_fdtd_nci_corr: the two z stencils (NCIGodfreyFilter::ComputeStencils); grows the guard cells
int orc_sim_set_nci_corrector(void* h, const double* stencil_exeybz, const double* stencil_bxbyez) {
    Sim* s = static_cast<Sim*>(h);
    if (s->boxes.size() != 1 || s->nspecies) return 1;
    s->use_nci = true;
    for (int i = 0; i < 5; ++i) { s->nci_stencil[0][i] = stencil_exeybz[i]; s->nci_stencil[1][i] = stencil_bxbyez[i]; }
    guard_cells(*s);
    alloc_box(*s, s->boxes[0]);
    return 0;
}
int orc_nci_table_index(double cdtodz, int tab_length) { return nci_table_index(cdtodz, tab_length); }
void orc_nci_godfrey_stencil(const double* row_lo, const double* row_hi, int index, int tab_length, double cdtodz, double* out) {
    nci_godfrey_stencil(row_lo, row_hi, index, tab_length, cdtodz, out);
}
void orc_apply_nci_filter(const pic_fab* src, const pic_fab* dst, const double* stencil_z, const int* tlo, const int* thi) {
    apply_nci_filter(*src, *dst, stencil_z, tlo, thi);
}
// warpx.gamma_boost with warpx.boost_direction = z; call before adding species / lasers
int orc_sim_set_boost(void* h, double gamma_boost, double beta_boost) {
    Sim* s = static_cast<Sim*>(h);
    if (s->nspecies || !s->lasers.empty()) return 1;
    s->gamma_boost = gamma_boost; s->beta_boost = beta_boost;
    return 0;
}
// A species created by its plasma injector (PhysicalParticleContainer::InitData -> AddPlasma over
// the whole domain, PhysicalParticleContainer.cpp:450-454,855-922)
int orc_sim_add_plasma(void* h, double q, double m, const pic_plasma_injector* inj) {
    Sim* s = static_cast<Sim*>(h);
    if (s->boxes.size() != 1) return -1;
    Sim::Box& b = s->boxes[0];
    b.sp.emplace_back();
    Species& sp = b.sp.back();
    sp.q = q; sp.m = m; sp.has_injector = true; sp.inj = *inj;
    sp.inj.gamma_boost = s->gamma_boost; sp.inj.beta_boost = s->beta_boost;
    if (s->do_moving_window)                                     // WarpX.cpp:288-307
        sp.current_injection_position = s->mw_v > 0 ? s->geom.prob_hi[s->mw_dir] : s->geom.prob_lo[s->mw_dir];
    add_plasma(sp.inj, s->geom, s->dx, s->geom.prob_lo, s->geom.prob_hi, sp.a);
    sp.z_inj = sp.a[2];
    return s->nspecies++;
}
// lasers.names / <laser>.* (LaserParticleContainer ctor + InitData)
int orc_sim_add_laser(void* h, const pic_laser_antenna* prm) {
    Sim* s = static_cast<Sim*>(h);
    if (s->boxes.size() != 1) return -1;
    s->lasers.emplace_back();
    Sim::Laser& L = s->lasers.back();
    pic_laser_antenna q = *prm;
    q.gamma_boost = s->gamma_boost; q.beta_boost = s->beta_boost;
    L.ant = antenna_setup(q, s->dx);
    antenna_init_particles(L.ant, s->geom.prob_lo, s->geom.prob_hi, L.a);     // m_laser_injection_box = ProbDomain (:224)
    return (int)s->lasers.size() - 1;
}
long orc_sim_laser_np(void* h, int il) { return (long)static_cast<Sim*>(h)->lasers[il].a[0].size(); }
void orc_sim_get_laser_particles(void* h, int il, int comp, double* out) {
    auto& v = static_cast<Sim*>(h)->lasers[il].a[comp];
    std::memcpy(out, v.data(), v.size() * sizeof(double));
}
void orc_sim_laser_info(void* h, int il, double* out /* S_X S_Y mobility weight */) {
    const Antenna& a = static_cast<Sim*>(h)->lasers[il].ant;
    out[0] = a.S_X; out[1] = a.S_Y; out[2] = a.mobility; out[3] = a.weight;
}
void orc_sim_get_z_inj(void* h, int isp, double* out) {
    auto& v = static_cast<Sim*>(h)->boxes[0].sp[isp].z_inj;
    std::memcpy(out, v.data(), v.size() * sizeof(double));
}
double orc_sim_time(void* h) { return static_cast<Sim*>(h)->cur_time; }
void orc_sim_prob_domain(void* h, double* out /* lo[3] hi[3] */) {
    Sim* s = static_cast<Sim*>(h);
    for (int d = 0; d < 3; ++d) { out[d] = s->geom.prob_lo[d]; out[3 + d] = s->geom.prob_hi[d]; }
}
// ---- stage-level entry points of the laser-wakefield additions (host pointers) ---------------
void orc_apply_pec_field(const pic_fab* F, int is_E, const pic_geom* g, const pic_boundaries* b, const int* ng_fg) {
    apply_pec_field(F, is_E != 0, *g, *b, ng_fg);
}
void orc_apply_pec_current(const pic_fab* J, const pic_geom* g, const pic_boundaries* b) { apply_pec_current(J, *g, *b); }
void orc_shift_fab(const pic_fab* f, const pic_geom* g, int num_shift, int dir, double external_field) {
    shift_fab(*f, *g, num_shift, dir, external_field);
}
// AddPlasma into caller arrays (x y z w [uz]; ux = uy = 0): returns the count, -1 if capacity is too small
long orc_add_plasma(const pic_plasma_injector* inj, const pic_geom* g, const double* part_lo, const double* part_hi,
                    double* x, double* y, double* z, double* w, long capacity, double t, double* uz) {
    double dx[3];
    for (int d = 0; d < 3; ++d) dx[d] = (g->prob_hi[d] - g->prob_lo[d]) / g->n_cell[d];
    std::vector<double> out[7];
    const long n = add_plasma(*inj, *g, dx, part_lo, part_hi, out, t);
    if (n > capacity) return -1;
    for (long i = 0; i < n; ++i) { x[i] = out[0][i]; y[i] = out[1][i]; z[i] = out[2][i]; w[i] = out[3][i]; }
    if (uz) for (long i = 0; i < n; ++i) uz[i] = out[6][i];
    return n;
}
// ApplyBoundaryConditions: positions / momenta are updated in place, keep[ip] = 0 marks lost particles
void orc_apply_particle_boundaries(const pic_soa* p, const pic_geom* g, const pic_boundaries* b, char* keep) {
    std::vector<char> k;
    apply_particle_boundaries(*p, *g, *b, k);
    std::memcpy(keep, k.data(), k.size());
}
long orc_antenna_particles(const pic_laser_antenna* prm, const double* dx, const double* box_lo, const double* box_hi,
                           double* x, double* y, double* z, double* w, long capacity) {
    const Antenna a = antenna_setup(*prm, dx);
    std::vector<double> out[7];
    antenna_init_particles(a, box_lo, box_hi, out);
    const long n = (long)out[0].size();
    if (n > capacity) return -1;
    for (long i = 0; i < n; ++i) { x[i] = out[0][i]; y[i] = out[1][i]; z[i] = out[2][i]; w[i] = out[3][i]; }
    return n;
}
void orc_antenna_push(const pic_laser_antenna* prm, const double* dx, const pic_soa* p, double t, double dt) {
    const Antenna a = antenna_setup(*prm, dx);
    antenna_push(a, *p, t, dt);
}

void orc_sim_destroy(void* h) { delete static_cast<Sim*>(h); }
double orc_sim_dt(void* h) { return static_cast<Sim*>(h)->dt; }
void orc_sim_guards(void* h, int* out /* ng_EB[3], ng_J[3], ng_FG[3], ng_FS[3] */) {
    Sim* s = static_cast<Sim*>(h);
    for (int d = 0; d < 3; ++d) { out[d] = s->ng_EB[d]; out[3 + d] = s->ng_J[d]; out[6 + d] = s->ng_FG[d]; out[9 + d] = s->ng_FS[d]; }
}
int orc_sim_nboxes(void* h) { return (int)static_cast<Sim*>(h)->boxes.size(); }

// Adds a species; particles are distributed to their owning boxes.
int orc_sim_add_species(void* h, double q, double m, long np, const double* x, const double* y,
                        const double* z, const double* w, const double* ux, const double* uy,
                        const double* uz) {
    Sim* s = static_cast<Sim*>(h);
    const double* src[7] = {x, y, z, w, ux, uy, uz};
    for (auto& b : s->boxes) { b.sp.emplace_back(); b.sp.back().q = q; b.sp.back().m = m; }
    for (long ip = 0; ip < np; ++ip) {
        int owner[3];
        const double pos[3] = {x[ip], y[ip], z[ip]};
        for (int d = 0; d < 3; ++d) {
            int cell = (int)std::floor((pos[d] - s->geom.prob_lo[d]) * s->dinv[d]);
            cell = std::min(std::max(cell, 0), s->geom.n_cell[d] - 1);
            owner[d] = cell / (s->geom.n_cell[d] / s->nb[d]);
        }
        Sim::Box& b = s->boxes[owner[0] + (size_t)s->nb[0] * (owner[1] + (size_t)s->nb[1] * owner[2])];
        for (int a = 0; a < 7; ++a) b.sp.back().a[a].push_back(src[a][ip]);
    }
    return s->nspecies++;
}
// Evolve(nsteps): the last step of this call synchronises u with x (WarpXEvolve.cpp:221-226)
// when `synchronize_last` is set (what a full WarpX run does at max_step).
void orc_sim_evolve(void* h, int nsteps, int synchronize_last) {
    Sim* s = static_cast<Sim*>(h);
    for (int n = 0; n < nsteps; ++n) one_step(*s, synchronize_last && n == nsteps - 1);
}
long orc_sim_np(void* h, int isp) {
    Sim* s = static_cast<Sim*>(h); long n = 0;
    for (auto& b : s->boxes) n += (long)b.sp[isp].a[0].size();
    return n;
}
// comp: 0..6 = x y z w ux uy uz; concatenated over boxes in box order
void orc_sim_get_particles(void* h, int isp, int comp, double* out) {
    Sim* s = static_cast<Sim*>(h);
    for (auto& b : s->boxes) {
        auto& v = b.sp[isp].a[comp];
        std::memcpy(out, v.data(), v.size() * sizeof(double)); out += v.size();
    }
}
long orc_sim_box_np(void* h, int ibox, int isp) { return (long)static_cast<Sim*>(h)->boxes[ibox].sp[isp].a[0].size(); }
// field access: comp 0..8 = Ex Ey Ez Bx By Bz jx jy jz
void orc_sim_fab(void* h, int ibox, int comp, pic_fab* out) { *out = static_cast<Sim*>(h)->boxes[ibox].fab[comp]; }
double orc_sim_checksum_field(void* h, int comp) {
    Sim* s = static_cast<Sim*>(h); double t = 0;
    for (auto& b : s->boxes) t += checksum_cell_centered(b.fab[comp], b.lo, b.hi);
    return t;
}
// FieldEnergy (Diagnostics/ReducedDiags/FieldEnergy.cpp:120-144): out = {E energy, B energy}
void orc_sim_field_energy(void* h, double* out) {
    Sim* s = static_cast<Sim*>(h);
    const double dV = s->dx[0] * s->dx[1] * s->dx[2];
    double e2 = 0, b2 = 0;
    std::vector<pic_fab> fabs(s->boxes.size());
    for (int c = 0; c < 6; ++c) {
        for (size_t b = 0; b < s->boxes.size(); ++b) fabs[b] = s->boxes[b].fab[c];
        (c < 3 ? e2 : b2) += sum_squares_unique(fabs.data(), (int)fabs.size(), s->geom);
    }
    out[0] = 0.5 * e2 * EP0 * dV;
    out[1] = 0.5 * b2 / MU0 * dV;
}
// The `rho` diagnostic of a plotfile (Diagnostics/ComputeDiagFunctors/RhoFunctor.cpp:35-81): every
// container deposits into its own nodal rho with ng_depos_rho guard cells (Particles/
// WarpXParticleContainer.cpp:1287-1310; GuardCellManager.cpp:130-165) and applies the PEC / reflecting
// boundary (:1277-1283), the containers are added (Particles/MultiParticleContainer.cpp:593-612), then
// WarpX::ApplyFilterandSumBoundaryRho (Parallelization/WarpXComm.cpp:1552-1568): with the bilinear
// filter the filtered copy has stencil_length-1 more guard cells and is summed back into rho.
// Returns the checksum of the cell-centred rho (single box).
double orc_sim_rho_checksum(void* h) {
    Sim* s = static_cast<Sim*>(h);
    if (s->boxes.size() != 1) return -1.0;
    Sim::Box& b = s->boxes[0];
    int ng = 0;
    for (int d = 0; d < 3; ++d) {
        int base = s->nox;
        if (s->do_moving_window) base = std::max(base, 2);
        ng = std::max(ng, base + 1 + (int)std::ceil(C_LIGHT * s->dt / s->dx[d]));
    }
    auto make = [&](int g, std::vector<double>& store) {
        pic_fab f;
        for (int d = 0; d < 3; ++d) { f.stag[d] = 1; f.ng[d] = g; f.lo[d] = b.lo[d] - g; f.hi[d] = b.hi[d] + 1 + g; }
        store.assign((size_t)fab_size(f), 0.0);
        f.p = store.data();
        return f;
    };
    std::vector<double> tot_s, one_s, filt_s;
    pic_fab rho = make(ng, tot_s);
    double xyzmin[3]; int lo[3];
    const int ngv[3] = {ng, ng, ng};
    lower_corner(*s, b, ngv, xyzmin, lo);
    auto add_container = [&](const pic_soa& P, double q) {
        pic_fab one = make(ng, one_s);
        deposit_charge<Leaf>(P, one, s->dinv, xyzmin, lo, q, s->nox);
        if (s->any_pec) apply_pec_rho(one, s->geom, s->bnd);
        for (size_t n = 0; n < tot_s.size(); ++n) tot_s[n] += one_s[n];
    };
    for (auto& sp : b.sp) add_container(sp.soa(), sp.q);
    for (auto& L : s->lasers) add_container(laser_soa(L), 1.0);
    if (s->use_filter) {
        int ngf = ng;
        for (int d = 0; d < 3; ++d) ngf = std::max(ngf, ng + s->npass[d]);
        pic_fab rf = make(ng, filt_s);                          // per-direction growth below
        for (int d = 0; d < 3; ++d) { rf.ng[d] = ng + s->npass[d]; rf.lo[d] = b.lo[d] - rf.ng[d]; rf.hi[d] = b.hi[d] + 1 + rf.ng[d]; }
        filt_s.assign((size_t)fab_size(rf), 0.0);
        rf.p = filt_s.data();
        apply_filter(rho, rf, s->npass);
        // WarpXSumGuardCells(rho, rf, ...): rho = 0, then every point of rho receives all copies of rf
        int src_ng[3];
        for (int d = 0; d < 3; ++d) src_ng[d] = rf.ng[d];
        sum_boundary(&rf, 1, src_ng, src_ng, s->geom);
        W R(rho), F(rf);
        for (int k = rho.lo[2]; k <= rho.hi[2]; ++k)
            for (int j = rho.lo[1]; j <= rho.hi[1]; ++j)
                for (int i = rho.lo[0]; i <= rho.hi[0]; ++i) R(i, j, k) = F(i, j, k);
    } else {
        sum_boundary(&rho, 1, ngv, ngv, s->geom);
    }
    return checksum_cell_centered(rho, b.lo, b.hi);
}
int orc_deposit_charge(const pic_soa* p, const pic_fab* rho, const double* dinv, const double* xyzmin, const int* lo,
                       double q, int nox) {
    return deposit_charge<Leaf>(*p, *rho, dinv, xyzmin, lo, q, nox);
}
void orc_apply_pec_rho(const pic_fab* rho, const pic_geom* g, const pic_boundaries* b) { apply_pec_rho(*rho, *g, *b); }
void orc_particle_energy(const pic_soa* p, double mass, double* out) { particle_energy(*p, mass, out); }
// ParticleEnergy of species isp: out = {total kinetic energy [J], sum of weights}
void orc_sim_particle_energy(void* h, int isp, double* out) {
    Sim* s = static_cast<Sim*>(h);
    out[0] = out[1] = 0.0;
    for (auto& b : s->boxes) {
        double o[2];
        pic_soa P = b.sp[isp].soa();
        particle_energy(P, b.sp[isp].m, o);
        out[0] += o[0]; out[1] += o[1];
    }
}
void orc_sim_timers(void* h, double* out /* push, deposit, fdtd, halo, other */) {
    Sim* s = static_cast<Sim*>(h);
    out[0] = s->t_push; out[1] = s->t_dep; out[2] = s->t_fdtd; out[3] = s->t_halo; out[4] = s->t_other;
}
int orc_num_threads() {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
void orc_set_num_threads(int n) {
#ifdef _OPENMP
    omp_set_num_threads(n);
#else
    (void)n;
#endif
}

}  // extern "C"
