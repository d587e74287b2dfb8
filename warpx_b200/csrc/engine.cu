// C++ host driver of the PIC step: the sequence of WarpX::Evolve / OneStep_nosub for a single-level,
// periodic, explicit FDTD run on ONE rank, expressed as calls through the C ABI of this library.
//
// Mirrors (paths relative to Source/ of ECP-WarpX/WarpX):
//   pic_engine_evolve            <- WarpX::Evolve                          Evolve/WarpXEvolve.cpp:93-347
//   explicit_fill_boundary_eb    <- ExplicitFillBoundaryEBUpdateAux        :473-531
//   one_step_nosub               <- WarpX::OneStep_nosub                   :353-455
//   push_particles_and_deposit   <- MultiParticleContainer::Evolve         Particles/MultiParticleContainer.cpp:460-482
//                                   PhysicalParticleContainer::Evolve      Particles/PhysicalParticleContainer.cpp:1812-2095
//   sync_current                 <- WarpX::SyncCurrent / SumBoundaryJ      Parallelization/WarpXComm.cpp:1073-1240,1386-1424
//   synchronize                  <- WarpX::Synchronize                     Evolve/WarpXEvolve.cpp:64-91
//   handle_particles_at_boundaries <- WarpX::HandleParticlesAtBoundaries   :533-581
//   guard cells                  <- guardCellManager::Init                 Parallelization/GuardCellManager.cpp:62-161,310-343
//   dt                           <- WarpX::ComputeDt                       Evolve/WarpXComputeDt.cpp:56-95
// All memory is borrowed from the caller (fields, particle SoA double buffers, bins, sort scratch);
// every stage is an asynchronous launch on the caller's stream.
// Non-periodic domains (pic_engine_set_boundaries / set_moving_window / set_injector / add_laser, one
// rank): PEC walls after every field push and on J (BoundaryConditions/WarpXFieldBoundaries.cpp:51-190),
// WarpX::MoveWindow with continuous injection (Utils/WarpXMovingWindow.cpp:139-476), laser antennas
// (Particles/LaserParticleContainer.cpp:563-700), absorbing / reflecting particle boundaries
// (Particles/WarpXParticleContainer.cpp:1574-1638) -- the additions of the laser-wakefield decks.
// Multi-rank (one process per GPU, one brick per rank, pic_engine_set_comm): the guard-cell
// exchanges and the particle migration go through NCCL send/recv on the same stream (csrc/comm.cu),
// as three axis sweeps with two neighbours each; the host reads 32 bytes once per step (new particle
// count, overflow status, peak migration count).  warpx_b200/engine.py keeps a Python mirror of the
// same sequence (torch.distributed transport) for per-stage timing and as a cross-check.
#include "pic_common.cuh"
#include "comm.cuh"
#include <cmath>
#include <atomic>
#include <vector>

namespace pic {

struct Species {
    double q, m;
    pic_soa buf[2];        // counting sort permutes buf[cur] -> buf[1-cur]
    int cur;
    pic_bins bins;
    bool has_bins;
    void* sort_work;
    pic_escape_list esc;   // particles the last position push moved out of the domain -- over several ranks: out of
    bool has_esc;          // the rank's brick (engine-owned)
    bool esc_valid = false;  // the list describes the current particle order (set by the push, cleared by whatever reorders)
    // neighbour migration (multi-rank), engine-owned device scratch
    long capacity = 0;           // entries of every SoA array of both buffers
    int mig_cap_max = 0, mig_cap = 0;
    int* mig_counts = nullptr;   // [2]
    int* mig_idx[2] = {nullptr, nullptr};
    double* mig_msg[4] = {nullptr, nullptr, nullptr, nullptr};   // send lo/hi, recv lo/hi
    int* mig_work = nullptr;
    int* mig_head = nullptr;     // pinned host, 8 ints
    // plasma injector (continuous injection behind the moving window) and absorbing boundaries
    bool has_injector = false;
    pic_plasma_injector inj{};
    double current_injection_position = 0.0;     // WarpXParticleContainer::m_current_injection_position
    uint64_t next_id = 0;
    int* bnd_work = nullptr;     // pic_particles_boundary_workspace_ints(bnd_cap) ints, engine-owned
    int bnd_cap = 0;
    bool bins_stale = false;     // particles were removed / the window moved: re-sort before the next step
};

// Laser antenna: its own particle container (LaserParticleContainer), no gather, order-agnostic deposit
struct Laser {
    pic_laser_antenna prm;
    pic_soa P;                   // borrowed device arrays, P.np particles
    long capacity;
    int* bnd_work = nullptr;
    int bnd_cap = 0;
    double* w_owned = nullptr;   // multi-rank: weights masked to this rank's brick (engine-owned)
};

// Per-stage CUDA-event timing of the step driver (pic_engine_enable_timing / pic_engine_stage_ms): the events are
// recorded on the stream the stages are launched on, inside the same pic_engine_evolve calls a benchmark times.
enum { ST_FILL_EB = 0, ST_GATHER_PUSH, ST_ZERO_J, ST_DEPOSIT, ST_SYNC_J, ST_EVOLVE_B, ST_FILL_B, ST_EVOLVE_E, ST_FILL_E,
       ST_WRAP, ST_MIGRATE, ST_SORT, ST_NCI, ST_WINDOW, ST_PUSHP, ST_FILTER, ST_FLUID, ST_COUNT };
static const char* const stage_names[ST_COUNT] = {"fill_boundary_eb", "gather_push", "zero_j", "deposit", "sync_current",
    "evolve_b", "fill_boundary_b", "evolve_e", "fill_boundary_e", "wrap", "migrate", "sort", "nci_filter", "move_window", "push_p", "filter_j",
    "fluid"};
// Cold fluid species (WarpXFluidContainer): two borrowed states of N, NUx, NUy, NUz; the advection writes one from the
// other and `cur` names the current one.
struct Fluid {
    double q, m;
    pic_fab U[2][4];
    int cur = 0;
};

struct StageRec { int st; cudaEvent_t a, b; };
struct Timing {
    bool on = false;
    std::vector<cudaEvent_t> pool;
    size_t used = 0;
    std::vector<StageRec> recs;
    double ms[ST_COUNT] = {};
    long calls[ST_COUNT] = {};
    cudaEvent_t get() {
        if (used == pool.size()) { cudaEvent_t ev = nullptr; cudaEventCreate(&ev); pool.push_back(ev); }
        return pool[used++];
    }
};

struct Engine {
    Timing tm;
    pic_geom geom;
    int box_lo[3], box_hi[3];
    int nox, galerkin, pusher, solver, sort_interval;
    double dx[3], dinv[3], dt;
    int ng_EB[3], ng_J[3], ng_FG[3], ng_FS[3];
    int use_filter = 0, npass[3] = {1, 1, 1};   // warpx.use_filter / filter_npass_each_dir
    // With the filter the particles deposit into the engine's own copies of J and ApplyFilterJ writes from there
    // straight into the caller's arrays (no copy back): jdep[c] = fab[6 + c] with its own memory.
    pic_fab jdep[3];
    bool jdep_alloc = false;
    pic_stencil st;
    pic_fab fab[9];        // Ex Ey Ez Bx By Bz jx jy jz
    std::vector<Species> species;
    bool is_synchronized = true;
    long istep = 0;
    // multi-rank
    Comm* comm = nullptr;
    int nb[3] = {1, 1, 1}, coord[3] = {0, 0, 0};
    double* hbuf[4] = {nullptr, nullptr, nullptr, nullptr};      // halo send lo/hi, recv lo/hi
    size_t hbuf_doubles = 0;
    // non-periodic domains
    pic_boundaries bnd{};
    bool any_pec = false, all_periodic = true;
    bool do_moving_window = false;
    int mw_dir = 2;
    double mw_v = 0.0, mw_x = 0.0;               // moving_window_v [m/s], moving_window_x
    double gamma_boost = 1.0, beta_boost = 0.0;  // warpx.gamma_boost, boost_direction = z
    bool use_nci = false;                        // particles.use_fdtd_nci_corr
    double nci_stencil[2][5];                    // [0] Ex Ey Bz, [1] Bx By Ez
    pic_fab nci_fab[6];                          // filtered copies of E, B (engine-owned)
    bool nci_alloc = false;
    double cur_time = 0.0;                       // t_new[0]
    double* shift_tmp = nullptr;                 // one component-sized scratch array
    size_t shift_tmp_bytes = 0;
    int* host_count = nullptr;                   // pinned host int (particles lost per boundary pass)
    std::vector<Laser> lasers;
    std::vector<Fluid> fluids;
};

struct Stage {      // records the events of one stage when timing is on
    Engine& e; int st; cudaStream_t s; cudaEvent_t a = nullptr;
    Stage(Engine& e_, int st_, void* s_) : e(e_), st(st_), s((cudaStream_t)s_) {
#ifndef PIC_SIMT_HOST
        if (e.tm.on) { a = e.tm.get(); cudaEventRecord(a, s); }
#endif
    }
    ~Stage() {
#ifndef PIC_SIMT_HOST
        if (a) { cudaEvent_t b = e.tm.get(); cudaEventRecord(b, s); e.tm.recs.push_back({st, a, b}); }
#endif
    }
};
// fold the recorded events into the per-stage sums (synchronises on the last event)
static void collect_timing(Engine& e) {
#ifndef PIC_SIMT_HOST
    for (const StageRec& r : e.tm.recs) {
        float ms = 0.f;
        cudaEventSynchronize(r.b);
        if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) { e.tm.ms[r.st] += ms; e.tm.calls[r.st] += 1; }
    }
#endif
    e.tm.recs.clear();
    e.tm.used = 0;
}

static bool spans(const Engine& e, int dim) { return e.comm == nullptr || e.nb[dim] == 1; }
static int neighbour(const Engine& e, int dim, int side) {
    int c[3] = {e.coord[0], e.coord[1], e.coord[2]};
    c[dim] = (c[dim] + (side ? 1 : -1) + e.nb[dim]) % e.nb[dim];
    return c[0] + e.nb[0] * (c[1] + e.nb[1] * c[2]);
}

// A brick at a non-periodic domain face has no neighbour beyond it.
static bool has_neighbour(const Engine& e, int dim, int side) {
    if (e.geom.periodic[dim]) return true;
    const int c = e.coord[dim] + (side ? 1 : -1);
    return c >= 0 && c < e.nb[dim];
}

#define ENG_NCCL(x) do { if (int rc_ = (x)) return nccl_fail("pic_engine", rc_); } while (0)

// Low/high neighbour exchange along one axis.  A message travelling upwards (sent to hi, received
// from lo) is posted first on both sides: with two bricks per axis both neighbours are the same
// rank and NCCL matches sends and receives of a pair of ranks in posting order.
static int exchange(Engine& e, int dim, const double* s_lo, const double* s_hi, double* r_lo, double* r_hi,
                    size_t n, cudaStream_t s) {
    const int lo = neighbour(e, dim, 0), hi = neighbour(e, dim, 1);
    ENG_NCCL(g_nccl.GroupStart());
    ENG_NCCL(g_nccl.Send(s_hi, n, PIC_NCCL_FLOAT64, hi, e.comm->comm, s));
    ENG_NCCL(g_nccl.Recv(r_lo, n, PIC_NCCL_FLOAT64, lo, e.comm->comm, s));
    ENG_NCCL(g_nccl.Send(s_lo, n, PIC_NCCL_FLOAT64, lo, e.comm->comm, s));
    ENG_NCCL(g_nccl.Recv(r_hi, n, PIC_NCCL_FLOAT64, hi, e.comm->comm, s));
    ENG_NCCL(g_nccl.GroupEnd());
    return 0;
}

// The same exchange along a NON-periodic axis: the bricks at the domain faces skip the missing side.
static int exchange_np(Engine& e, int dim, const double* s_lo, const double* s_hi, double* r_lo, double* r_hi,
                       size_t n, cudaStream_t s) {
    const bool hl = has_neighbour(e, dim, 0), hh = has_neighbour(e, dim, 1);
    const int lo = neighbour(e, dim, 0), hi = neighbour(e, dim, 1);
    ENG_NCCL(g_nccl.GroupStart());
    if (hh) ENG_NCCL(g_nccl.Send(s_hi, n, PIC_NCCL_FLOAT64, hi, e.comm->comm, s));
    if (hl) ENG_NCCL(g_nccl.Recv(r_lo, n, PIC_NCCL_FLOAT64, lo, e.comm->comm, s));
    if (hl) ENG_NCCL(g_nccl.Send(s_lo, n, PIC_NCCL_FLOAT64, lo, e.comm->comm, s));
    if (hh) ENG_NCCL(g_nccl.Recv(r_hi, n, PIC_NCCL_FLOAT64, hi, e.comm->comm, s));
    ENG_NCCL(g_nccl.GroupEnd());
    return 0;
}

static void stencil_coefficients(int solver, const double dx[3], pic_stencil* st) {
    // FiniteDifferenceSolver ctor: Yee CartesianYeeAlgorithm.H:30-42, CKC CartesianCKCAlgorithm.H:31-101
    st->algo = solver;
    for (int n = 0; n < 5; ++n) st->cx[n] = st->cy[n] = st->cz[n] = 0.0;
    const double ix = 1.0 / dx[0], iy = 1.0 / dx[1], iz = 1.0 / dx[2];
    st->cx[0] = ix; st->cy[0] = iy; st->cz[0] = iz;
    if (solver != PIC_SOLVER_CKC) return;
    const double delta = fmax(ix, fmax(iy, iz));
    const double rx = (ix / delta) * (ix / delta), ry = (iy / delta) * (iy / delta), rz = (iz / delta) * (iz / delta);
    const double beta = 0.125 * (1.0 - rx * ry * rz / (ry * rz + rz * rx + rx * ry));
    const double irf = 1.0 / (ry * rz + rz * rx + rx * ry);
    const double gx = ry * rz * (0.0625 - 0.125 * ry * rz * irf);
    const double gy = rx * rz * (0.0625 - 0.125 * rx * rz * irf);
    const double gz = rx * ry * (0.0625 - 0.125 * rx * ry * irf);
    st->cx[1] = (1.0 - 2.0 * ry * beta - 2.0 * rz * beta - 4.0 * gx) * ix;
    st->cy[1] = (1.0 - 2.0 * rx * beta - 2.0 * rz * beta - 4.0 * gy) * iy;
    st->cz[1] = (1.0 - 2.0 * rx * beta - 2.0 * ry * beta - 4.0 * gz) * iz;
    st->cx[2] = ry * beta * ix; st->cx[3] = rz * beta * ix; st->cx[4] = gx * ix;
    st->cy[2] = rz * beta * iy; st->cy[3] = rx * beta * iy; st->cy[4] = gy * iy;
    st->cz[2] = rx * beta * iz; st->cz[3] = ry * beta * iz; st->cz[4] = gz * iz;
}

static double max_dt(int solver, const double dx[3]) {
    if (solver == PIC_SOLVER_YEE)
        return 1.0 / (sqrt(1.0 / (dx[0] * dx[0]) + 1.0 / (dx[1] * dx[1]) + 1.0 / (dx[2] * dx[2])) * C_LIGHT);
    return fmin(dx[0], fmin(dx[1], dx[2])) / C_LIGHT;
}

static void guard_cells(Engine& e) {
    for (int d = 0; d < 3; ++d) {
        const int ngt = e.nox;
        int ng = (ngt % 2) ? ngt + 1 : ngt;
        int ngJ = ngt;
        if (e.use_nci && d == 2) { const int n4 = ngt + 4; ng = (n4 % 2) ? n4 + 1 : n4; }   // GuardCellManager.cpp:87-90 (m_stencil_width = 4)
        if (e.do_moving_window) { ng = ng > 2 ? ng : 2; ngJ = ngJ > 2 ? ngJ : 2; }   // GuardCellManager.cpp:103-115
        e.ng_J[d] = ngJ + (int)ceil(C_LIGHT * 0.5 * e.dt / e.dx[d]);
        if (e.use_filter) e.ng_J[d] += e.npass[d];     // + stencil_length - 1, GuardCellManager.cpp:169-172
        e.ng_FS[d] = 1;
        ng = ng > e.ng_FS[d] ? ng : e.ng_FS[d];
        e.ng_EB[d] = ng;
        int fg = (e.nox + 1) / 2;
        fg = fg < ng ? fg : ng;
        if (e.use_nci && d == 2) { fg += 4; fg = fg < ng ? fg : ng; }   // :319-330
        e.ng_FG[d] = fg > e.ng_FS[d] ? fg : e.ng_FS[d];
    }
}

static void lower_corner(const Engine& e, const int ng[3], double xyzmin[3], int lo[3]) {
    // WarpX::LowerCorner of the box grown by ng (WarpX.cpp:2851-2874): prob_lo + index * dx
    for (int d = 0; d < 3; ++d) {
        lo[d] = e.box_lo[d] - ng[d];
        xyzmin[d] = e.geom.prob_lo[d] + e.dx[d] * lo[d];
    }
}

#define ENG_CALL(x) do { if (int rc_ = (x)) return rc_; } while (0)

// The four halo message buffers hold at least n doubles each.  A failed allocation leaves the engine without
// buffers (size 0, null pointers) instead of dangling ones: a later sweep allocates again or fails cleanly.
static int grow_halo_buffers(Engine& e, size_t n) {
    if (n <= e.hbuf_doubles) return 0;
    e.hbuf_doubles = 0;
    for (int b = 0; b < 4; ++b) { if (e.hbuf[b]) cudaFree(e.hbuf[b]); e.hbuf[b] = nullptr; }
    for (int b = 0; b < 4; ++b)
        if (cudaMalloc(&e.hbuf[b], sizeof(double) * n) != cudaSuccess) {
            cudaGetLastError();
            for (int c = 0; c < 4; ++c) { if (e.hbuf[c]) cudaFree(e.hbuf[c]); e.hbuf[c] = nullptr; }
            return fail("pic_engine: halo buffer allocation failed");
        }
    e.hbuf_doubles = n;
    return 0;
}

// One axis sweep of FillBoundary (mode 0) / SumBoundary (mode 1) over nfab components: local kernels
// when this rank spans the periodic domain along dim, otherwise pack -> NCCL -> unpack(+add) with
// one message per direction carrying the slabs of all components.
// all_guards: the refresh after SumBoundary also covers the guards beyond a non-periodic face (they are
// part of SumBoundary's destination); a plain FillBoundary leaves them alone (see pic_fill_boundary_local).
static int halo_sweep(Engine& e, const pic_fab* fabs, int nfab, int dim, int ng, int mode, void* s, bool all_guards = false) {
    if (ng == 0 && mode == 0) return 0;
    if (!e.geom.periodic[dim]) {
        if (spans(e, dim)) return 0;         // the box spans the domain: no image, the guards beyond the faces keep their values
        // slabs along a non-periodic axis: per-side pack / unpack, the face bricks skip the missing side
        size_t n = 0;
        for (int c = 0; c < nfab; ++c) n += (size_t)pic_halo_slab_count(&fabs[c], dim, ng, mode);
        if (n == 0) return 0;
        ENG_CALL(grow_halo_buffers(e, n));
        for (int side = 0; side < 2; ++side) {
            if (!has_neighbour(e, dim, side)) continue;
            size_t off = 0;
            for (int c = 0; c < nfab; ++c) {
                ENG_CALL(pic_halo_pack(&fabs[c], dim, side, ng, mode, e.hbuf[side] + off, s));
                off += (size_t)pic_halo_slab_count(&fabs[c], dim, ng, mode);
            }
        }
        ENG_CALL(exchange_np(e, dim, e.hbuf[0], e.hbuf[1], e.hbuf[2], e.hbuf[3], n, (cudaStream_t)s));
        for (int side = 0; side < 2; ++side) {
            if (!has_neighbour(e, dim, side)) continue;
            size_t off = 0;
            for (int c = 0; c < nfab; ++c) {
                ENG_CALL(pic_halo_unpack(&fabs[c], dim, side, ng, mode, e.hbuf[2 + side] + off, s));
                off += (size_t)pic_halo_slab_count(&fabs[c], dim, ng, mode);
            }
        }
        return 0;
    }
    if (spans(e, dim)) {
        pic_geom gfull = e.geom;
        if (all_guards) gfull.periodic[0] = gfull.periodic[1] = gfull.periodic[2] = 1;
        // all components of the exchange in one launch
        return pic_boundary_local_multi(fabs, nfab, dim, ng, mode, (mode == 0 && all_guards) ? &gfull : &e.geom, s);
    }
    size_t n = 0;
    for (int c = 0; c < nfab; ++c) n += (size_t)pic_halo_slab_count(&fabs[c], dim, ng, mode);
    ENG_CALL(grow_halo_buffers(e, n));
    ENG_CALL(pic_halo_pack_multi(fabs, nfab, dim, ng, mode, e.hbuf[0], e.hbuf[1], s));
    ENG_CALL(exchange(e, dim, e.hbuf[0], e.hbuf[1], e.hbuf[2], e.hbuf[3], n, (cudaStream_t)s));
    ENG_CALL(pic_halo_unpack_multi(fabs, nfab, dim, ng, mode, e.hbuf[2], e.hbuf[3], s));
    return 0;
}

static int fill_boundary(Engine& e, int c0, int c1, const int ng[3], void* s, bool all_guards = false) {
    for (int d = 0; d < 3; ++d) ENG_CALL(halo_sweep(e, &e.fab[c0], c1 - c0, d, ng[d], 0, s, all_guards));
    return 0;
}

// PIC_HALO_TWO_PASS=1: SumBoundary and the refresh of J as two exchanges per axis (the round-1 path), for comparison
static const bool g_halo_two_pass = [] { const char* v = getenv("PIC_HALO_TWO_PASS"); return v && atoi(v) != 0; }();

static std::atomic<long> g_fused_sum_exchanges{0};
extern "C" long pic_engine_fused_sum_exchanges(void) { return g_fused_sum_exchanges.load(); }

static int sync_current(Engine& e, void* s) {
    // (WarpX::ApplyFilterJ, WarpXComm.cpp:1357-1374 -- filter over the grown box into a temporary, copy back -- ran just
    //  before as its own stage: the temporary is where the particles deposited, the result landed in J itself)
    // Between two ranks along a periodic axis both passes are ONE exchange (halo.cu, mode 2: each rank sends the whole
    // overlap zone and adds what it receives): three exchanges less per step on a 2 x 2 x 2 brick grid.
    bool fused[3];
    for (int d = 0; d < 3; ++d) {
        fused[d] = e.geom.periodic[d] && !spans(e, d) && !g_halo_two_pass;
        for (int c = 6; c < 9 && fused[d]; ++c)
            fused[d] = 2 * e.ng_J[d] + e.fab[c].stag[d] <= e.box_hi[d] - e.box_lo[d] + 1;
        if (fused[d]) ++g_fused_sum_exchanges;
        ENG_CALL(halo_sweep(e, &e.fab[6], 3, d, e.ng_J[d], fused[d] ? 2 : 1, s));
    }
    for (int d = 0; d < 3; ++d)
        if (!fused[d]) ENG_CALL(halo_sweep(e, &e.fab[6], 3, d, e.ng_J[d], 0, s, true));
    // reflect J over PEC / reflecting boundaries (WarpX::SyncCurrentAndRho, WarpXEvolve.cpp:629-640)
    if (!e.all_periodic) ENG_CALL(pic_apply_pec_current(&e.fab[6], &e.geom, &e.bnd, s));
    return 0;
}

static int push(Engine& e, Species& sp, double dt, int push_position, void* s) {
    double xyzmin[3]; int lo[3];
    lower_corner(e, e.ng_EB, xyzmin, lo);
    const pic_soa& P = sp.buf[sp.cur];
    if (push_position && sp.has_esc) {
        cudaMemsetAsync(sp.esc.count, 0, sizeof(int), (cudaStream_t)s);
        // Over several ranks the push lists what leaves the BRICK (a superset by 1e-6 cell, so that round-off at a face
        // cannot hide a particle from the classification, which decides by cell index): the periodic wrap and the
        // migration sweeps then visit the listed particles only.  The domain moves with the window: set every step.
        for (int d = 0; d < 3; ++d) {
            const double eps = 1e-6 * e.dx[d];
            if (!spans(e, d)) {
                sp.esc.lo[d] = e.geom.prob_lo[d] + e.dx[d] * e.box_lo[d] + eps;
                sp.esc.hi[d] = e.geom.prob_lo[d] + e.dx[d] * (e.box_hi[d] + 1) - eps;
            } else {
                sp.esc.lo[d] = e.geom.periodic[d] ? e.geom.prob_lo[d] : -INFINITY;
                sp.esc.hi[d] = e.geom.periodic[d] ? e.geom.prob_hi[d] : INFINITY;
            }
        }
        sp.esc_valid = true;
    }
    // the main push gathers from the NCI-filtered copies (PhysicalParticleContainer.cpp:1900-1911); PushP does not
    const pic_fab* EB = (e.use_nci && push_position) ? e.nci_fab : e.fab;
    return pic_gather_push(&P, 0, P.np, &EB[0], &EB[3], e.dinv, xyzmin, lo, sp.q, sp.m, dt, e.nox,
                           e.galerkin, e.pusher, push_position, sp.has_bins ? &sp.bins : nullptr,
                           sp.has_esc ? &sp.esc : nullptr, s);
}

// PhysicalParticleContainer::applyNCIFilter for the rank's box (one tile): E, B -> the engine's filtered copies
static int apply_nci(Engine& e, void* s) {
    if (!e.nci_alloc) {
        for (int c = 0; c < 6; ++c) {
            e.nci_fab[c] = e.fab[c];
            e.nci_fab[c].p = nullptr;
            if (cudaMalloc(&e.nci_fab[c].p, sizeof(double) * (size_t)fab_size(e.fab[c])) != cudaSuccess)
                return fail("pic_engine: cannot allocate the NCI-filtered field copies");
            cudaMemsetAsync(e.nci_fab[c].p, 0, sizeof(double) * (size_t)fab_size(e.fab[c]), (cudaStream_t)s);
        }
        e.nci_alloc = true;
    }
    for (int c = 0; c < 6; ++c) {
        const bool exeybz = (c == 0 || c == 1 || c == 5);              // :2132-2163
        ENG_CALL(pic_apply_nci_filter(&e.fab[c], &e.nci_fab[c], e.nci_stencil[exeybz ? 0 : 1], e.box_lo, e.box_hi, e.nox, s));
    }
    return 0;
}

static int push_particles_and_deposit(Engine& e, void* s) {
    {
        Stage t(e, ST_ZERO_J, s);
        if (e.use_filter && !e.jdep_alloc) {
            for (int c = 0; c < 3; ++c) {
                e.jdep[c] = e.fab[6 + c];
                e.jdep[c].p = nullptr;
                if (cudaMalloc(&e.jdep[c].p, sizeof(double) * (size_t)fab_size(e.fab[6 + c])) != cudaSuccess)
                    return fail("pic_engine: cannot allocate the deposition copy of J (filter)");
            }
            e.jdep_alloc = true;
        }
        const pic_fab* Jd = e.use_filter ? e.jdep : &e.fab[6];
        for (int c = 0; c < 3; ++c)                     // J.setVal(0), MultiParticleContainer.cpp:467-478
            cudaMemsetAsync(Jd[c].p, 0, sizeof(double) * (size_t)fab_size(Jd[c]), (cudaStream_t)s);
    }
    const pic_fab* Jd = e.use_filter ? e.jdep : &e.fab[6];
    double xyzmin[3]; int lo[3];
    lower_corner(e, e.ng_J, xyzmin, lo);
    if (e.use_nci && !e.species.empty()) { Stage t(e, ST_NCI, s); ENG_CALL(apply_nci(e, s)); }
    for (auto& sp : e.species) {
        { Stage t(e, ST_GATHER_PUSH, s); ENG_CALL(push(e, sp, e.dt, 1, s)); }
        const pic_soa& P = sp.buf[sp.cur];
        Stage t(e, ST_DEPOSIT, s);
        ENG_CALL(pic_deposit_esirkepov(&P, 0, P.np, Jd, e.dinv, xyzmin, lo, sp.q, e.dt, -0.5 * e.dt,
                                       e.nox, sp.has_bins ? &sp.bins : nullptr, s));
    }
    // the antennas come after the species in allcontainers (MultiParticleContainer.cpp:60-75);
    // LaserParticleContainer::Evolve (:563-700): push at t^n, deposit with charge = 1 (:88)
    // Over several ranks every rank carries the whole antenna (a few thousand particles, pushed
    // identically everywhere) and deposits the particles inside its own brick.
    for (auto& L : e.lasers) {
        if (L.P.np == 0) continue;
        ENG_CALL(pic_laser_antenna_push(&L.prm, e.dx, &L.P, e.cur_time, e.dt, s));
        pic_soa dep = L.P;
        if (e.comm) {
            double own_lo[3], own_hi[3];
            for (int d = 0; d < 3; ++d) {
                own_lo[d] = (e.nb[d] == 1 || !has_neighbour(e, d, 0)) ? -INFINITY : e.geom.prob_lo[d] + e.dx[d] * e.box_lo[d];
                own_hi[d] = (e.nb[d] == 1 || !has_neighbour(e, d, 1)) ? INFINITY : e.geom.prob_lo[d] + e.dx[d] * (e.box_hi[d] + 1);
            }
            ENG_CALL(pic_particles_owned_weights(&L.P, own_lo, own_hi, L.w_owned, s));
            dep.w = L.w_owned;
        }
        ENG_CALL(pic_deposit_esirkepov(&dep, 0, dep.np, Jd, e.dinv, xyzmin, lo, 1.0, e.dt, -0.5 * e.dt,
                                       e.nox, nullptr, s));
    }
    return 0;
}

static int sort_species(Engine& e, Species& sp, void* s) {
    pic_soa& in = sp.buf[sp.cur];
    pic_soa& out = sp.buf[1 - sp.cur];
    out.np = in.np;
    for (int d = 0; d < 3; ++d) { sp.bins.box_lo[d] = e.box_lo[d]; sp.bins.box_hi[d] = e.box_hi[d]; }
    ENG_CALL(pic_sort_particles_by_cell(&in, &out, &e.geom, &sp.bins, sp.sort_work, s));
    sp.bins.np_binned = in.np;
    sp.cur = 1 - sp.cur;
    sp.has_bins = true;
    sp.esc_valid = false;
    return 0;
}

__global__ void peak_kernel(int* peak, const int* counts) { *peak = max(*peak, max(counts[0], counts[1])); }

// Neighbour migration after the periodic wrap (AMReX RedistributeLocal(1), WarpXEvolve.cpp:550-559):
// axis sweeps, classify -> pack into fixed-size messages -> NCCL -> arrivals fill the holes
// (csrc/migrate.cu).  The particle count stays on the device (work[0]) while the sweeps chain; the
// host reads {count, status, peak per-face count} once.  Every rank sizes the next step's messages
// from the all-reduced peak (8x headroom); the first step uses the worst case (one layer of cells).
// PIC_MIGRATE_FULL_SWEEP=1: classify every particle in every axis sweep (the round-1 path), for comparison
static const bool g_migrate_full_sweep = [] { const char* v = getenv("PIC_MIGRATE_FULL_SWEEP"); return v && atoi(v) != 0; }();

static std::atomic<long> g_listed_sweeps{0};
extern "C" long pic_engine_listed_sweeps(void) { return g_listed_sweeps.load(); }

static int migrate(Engine& e, Species& sp, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    pic_soa& P = sp.buf[sp.cur];
    const int cap = sp.mig_cap;
    const size_t nmsg = (size_t)pic_migrate_message_doubles(cap);
    for (int n = 0; n < 8; ++n) sp.mig_head[n] = 0;
    sp.mig_head[0] = (int)P.np;
    cudaMemcpyAsync(sp.mig_work, sp.mig_head, 8 * sizeof(int), cudaMemcpyHostToDevice, s);
    const int* np_dev = sp.mig_work;
    pic_soa view = P;
    view.np = sp.capacity;                       // launch bound only: the kernels read the count from np_dev
    // Who can leave: the particles the push of this step listed (nothing else moved since: periodic particle boundaries
    // remove nobody, no window shift re-drew the brick) -- else every particle is classified.
    const bool listed = sp.has_esc && sp.esc_valid && e.all_periodic && !e.do_moving_window && !g_migrate_full_sweep;
    for (int dim = 0; dim < 3; ++dim) {
        if (spans(e, dim)) continue;
        const bool np_dim = !e.geom.periodic[dim];
        if (listed) ++g_listed_sweeps;
        if (listed)
            ENG_CALL(pic_particles_classify_listed(&view, &e.geom, dim, e.box_lo[dim], e.box_hi[dim],
                                                   np_dim ? 2 : (e.nb[dim] == 2 ? 1 : 0), sp.mig_counts, sp.mig_idx[0],
                                                   sp.mig_idx[1], cap, np_dev, &sp.esc, s));
        else
        ENG_CALL(pic_particles_classify(&view, &e.geom, dim, e.box_lo[dim], e.box_hi[dim],
                                        np_dim ? 2 : (e.nb[dim] == 2 ? 1 : 0),
                                        sp.mig_counts, sp.mig_idx[0], sp.mig_idx[1], cap, np_dev, s));
        peak_kernel<<<1, 1, 0, s>>>(sp.mig_work + 6, sp.mig_counts);
        count_launch();
        ENG_CALL(pic_migrate_pack(&view, sp.mig_idx[0], sp.mig_counts, cap, sp.mig_msg[0], s));
        ENG_CALL(pic_migrate_pack(&view, sp.mig_idx[1], sp.mig_counts + 1, cap, sp.mig_msg[1], s));
        if (np_dim) {
            // a missing neighbour sends nothing: its message reads "0 particles"
            for (int side = 0; side < 2; ++side)
                if (!has_neighbour(e, dim, side)) cudaMemsetAsync(sp.mig_msg[2 + side], 0, sizeof(double), s);
            ENG_CALL(exchange_np(e, dim, sp.mig_msg[0], sp.mig_msg[1], sp.mig_msg[2], sp.mig_msg[3], nmsg, s));
        } else
        ENG_CALL(exchange(e, dim, sp.mig_msg[0], sp.mig_msg[1], sp.mig_msg[2], sp.mig_msg[3], nmsg, s));
        ENG_CALL(pic_migrate_unpack(&view, sp.mig_counts, sp.mig_idx[0], sp.mig_idx[1], sp.mig_msg[2], sp.mig_msg[3], cap,
                                    sp.capacity, sp.mig_work, np_dev, s));
        if (listed) ENG_CALL(pic_migrate_note_appended(sp.mig_work, &sp.esc, s));     // arrivals may have to travel on
    }
    sp.esc_valid = false;            // holes were filled, tails moved: the list is spent
    ENG_NCCL(g_nccl.AllReduce(sp.mig_work + 6, sp.mig_work + 6, 1, PIC_NCCL_INT32, PIC_NCCL_MAX, e.comm->comm, s));
    cudaMemcpyAsync(sp.mig_head, sp.mig_work, 8 * sizeof(int), cudaMemcpyDeviceToHost, s);
    if (cudaStreamSynchronize(s) != cudaSuccess) return fail("pic_engine: migration failed (%s)", cudaGetErrorString(cudaGetLastError()));
    const int np_new = sp.mig_head[0], status = sp.mig_head[1], seen = sp.mig_head[6];
    if (status)
        return fail("pic_engine: particle migration overflow on rank %d (status %d, %d particles through one face, "
                    "message capacity %d, tile capacity %ld)", e.comm->rank, status, seen, cap, sp.capacity);
    P.np = np_new;
    long want = 16384;
    while (want < 8L * seen + 1024) want *= 2;
    // A window shift sends one whole layer of cells to the slab below, also right after steps that saw only
    // thermal crossers (c dt < dz: most steps do not shift): the capacity stays at the layer bound then.
    if (e.do_moving_window && e.nb[e.mw_dir] > 1) want = sp.mig_cap_max;
    sp.mig_cap = (int)(want < sp.mig_cap_max ? want : sp.mig_cap_max);
    return 0;
}

// WarpX::EvolveB / EvolveE end with ApplyBfieldBoundary / ApplyEfieldBoundary
// (FieldSolver/WarpXPushFieldsEM.cpp:926,990): PEC over the valid points grown by ng_FieldGather.
static int evolve_b(Engine& e, double dt, void* s) {
    ENG_CALL(pic_evolve_b(&e.fab[3], &e.fab[0], &e.st, dt, s));
    if (e.any_pec) ENG_CALL(pic_apply_pec_field(&e.fab[3], 0, &e.geom, &e.bnd, e.ng_FG, s));
    return 0;
}
static int evolve_e(Engine& e, double dt, void* s) {
    ENG_CALL(pic_evolve_e(&e.fab[0], &e.fab[3], &e.fab[6], &e.st, dt, s));
    if (e.any_pec) ENG_CALL(pic_apply_pec_field(&e.fab[0], 1, &e.geom, &e.bnd, e.ng_FG, s));
    return 0;
}

static int shift_component(Engine& e, int c, int num_shift, void* s) {
    const size_t bytes = sizeof(double) * (size_t)fab_size(e.fab[c]);
    if (bytes > e.shift_tmp_bytes) {
        if (e.shift_tmp) cudaFree(e.shift_tmp);
        if (cudaMalloc(&e.shift_tmp, bytes) != cudaSuccess) return fail("pic_engine: moving-window scratch allocation failed");
        e.shift_tmp_bytes = bytes;
    }
    return pic_shift_fab(&e.fab[c], e.shift_tmp, &e.geom, num_shift, e.mw_dir, 0.0 /* no external field */, s);
}

// WarpX::MoveWindow (Utils/WarpXMovingWindow.cpp:139-476), one level, lab or z-boosted frame, no PML: advance
// moving_window_x; when it has covered whole cells shift E, B (and J when move_j), move the problem
// domain, and let the continuously injected species fill the uncovered slab.
static int move_window(Engine& e, bool move_j, int* num_moved, void* s) {
    *num_moved = 0;
    if (!e.do_moving_window) return 0;
    const int dir = e.mw_dir;
    e.mw_x += (e.mw_v - e.beta_boost * C_LIGHT) / (1 - e.mw_v * e.beta_boost / C_LIGHT) * e.dt;   // :156
    // UpdateInjectionPosition (:59-136): a plasma at rest in the lab drifts with -beta_boost c in the
    // boosted frame (v' = (v - c beta) / (1 - v beta / c) with v = 0, times boost_direction[dir])
    if (e.gamma_boost > 1.)
        for (auto& sp : e.species) {
            if (!sp.has_injector || !sp.inj.do_continuous_injection) continue;
            double v_shift = 0.0;
            v_shift = (v_shift - C_LIGHT * e.beta_boost) / (1. - v_shift * e.beta_boost / C_LIGHT);
            v_shift *= (dir == 2) ? 1 : 0;
            sp.current_injection_position += v_shift * e.dt;
        }
    const double cdx = e.dx[dir];
    const int nsb = static_cast<int>((e.mw_x - e.geom.prob_lo[dir]) / cdx);              // :171
    if (nsb == 0) return 0;
    e.geom.prob_lo[dir] = e.geom.prob_lo[dir] + nsb * cdx;                                // :181-186
    e.geom.prob_hi[dir] = e.geom.prob_hi[dir] + nsb * cdx;
    if (e.comm && e.nb[dir] > 1) {
        // FillBoundary of shiftMF's temporary (:499-505): the planes the shift pulls in from the next slab
        const int mag = nsb > 0 ? nsb : -nsb;
        ENG_CALL(halo_sweep(e, &e.fab[0], 6, dir, mag, 0, s));
        if (move_j) ENG_CALL(halo_sweep(e, &e.fab[6], 3, dir, mag, 0, s));
    }
    for (int dim = 0; dim < 3; ++dim) {                                                   // :226-266
        ENG_CALL(shift_component(e, 3 + dim, nsb, s));
        ENG_CALL(shift_component(e, dim, nsb, s));
        if (move_j) ENG_CALL(shift_component(e, 6 + dim, nsb, s));
    }
    for (auto& sp : e.species) {                                                          // :388-438
        if (!sp.has_injector || !sp.inj.do_continuous_injection) continue;
        double new_pos = sp.current_injection_position;
        if (e.mw_v > 0.0)
            new_pos = sp.current_injection_position + floor((e.geom.prob_hi[dir] - sp.current_injection_position) / cdx) * cdx;
        else if (e.mw_v < 0.0)
            new_pos = sp.current_injection_position - floor((sp.current_injection_position - e.geom.prob_lo[dir]) / cdx) * cdx;
        double plo[3], phi[3];
        for (int d = 0; d < 3; ++d) { plo[d] = e.geom.prob_lo[d]; phi[d] = e.geom.prob_hi[d]; }
        if (e.mw_v > 0.0) { plo[dir] = sp.current_injection_position; phi[dir] = new_pos; }
        else if (e.mw_v < 0.0) { plo[dir] = new_pos; phi[dir] = sp.current_injection_position; }
        const bool ok = plo[0] < phi[0] && plo[1] < phi[1] && plo[2] < phi[2];            // RealBox::ok
        if (ok && sp.current_injection_position != new_pos) {
            pic_soa& P = sp.buf[sp.cur];
            // every rank advances the id counter by the global count; the rank whose brick contains the
            // slab creates the particles (tile_realbox.contains, :1141-1156)
            const long total = pic_add_plasma(&sp.inj, &e.geom, e.dx, nullptr, nullptr, plo, phi, nullptr, 0, 0, e.cur_time, s);
            const long added = pic_add_plasma(&sp.inj, &e.geom, e.dx, e.box_lo, e.box_hi, plo, phi, &P, sp.capacity, sp.next_id,
                                              e.cur_time /* t_new, already advanced (WarpXEvolve.cpp:232-246) */, s);
            if (added < 0 || total < 0) return 1;
            P.np += added;
            sp.next_id += (uint64_t)total;
            sp.current_injection_position = new_pos;
        }
    }
    for (auto& sp : e.species) sp.bins_stale = true;     // every particle changed cell along dir
    *num_moved = nsb;
    return 0;
}

// mypc->ApplyBoundaryConditions() over species and lasers (MultiParticleContainer.cpp:659-664) and the
// removal AMReX Redistribute performs: all marks first, ONE host read of the counts, then the compactions.
static int apply_particle_boundaries(Engine& e, void* stream) {
    if (e.all_periodic) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    const size_t nsp = e.species.size(), ncont = nsp + e.lasers.size();
    if (ncont == 0) return 0;
    for (size_t n = 0; n < ncont; ++n) {
        const bool is_sp = n < nsp;
        pic_soa& P = is_sp ? e.species[n].buf[e.species[n].cur] : e.lasers[n - nsp].P;
        int* work = is_sp ? e.species[n].bnd_work : e.lasers[n - nsp].bnd_work;
        const int cap = is_sp ? e.species[n].bnd_cap : e.lasers[n - nsp].bnd_cap;
        ENG_CALL(pic_particles_boundary_mark(&P, &e.geom, &e.bnd, work, cap, s));
        cudaMemcpyAsync(e.host_count + n, work, sizeof(int), cudaMemcpyDeviceToHost, s);
    }
    if (cudaStreamSynchronize(s) != cudaSuccess) return fail("pic_engine: particle boundary pass failed (%s)", cudaGetErrorString(cudaGetLastError()));
    for (size_t n = 0; n < ncont; ++n) {
        const int lost = e.host_count[n];
        if (lost == 0) continue;
        const bool is_sp = n < nsp;
        pic_soa& P = is_sp ? e.species[n].buf[e.species[n].cur] : e.lasers[n - nsp].P;
        int* work = is_sp ? e.species[n].bnd_work : e.lasers[n - nsp].bnd_work;
        const int cap = is_sp ? e.species[n].bnd_cap : e.lasers[n - nsp].bnd_cap;
        ENG_CALL(pic_particles_boundary_compact(&P, work, cap, lost, s));
        P.np -= lost;
        if (is_sp) e.species[n].bins_stale = true;
    }
    return 0;
}

// WarpXFluidContainer::Evolve (Source/Fluids/WarpXFluidContainer.cpp:257-314) on a periodic domain: GatherAndPush,
// the FillBoundary of N and NU with all 2 guard nodes (ApplyBcFluidsAndComms :413-417), AdvectivePush_Muscl into the
// other state, DepositCurrent into the J the particles deposit into (filtered afterwards like theirs).
static int evolve_fluid(Engine& e, Fluid& fl, void* s) {
    pic_fab* U = fl.U[fl.cur];
    ENG_CALL(pic_fluid_gather_push(U, &e.fab[0], &e.fab[3], fl.q, fl.m, e.dt, s));
    for (int d = 0; d < 3; ++d) ENG_CALL(halo_sweep(e, U, 4, d, 2, 0, s));
    ENG_CALL(pic_fluid_advect(U, fl.U[1 - fl.cur], e.dx, e.dt, nullptr, s));
    fl.cur = 1 - fl.cur;
    return pic_fluid_deposit_current(fl.U[fl.cur], e.use_filter ? e.jdep : &e.fab[6], fl.q, s);
}

static int one_step(Engine& e, bool last, void* s) {
    // ---- ExplicitFillBoundaryEBUpdateAux ----
    if (e.is_synchronized) {
        { Stage t(e, ST_FILL_EB, s); ENG_CALL(fill_boundary(e, 0, 6, e.ng_EB, s)); }                    // ng_alloc_EB, :487-488
        { Stage t(e, ST_PUSHP, s); for (auto& sp : e.species) ENG_CALL(push(e, sp, -0.5 * e.dt, 0, s)); }   // PushP(-dt/2), :492-504
        e.is_synchronized = false;
    } else {
        Stage t(e, ST_FILL_EB, s);
        ENG_CALL(fill_boundary(e, 0, 6, e.ng_FG, s));                    // :515-516
    }
    // ---- OneStep_nosub ----
    ENG_CALL(push_particles_and_deposit(e, s));
    for (auto& fl : e.fluids) { Stage t(e, ST_FLUID, s); ENG_CALL(evolve_fluid(e, fl, s)); }   // myfl->Evolve, :1171-1178
    if (e.use_filter) { Stage t(e, ST_FILTER, s); ENG_CALL(pic_apply_filter_multi(e.jdep, &e.fab[6], 3, e.npass, s)); }
    { Stage t(e, ST_SYNC_J, s); ENG_CALL(sync_current(e, s)); }
    { Stage t(e, ST_EVOLVE_B, s); ENG_CALL(evolve_b(e, 0.5 * e.dt, s)); }
    { Stage t(e, ST_FILL_B, s); ENG_CALL(fill_boundary(e, 3, 6, e.ng_FS, s)); }
    { Stage t(e, ST_EVOLVE_E, s); ENG_CALL(evolve_e(e, e.dt, s)); }
    { Stage t(e, ST_FILL_E, s); ENG_CALL(fill_boundary(e, 0, 3, e.ng_FS, s)); }
    { Stage t(e, ST_EVOLVE_B, s); ENG_CALL(evolve_b(e, 0.5 * e.dt, s)); }
    if (last) {                                                           // Synchronize(), :64-91
        { Stage t(e, ST_FILL_EB, s); ENG_CALL(fill_boundary(e, 0, 6, e.ng_FG, s)); }
        { Stage t(e, ST_PUSHP, s); for (auto& sp : e.species) ENG_CALL(push(e, sp, 0.5 * e.dt, 0, s)); }
        e.is_synchronized = true;
    }
    const long step = e.istep++;
    e.cur_time += e.dt;                                                   // :232
    // ---- MoveWindow(step+1, move_j = is_synchronized), :247 ----
    int num_moved = 0;
    { Stage t(e, ST_WINDOW, s); ENG_CALL(move_window(e, e.is_synchronized, &num_moved, s)); }
    // ---- HandleParticlesAtBoundaries ----
    {
        Stage t(e, ST_WRAP, s);
        for (auto& sp : e.species) {
            // amrex enforcePeriodic: only the particles the push of this step moved out of the domain
            // (done before the removal below, while the indices listed by the push are still valid; the
            // two act on different directions)
            if (sp.has_esc) ENG_CALL(pic_particles_wrap_listed(&sp.buf[sp.cur], &e.geom, &sp.esc, s));
            else ENG_CALL(pic_particles_wrap_periodic(&sp.buf[sp.cur], &e.geom, s));
        }
        for (auto& L : e.lasers) ENG_CALL(pic_particles_wrap_periodic(&L.P, &e.geom, s));
        ENG_CALL(apply_particle_boundaries(e, s));
    }
    for (auto& sp : e.species) {
        if (e.comm) { Stage t(e, ST_MIGRATE, s); ENG_CALL(migrate(e, sp, s)); }
        const bool due = e.sort_interval > 0 && (step + 1) % e.sort_interval == 0;
        if (sp.sort_work && (due || (sp.bins_stale && sp.has_bins))) { Stage t(e, ST_SORT, s); ENG_CALL(sort_species(e, sp, s)); }
        sp.bins_stale = false;
    }
    if (e.tm.on && e.tm.recs.size() > 4096) collect_timing(e);          // bound the event pool of long runs
    return 0;
}

}  // namespace pic

using namespace pic;

static int alloc_boundary_scratch(long capacity, int** work, int* cap);
static int grow_host_counts(Engine& e);

// Defaults of the kernel-variant switches from the environment (PIC_FDTD_MODE, PIC_DEPOSIT_MODE, PIC_GATHER_MODE):
// lets a launcher pin a variant without touching the host code.  Applied once, when the library is loaded.
extern "C" void pic_set_fdtd_mode(int mode);
extern "C" void pic_set_deposit_mode(int mode);
extern "C" void pic_set_gather_mode(int mode);
namespace {
struct EnvDefaults {
    EnvDefaults() {
        if (const char* v = getenv("PIC_FDTD_MODE")) pic_set_fdtd_mode(atoi(v));
        if (const char* v = getenv("PIC_DEPOSIT_MODE")) pic_set_deposit_mode(atoi(v));
        if (const char* v = getenv("PIC_GATHER_MODE")) pic_set_gather_mode(atoi(v));
    }
};
}  // namespace
extern "C" void pic_apply_env_defaults(void) { static EnvDefaults once; (void)once; }

extern "C" void* pic_engine_create(const pic_geom* geom, const int box_lo[3], const int box_hi[3], int nox,
                                   int galerkin, int pusher, int solver, double cfl, double dt,
                                   int sort_interval, int use_filter, const int filter_npass[3]) {
    Engine* e = new Engine();
    e->geom = *geom;
    e->use_filter = use_filter ? 1 : 0;
    for (int d = 0; d < 3; ++d) e->npass[d] = filter_npass ? filter_npass[d] : 1;
    for (int d = 0; d < 3; ++d) {
        e->box_lo[d] = box_lo[d]; e->box_hi[d] = box_hi[d];
        e->dx[d] = (geom->prob_hi[d] - geom->prob_lo[d]) / geom->n_cell[d];
        e->dinv[d] = 1.0 / e->dx[d];
    }
    e->nox = nox; e->galerkin = galerkin; e->pusher = pusher; e->solver = solver; e->sort_interval = sort_interval;
    e->dt = dt > 0 ? dt : cfl * max_dt(solver, e->dx);
    stencil_coefficients(solver, e->dx, &e->st);
    guard_cells(*e);
    return e;
}
extern "C" void pic_engine_destroy(void* h) {
    Engine* e = static_cast<Engine*>(h);
    if (e && e->jdep_alloc) for (int c = 0; c < 3; ++c) cudaFree(e->jdep[c].p);
    if (e) {
#ifndef PIC_SIMT_HOST
        for (cudaEvent_t ev : e->tm.pool) cudaEventDestroy(ev);
#endif
        for (auto& sp : e->species) {
            if (sp.has_esc) cudaFree(sp.esc.count);
            if (sp.mig_counts) cudaFree(sp.mig_counts);
            for (int b = 0; b < 2; ++b) if (sp.mig_idx[b]) cudaFree(sp.mig_idx[b]);
            for (int b = 0; b < 4; ++b) if (sp.mig_msg[b]) cudaFree(sp.mig_msg[b]);
            if (sp.mig_work) cudaFree(sp.mig_work);
            if (sp.mig_head) cudaFreeHost(sp.mig_head);
            if (sp.bnd_work) cudaFree(sp.bnd_work);
        }
        for (auto& L : e->lasers) { if (L.bnd_work) cudaFree(L.bnd_work); if (L.w_owned) cudaFree(L.w_owned); }
        if (e->shift_tmp) cudaFree(e->shift_tmp);
        if (e->nci_alloc) for (int c = 0; c < 6; ++c) cudaFree(e->nci_fab[c].p);
        if (e->host_count) cudaFreeHost(e->host_count);
        for (int b = 0; b < 4; ++b) if (e->hbuf[b]) cudaFree(e->hbuf[b]);
    }
    delete e;
}
extern "C" double pic_engine_dt(void* h) { return static_cast<Engine*>(h)->dt; }
// Per-stage timing of pic_engine_evolve with CUDA events on the launching stream: switch on (the sums are reset),
// run steps, read with pic_engine_stage_ms (synchronises on the recorded events).
extern "C" int pic_engine_enable_timing(void* h, int on) {
    Engine* e = static_cast<Engine*>(h);
    collect_timing(*e);
    for (int n = 0; n < ST_COUNT; ++n) { e->tm.ms[n] = 0.0; e->tm.calls[n] = 0; }
    e->tm.on = on != 0;
    return 0;
}
extern "C" int pic_engine_stage_count(void) { return ST_COUNT; }
extern "C" const char* pic_engine_stage_name(int n) { return (n >= 0 && n < ST_COUNT) ? stage_names[n] : ""; }
// total milliseconds and number of calls of every stage since pic_engine_enable_timing(h, 1)
extern "C" int pic_engine_stage_ms(void* h, double ms[], long calls[]) {
    Engine* e = static_cast<Engine*>(h);
    collect_timing(*e);
    for (int n = 0; n < ST_COUNT; ++n) { ms[n] = e->tm.ms[n]; calls[n] = e->tm.calls[n]; }
    return 0;
}
extern "C" void pic_engine_guards(void* h, int out[12]) {
    Engine* e = static_cast<Engine*>(h);
    for (int d = 0; d < 3; ++d) { out[d] = e->ng_EB[d]; out[3 + d] = e->ng_J[d]; out[6 + d] = e->ng_FG[d]; out[9 + d] = e->ng_FS[d]; }
}
extern "C" int pic_engine_set_fields(void* h, const pic_fab fabs[9]) {
    Engine* e = static_cast<Engine*>(h);
    if (e->jdep_alloc) { for (int c = 0; c < 3; ++c) cudaFree(e->jdep[c].p); e->jdep_alloc = false; }   // new shapes
    for (int c = 0; c < 9; ++c) {
        e->fab[c] = fabs[c];
        const int* ng = c < 6 ? e->ng_EB : e->ng_J;
        for (int d = 0; d < 3; ++d)
            PIC_REQUIRE(fabs[c].ng[d] >= ng[d], "pic_engine_set_fields: component %d has %d guard cells, needs %d", c, fabs[c].ng[d], ng[d]);
    }
    // the guard cells are final now (the moving window and the NCI corrector may have grown ng_J after
    // pic_engine_set_boundaries checked it): a box along a non-periodic direction must hold both mirror images
    for (int d = 0; d < 3; ++d)
        PIC_REQUIRE(e->geom.periodic[d] || e->box_hi[d] - e->box_lo[d] + 1 >= 2 * e->ng_J[d],
                    "pic_engine_set_fields: the box is too thin along the non-periodic direction %d (%d cells, ng_J = %d)",
                    d, e->box_hi[d] - e->box_lo[d] + 1, e->ng_J[d]);
    return 0;
}
// bufA holds the particles; bufB is the sort target.  cell_start / sort_work may be NULL (no bins).
extern "C" int pic_engine_add_species(void* h, double q, double m, const pic_soa* bufA, const pic_soa* bufB,
                                      long capacity, int* cell_start, const int tile[3], void* sort_work,
                                      void* stream) {
    Engine* e = static_cast<Engine*>(h);
    PIC_REQUIRE(capacity >= bufA->np, "pic_engine_add_species: capacity %ld < np %ld", capacity, (long)bufA->np);
    PIC_REQUIRE(e->fluids.empty(), "pic_engine_add_species: runs with fluid species take no particle species yet");
    Species sp;
    sp.capacity = capacity;
    sp.q = q; sp.m = m; sp.buf[0] = *bufA; sp.buf[1] = *bufB; sp.cur = 0; sp.has_bins = false; sp.sort_work = sort_work;
    sp.bins.cell_start = cell_start;
    for (int d = 0; d < 3; ++d) sp.bins.tile[d] = tile ? tile[d] : 8;
    sp.bins.np_binned = 0;
    // escape list: a layer of one cell next to every domain face can leave per step at most
    sp.has_esc = false;
    {
        const long cap = capacity / 16 + 65536;
        int* mem = nullptr;
        if (cudaMalloc(&mem, sizeof(int) * (size_t)(cap + 1)) == cudaSuccess) {
            sp.esc.count = mem; sp.esc.idx = mem + 1; sp.esc.capacity = (int)cap;
            for (int d = 0; d < 3; ++d) {
                sp.esc.lo[d] = e->geom.periodic[d] ? e->geom.prob_lo[d] : -INFINITY;
                sp.esc.hi[d] = e->geom.periodic[d] ? e->geom.prob_hi[d] : INFINITY;
            }
            sp.has_esc = true;
        } else {
            cudaGetLastError();      // no list: the engine wraps with the full sweep
        }
    }
    if (e->comm) {
        // migration scratch; worst case per face and step = one full layer of cells ~ capacity/256
        sp.mig_cap_max = (int)(capacity / 256 > 65536 ? capacity / 256 : 65536);
        if (e->do_moving_window) {
            // every shift sends one whole layer of cells to the slab below
            const long layer = capacity / (e->box_hi[e->mw_dir] - e->box_lo[e->mw_dir] + 1);
            if (2 * layer + 65536 > sp.mig_cap_max) sp.mig_cap_max = (int)(2 * layer + 65536);
        }
        sp.mig_cap = sp.mig_cap_max;
        const size_t nmsg = (size_t)pic_migrate_message_doubles(sp.mig_cap_max);
        bool ok = cudaMalloc(&sp.mig_counts, 2 * sizeof(int)) == cudaSuccess;
        for (int b = 0; b < 2 && ok; ++b) ok = cudaMalloc(&sp.mig_idx[b], sizeof(int) * (size_t)sp.mig_cap_max) == cudaSuccess;
        for (int b = 0; b < 4 && ok; ++b) ok = cudaMalloc(&sp.mig_msg[b], sizeof(double) * nmsg) == cudaSuccess;
        ok = ok && cudaMalloc(&sp.mig_work, (size_t)pic_migrate_workspace_bytes(sp.mig_cap_max)) == cudaSuccess;
        ok = ok && cudaMallocHost(&sp.mig_head, 8 * sizeof(int)) == cudaSuccess;
        if (!ok) return fail("pic_engine_add_species: cannot allocate the migration buffers");
        for (int b = 0; b < 4; ++b) cudaMemsetAsync(sp.mig_msg[b], 0, sizeof(double) * nmsg, (cudaStream_t)stream);
        cudaMemsetAsync(sp.mig_work, 0, (size_t)pic_migrate_workspace_bytes(sp.mig_cap_max), (cudaStream_t)stream);
    }
    if (!e->all_periodic) ENG_CALL(alloc_boundary_scratch(capacity, &sp.bnd_work, &sp.bnd_cap));
    e->species.push_back(sp);
    ENG_CALL(grow_host_counts(*e));
    if (cell_start && sort_work) return sort_species(*e, e->species.back(), stream);
    return 0;
}
// Multi-rank: this rank's brick is box_lo..box_hi of pic_engine_create, rank = coord[0] + nb[0]*(coord[1]
// + nb[1]*coord[2]) in the communicator (pic_comm_create).  Call before pic_engine_add_species.
extern "C" int pic_engine_set_comm(void* h, void* comm, const int nb[3]) {
    Engine* e = static_cast<Engine*>(h);
    Comm* c = static_cast<Comm*>(comm);
    PIC_REQUIRE(c && c->comm, "pic_engine_set_comm: no communicator");
    PIC_REQUIRE(nb[0] * nb[1] * nb[2] == c->nranks, "pic_engine_set_comm: brick grid %dx%dx%d != %d ranks", nb[0], nb[1], nb[2], c->nranks);
    PIC_REQUIRE(e->species.empty(), "pic_engine_set_comm: call before pic_engine_add_species");
    if (e->do_moving_window)      // the shift folds the periodic refresh of the other directions into its read
        for (int d = 0; d < 3; ++d)
            PIC_REQUIRE(d == e->mw_dir || nb[d] == 1, "pic_engine_set_comm: a moving window needs slabs along its direction (nb[%d] = %d)", d, nb[d]);
    e->comm = c;
    int r = c->rank;
    for (int d = 0; d < 3; ++d) {
        e->nb[d] = nb[d];
        e->coord[d] = r % nb[d];
        r /= nb[d];
        const int width = e->geom.n_cell[d] / nb[d];
        PIC_REQUIRE(width * nb[d] == e->geom.n_cell[d] && e->box_lo[d] == e->coord[d] * width &&
                    e->box_hi[d] == e->box_lo[d] + width - 1,
                    "pic_engine_set_comm: box [%d,%d] along %d is not brick %d of %d", e->box_lo[d], e->box_hi[d], d, e->coord[d], nb[d]);
    }
    return 0;
}
// ---- the decomposition as a guard-cell context: the one-call replacements of the reference's comm wrappers ----
// ablastr::utils::communication::FillBoundary(mf, ng, ..., period) (Source/ablastr/utils/Communication.cpp:71-115) as
// called by WarpX::FillBoundaryE/B (Source/Parallelization/WarpXComm.cpp:699-827): guards <- valid, over the bricks.
extern "C" int pic_halo_copy(void* h, const pic_fab* fabs, int nfab, const int ng[3], void* stream) {
    Engine* e = static_cast<Engine*>(h);
    PIC_REQUIRE(fabs && nfab > 0, "pic_halo_copy: no components");
    for (int c = 0; c < nfab; ++c)
        for (int d = 0; d < 3; ++d) PIC_REQUIRE(ng[d] >= 0 && ng[d] <= fabs[c].ng[d], "pic_halo_copy: ng[%d] = %d exceeds the allocated guard cells", d, ng[d]);
    for (int d = 0; d < 3; ++d) ENG_CALL(halo_sweep(*e, fabs, nfab, d, ng[d], 0, stream));
    return 0;
}
// ablastr::utils::communication::SumBoundary(mf, icomp, ncomp, src_ng, dst_ng, ..., period) (:148-175) as called by
// WarpXSumGuardCells (Source/Parallelization/WarpXSumGuardCells.cpp:17-24): valid += guards of the neighbours within
// src_ng, then the first dst_ng guard cells take the summed values (WarpX passes dst_ng = all guards).
extern "C" int pic_halo_add(void* h, const pic_fab* fabs, int nfab, const int src_ng[3], const int dst_ng[3], void* stream) {
    Engine* e = static_cast<Engine*>(h);
    PIC_REQUIRE(fabs && nfab > 0, "pic_halo_add: no components");
    for (int c = 0; c < nfab; ++c)
        for (int d = 0; d < 3; ++d)
            PIC_REQUIRE(src_ng[d] >= 0 && src_ng[d] <= fabs[c].ng[d] && dst_ng[d] >= 0 && dst_ng[d] <= fabs[c].ng[d],
                        "pic_halo_add: src_ng / dst_ng exceed the allocated guard cells along %d", d);
    // beyond a non-periodic domain face AMReX zeroes the guard layers between src_ng and dst_ng (they are not in its
    // temporary); WarpX always sums with src_ng = dst_ng = all guards there (WarpXComm.cpp:1396-1420), which is the
    // case built here
    for (int d = 0; d < 3; ++d)
        PIC_REQUIRE(e->geom.periodic[d] || src_ng[d] == dst_ng[d],
                    "pic_halo_add: along the non-periodic direction %d src_ng (%d) and dst_ng (%d) must be equal", d, src_ng[d], dst_ng[d]);
    for (int d = 0; d < 3; ++d) ENG_CALL(halo_sweep(*e, fabs, nfab, d, src_ng[d], 1, stream));
    for (int d = 0; d < 3; ++d) ENG_CALL(halo_sweep(*e, fabs, nfab, d, dst_ng[d], 0, stream, true));
    return 0;
}

// WarpX::HandleParticlesAtBoundaries (Source/Evolve/WarpXEvolve.cpp:533-564) as one call, for a host that keeps its
// own step loop: periodic wrap (amrex enforcePeriodic), ApplyBoundaryConditions on the non-periodic faces + removal,
// and the move of every particle that left this rank's brick to the neighbour that owns it (RedistributeLocal(1):
// at most one brick per call and direction).  Acts on the species and antennas registered with the engine; the
// particle counts are read back with pic_engine_species_buffer / pic_engine_laser_np.  The cell bins of a species
// are stale afterwards (particles appended / removed): sort before the next binned gather.
extern "C" int pic_engine_redistribute(void* h, void* stream) {
    Engine* e = static_cast<Engine*>(h);
    for (auto& sp : e->species) ENG_CALL(pic_particles_wrap_periodic(&sp.buf[sp.cur], &e->geom, stream));
    for (auto& L : e->lasers) ENG_CALL(pic_particles_wrap_periodic(&L.P, &e->geom, stream));
    ENG_CALL(apply_particle_boundaries(*e, stream));
    for (auto& sp : e->species) {
        sp.esc_valid = false;            // the caller moved the particles, not the push: classify every one
        if (e->comm) ENG_CALL(migrate(*e, sp, stream));
        sp.bins_stale = true;
    }
    return 0;
}

// ---- non-periodic runs ------------------------------------------------------------------------
static int alloc_boundary_scratch(long capacity, int** work, int* cap) {
    const long c = capacity / 16 + 65536;
    *cap = (int)(c < capacity + 1 ? c : capacity + 1);
    if (cudaMalloc(work, sizeof(int) * (size_t)pic_particles_boundary_workspace_ints(*cap)) != cudaSuccess)
        return fail("pic_engine: cannot allocate the particle-boundary scratch");
    return 0;
}
static int grow_host_counts(Engine& e) {
    const size_t n = e.species.size() + e.lasers.size() + 1;
    int* mem = nullptr;
    if (cudaMallocHost(&mem, sizeof(int) * n) != cudaSuccess) return fail("pic_engine: cannot allocate pinned host memory");
    if (e.host_count) cudaFreeHost(e.host_count);
    e.host_count = mem;
    return 0;
}
extern "C" int pic_engine_set_boundaries(void* h, const pic_boundaries* b) {
    Engine* e = static_cast<Engine*>(h);
    PIC_REQUIRE(e->species.empty() && e->lasers.empty(), "pic_engine_set_boundaries: call before adding particles");
    e->bnd = *b;
    e->any_pec = false; e->all_periodic = true;
    for (int d = 0; d < 3; ++d) {
        const bool per = b->field_lo[d] == PIC_FIELD_PERIODIC;
        PIC_REQUIRE(per == (b->field_hi[d] == PIC_FIELD_PERIODIC), "pic_engine_set_boundaries: direction %d is periodic on one side only", d);
        e->geom.periodic[d] = per ? 1 : 0;
        if (per) e->bnd.particle_lo[d] = e->bnd.particle_hi[d] = PIC_PARTICLE_PERIODIC;
        else {
            PIC_REQUIRE(b->particle_lo[d] != PIC_PARTICLE_PERIODIC && b->particle_hi[d] != PIC_PARTICLE_PERIODIC,
                        "pic_engine_set_boundaries: periodic particles on the non-periodic direction %d", d);
            PIC_REQUIRE(e->box_hi[d] - e->box_lo[d] + 1 >= 2 * e->ng_J[d],
                        "pic_engine_set_boundaries: the box is too thin along the non-periodic direction %d", d);
            e->all_periodic = false;
        }
        e->any_pec = e->any_pec || b->field_lo[d] == PIC_FIELD_PEC || b->field_hi[d] == PIC_FIELD_PEC;
    }
    return 0;
}
extern "C" int pic_engine_set_moving_window(void* h, int dir, double v_over_c) {
    Engine* e = static_cast<Engine*>(h);
    PIC_REQUIRE(dir >= 0 && dir < 3, "pic_engine_set_moving_window: bad direction");
    PIC_REQUIRE(!e->geom.periodic[dir], "The problem must be non-periodic in the moving window direction");   // WarpX.cpp:646-648
    PIC_REQUIRE(e->species.empty() && e->lasers.empty(), "pic_engine_set_moving_window: call before adding particles");
    PIC_REQUIRE(e->comm == nullptr, "pic_engine_set_moving_window: call before pic_engine_set_comm");
    e->do_moving_window = true; e->mw_dir = dir; e->mw_v = v_over_c * C_LIGHT;
    e->mw_x = e->geom.prob_lo[dir];                      // WarpX.cpp:649
    guard_cells(*e);
    return 0;
}
// warpx.gamma_boost (Source/Utils/WarpXUtil.cpp:114-121) with warpx.boost_direction = z
extern "C" int pic_engine_set_boost(void* h, double gamma_boost, double beta_boost) {
    Engine* e = static_cast<Engine*>(h);
    PIC_REQUIRE(gamma_boost >= 1. && beta_boost >= 0. && beta_boost < 1., "pic_engine_set_boost: need gamma_boost >= 1 and 0 <= beta_boost < 1");
    PIC_REQUIRE((gamma_boost > 1.) == (beta_boost > 0.), "pic_engine_set_boost: gamma_boost and beta_boost disagree");
    PIC_REQUIRE(e->lasers.empty(), "pic_engine_set_boost: call before pic_engine_add_laser");
    for (auto& sp : e->species) PIC_REQUIRE(!sp.has_injector, "pic_engine_set_boost: call before pic_engine_set_injector");
    e->gamma_boost = gamma_boost; e->beta_boost = beta_boost;
    return 0;
}
// particles.use_fdtd_nci_corr (MultiParticleContainer.cpp:327, WarpX::InitNCICorrector, WarpXInitData.cpp:858-890)
extern "C" int pic_engine_set_nci_corrector(void* h, const double stencil_exeybz[5], const double stencil_bxbyez[5]) {
    Engine* e = static_cast<Engine*>(h);
    PIC_REQUIRE(e->species.empty() && e->lasers.empty(), "pic_engine_set_nci_corrector: call before adding particles");
    PIC_REQUIRE(e->comm == nullptr, "pic_engine_set_nci_corrector: call before pic_engine_set_comm");
    e->use_nci = true;
    for (int i = 0; i < 5; ++i) { e->nci_stencil[0][i] = stencil_exeybz[i]; e->nci_stencil[1][i] = stencil_bxbyez[i]; }
    guard_cells(*e);
    return 0;
}
static bool same_boost(const Engine& e, double gamma_boost, double beta_boost) {
    const bool boosted = gamma_boost > 1.;
    return boosted ? (gamma_boost == e.gamma_boost && beta_boost == e.beta_boost) : !(e.gamma_boost > 1.);
}
extern "C" int pic_engine_set_injector(void* h, int isp, const pic_plasma_injector* inj) {
    Engine* e = static_cast<Engine*>(h);
    PIC_REQUIRE(isp >= 0 && isp < (int)e->species.size(), "pic_engine_set_injector: no species %d", isp);
    PIC_REQUIRE(same_boost(*e, inj->gamma_boost, inj->beta_boost), "pic_engine_set_injector: the injector's gamma_boost / beta_boost differ from pic_engine_set_boost");
    Species& sp = e->species[isp];
    sp.has_injector = true; sp.inj = *inj;
    // ids continue after the particles the injector created at start-up on ALL ranks
    const long created = pic_add_plasma(inj, &e->geom, e->dx, nullptr, nullptr, e->geom.prob_lo, e->geom.prob_hi,
                                        nullptr, 0, 0, 0.0, nullptr);
    PIC_REQUIRE(created >= 0, "pic_engine_set_injector: bad injector");
    sp.next_id = (uint64_t)created;
    if (e->do_moving_window)                            // WarpX.cpp:288-307
        sp.current_injection_position = e->mw_v > 0 ? e->geom.prob_hi[e->mw_dir] : e->geom.prob_lo[e->mw_dir];
    return 0;
}
extern "C" int pic_engine_add_laser(void* h, const pic_laser_antenna* prm, const pic_soa* p, long capacity) {
    Engine* e = static_cast<Engine*>(h);
    PIC_REQUIRE(e->fluids.empty(), "pic_engine_add_laser: runs with fluid species take no antennas yet");
    double info[4];
    PIC_REQUIRE(same_boost(*e, prm->gamma_boost, prm->beta_boost), "pic_engine_add_laser: the antenna's gamma_boost / beta_boost differ from pic_engine_set_boost");
    ENG_CALL(pic_laser_antenna_info(prm, e->dx, info));
    PIC_REQUIRE(capacity >= p->np, "pic_engine_add_laser: capacity %ld < np %ld", capacity, (long)p->np);
    Laser L;
    L.prm = *prm; L.P = *p; L.capacity = capacity;
    if (!e->all_periodic) ENG_CALL(alloc_boundary_scratch(capacity, &L.bnd_work, &L.bnd_cap));
    if (e->comm && cudaMalloc(&L.w_owned, sizeof(double) * (size_t)(capacity > 0 ? capacity : 1)) != cudaSuccess)
        return fail("pic_engine_add_laser: cannot allocate the weight scratch");
    e->lasers.push_back(L);
    return grow_host_counts(*e);
}
extern "C" long pic_engine_laser_np(void* h, int il) { return (long)static_cast<Engine*>(h)->lasers[il].P.np; }
extern "C" double pic_engine_time(void* h) { return static_cast<Engine*>(h)->cur_time; }
// restart from a checkpoint: istep / t_new (WarpX::InitFromCheckpoint, Source/Diagnostics/WarpXIO.cpp:118-140)
extern "C" int pic_engine_set_step(void* h, long istep, double time) {
    Engine* e = static_cast<Engine*>(h);
    PIC_REQUIRE(istep >= 0, "pic_engine_set_step: negative step");
    e->istep = istep; e->cur_time = time;
    return 0;
}
extern "C" void pic_engine_prob_domain(void* h, double out[6]) {
    Engine* e = static_cast<Engine*>(h);
    for (int d = 0; d < 3; ++d) { out[d] = e->geom.prob_lo[d]; out[3 + d] = e->geom.prob_hi[d]; }
}
// which of the two buffers currently holds species isp, and its particle count
extern "C" int pic_engine_species_buffer(void* h, int isp, long* np) {
    Engine* e = static_cast<Engine*>(h);
    if (np) *np = e->species[isp].buf[e->species[isp].cur].np;
    return e->species[isp].cur;
}
// WarpX::Evolve(numsteps): the last step synchronises u with x when synchronize_last is set
extern "C" int pic_engine_evolve(void* h, int numsteps, int synchronize_last, void* stream) {
    Engine* e = static_cast<Engine*>(h);
    for (int n = 0; n < numsteps; ++n) ENG_CALL(one_step(*e, synchronize_last && n == numsteps - 1, stream));
    return 0;
}

// A cold fluid species (fluids.species_names): stateA holds the initial N, NUx, NUy, NUz on this engine's box with 2
// guard nodes, stateB is a second state of the same shape (borrowed; the driver advects from one into the other, see
// pic_engine_fluid_state).  One rank, periodic faces, no moving window, no boost, no particle species or antennas.
// Every precondition is checked before the engine is changed.
extern "C" int pic_engine_add_fluid_species(void* h, double q, double m, const pic_fab stateA[4], const pic_fab stateB[4]) {
    Engine* e = static_cast<Engine*>(h);
    PIC_REQUIRE(e && stateA && stateB, "pic_engine_add_fluid_species: null argument");
    PIC_REQUIRE(e->all_periodic, "pic_engine_add_fluid_species: every face must be periodic");
    PIC_REQUIRE(!e->do_moving_window, "pic_engine_add_fluid_species: moving windows are not supported");
    PIC_REQUIRE(e->gamma_boost == 1.0, "pic_engine_add_fluid_species: boosted frames are not supported");
    PIC_REQUIRE(e->comm == nullptr, "pic_engine_add_fluid_species: one rank only");
    PIC_REQUIRE(e->species.empty() && e->lasers.empty(), "pic_engine_add_fluid_species: runs with particle species or antennas take no fluids yet");
    PIC_REQUIRE(m > 0.0, "pic_engine_add_fluid_species: mass must be positive");
    for (int b = 0; b < 2; ++b)
        for (int c = 0; c < 4; ++c) {
            const pic_fab& f = (b ? stateB : stateA)[c];
            PIC_REQUIRE(f.p != nullptr, "pic_engine_add_fluid_species: component %d of state %d has no data", c, b);
            for (int d = 0; d < 3; ++d)
                PIC_REQUIRE(f.stag[d] == 1 && f.ng[d] == 2 && vlo(f, d) == e->box_lo[d] && vhi(f, d) == e->box_hi[d] + 1,
                            "pic_engine_add_fluid_species: a state is 4 all-nodal components on the engine's box with 2 guard nodes");
        }
    Fluid fl;
    fl.q = q; fl.m = m;
    for (int c = 0; c < 4; ++c) { fl.U[0][c] = stateA[c]; fl.U[1][c] = stateB[c]; }
    e->fluids.push_back(fl);
    return 0;
}
// Which of the two states of fluid i is current (0: stateA, 1: stateB); -1 if there is no such fluid.
extern "C" int pic_engine_fluid_state(void* h, int i) {
    Engine* e = static_cast<Engine*>(h);
    return (i >= 0 && i < (int)e->fluids.size()) ? e->fluids[i].cur : -1;
}
