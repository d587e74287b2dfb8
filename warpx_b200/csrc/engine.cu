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
// Fields, particle SoA double buffers, bins and sort scratch are borrowed from the caller; the driver's own scratch
// is held in Owned buffers.  Every stage is an asynchronous launch on the caller's stream.
// Non-periodic domains (pic_engine_set_boundaries / set_moving_window / set_injector / add_laser, one
// rank): PEC walls after every field push and on J (BoundaryConditions/WarpXFieldBoundaries.cpp:51-190),
// WarpX::MoveWindow with continuous injection (Utils/WarpXMovingWindow.cpp:139-476), laser antennas
// (Particles/LaserParticleContainer.cpp:563-700), absorbing / reflecting particle boundaries
// (Particles/WarpXParticleContainer.cpp:1574-1638) -- the additions of the laser-wakefield decks.
// Multi-rank (one process per GPU, one brick per rank, pic_engine_set_comm): the guard-cell
// exchanges and the particle migration go through NCCL send/recv on the same stream (csrc/comm.cu),
// as three axis sweeps with two neighbours each; the host reads 32 bytes once per step (new particle
// count, overflow status, peak migration count).  warpx_b200/engine.py::Simulation drives every run
// through this driver; per-stage timing is pic_engine_enable_timing / pic_engine_stage_ms.
#include "pic_common.cuh"
#include "comm.cuh"
#include <cmath>
#include <atomic>
#include <vector>

namespace pic {

bool gather_push_carries_permutation(int nox);      // gather_push.cu
int flux_list_escapes(const pic_escape_list* e, long first, long n, void* stream);   // flux_injection.cu

// Memory the engine owns: device memory, or pinned host memory when Pinned.  The only code in this file that
// allocates or frees; the memory goes with its owner.  Empty (null) until an allocation succeeds.
template <class T, bool Pinned = false>
class Owned {
public:
    Owned() = default;
    Owned(Owned&& o) noexcept { swap(o); }
    Owned& operator=(Owned&& o) noexcept { Owned(std::move(o)).swap(*this); return *this; }
    ~Owned() { release(); }
    // Replaces the memory with `bytes` new bytes.  A failure leaves the buffer empty and clears the sticky error.
    bool try_alloc(size_t bytes) {
        release();
        if ((Pinned ? cudaMallocHost(&p_, bytes) : cudaMalloc(&p_, bytes)) == cudaSuccess) { bytes_ = bytes; return true; }
        cudaGetLastError();
        p_ = nullptr;
        return false;
    }
    int alloc(size_t bytes, const char* what) { return try_alloc(bytes) ? 0 : fail("%s", what); }
    void release() {
        if (p_) (void)(Pinned ? cudaFreeHost(p_) : cudaFree(p_));
        p_ = nullptr;
        bytes_ = 0;
    }
    T* get() const { return p_; }
    size_t bytes() const { return bytes_; }
    explicit operator bool() const { return p_ != nullptr; }
private:
    void swap(Owned& o) noexcept { std::swap(p_, o.p_); std::swap(bytes_, o.bytes_); }
    T* p_ = nullptr;
    size_t bytes_ = 0;
};
template <class T> using DeviceBuf = Owned<T, false>;
template <class T> using PinnedBuf = Owned<T, true>;

// How the particles in buf[cur] of a species relate to its cell bins and to its escape list, changed only by the
// transitions below, which are named after what happened to the particles.
// A sort inside pic_engine_evolve stops at the permutation: the bins describe the new order, the particles still lie
// in buf[cur] in the old one, and the next gather + push moves them while it reads them anyway.  Everything else that
// reads particle arrays carries out the pending move first; no exported call returns with a permutation pending.
class ParticleOrder {
public:
    explicit ParticleOrder(const pic_bins& geometry) : bins_(geometry) { bins_.np_binned = 0; }   // cell_start, box, tile
    // a sort binned np particles; src: the move it left to do (slot i of the new order is particle src[i])
    void sorted(long np, const int* src) { bins_.np_binned = np; pending_src_ = src; has_bins_ = exact_ = true; esc_valid_ = false; }
    void moved() { pending_src_ = nullptr; }               // the pending move was carried out: buf[cur] -> buf[1 - cur]
    void pushed() { exact_ = false; esc_valid_ = true; }   // positions pushed: cells left, escapes listed
    void held() { esc_valid_ = true; }                     // not pushed (do_not_push): nothing escaped
    void cells_changed() { stale_ = true; }                // particles removed / appended, or the window moved them
    void escape_list_spent() { esc_valid_ = false; }       // migration filled holes and moved tails

    // the bins a collision reads must hold every particle's current cell
    bool collision_needs_sort(long np) const { return !exact_ || bins_.np_binned != np; }
    // the end-of-step sort is due by the interval or because the cells changed during the step; asking ends the step
    bool end_of_step_sort_due(bool interval_due) {
        const bool due = interval_due || (stale_ && has_bins_);
        stale_ = false;
        return due;
    }
    // migration may classify only the particles the escape list (where the species has one) names
    bool escape_list_current() const { return esc_valid_; }
    bool has_bins() const { return has_bins_; }
    const pic_bins& bins() const { return bins_; }
    const pic_bins* bins_if_sorted() const { return has_bins_ ? &bins_ : nullptr; }
    const int* pending() const { return pending_src_; }
private:
    pic_bins bins_;
    const int* pending_src_ = nullptr;
    bool has_bins_ = false, exact_ = false, stale_ = false, esc_valid_ = false;
};

// One <species>.injection_style = NFluxPerCell source (pic_engine_add_flux_injector) with its workspace
struct FluxInjector {
    pic_flux_injector prm;
    int index;                   // position among the engine's flux injectors: part of its streams' counter
    DeviceBuf<char> work;
};

struct Species {
    Species(double q_, double m_, const pic_bins& bins) : q(q_), m(m_), ord(bins) {}
    double q, m;
    pic_soa buf[2];        // counting sort permutes buf[cur] -> buf[1-cur]
    int cur = 0;
    ParticleOrder ord;
    void* sort_work = nullptr;
    // particles the last position push moved out of the domain -- over several ranks: out of the rank's brick.  Without
    // its memory the engine wraps with the full sweep.
    pic_escape_list esc{};
    DeviceBuf<int> esc_mem;      // esc.count, then esc.idx
    bool has_esc() const { return (bool)esc_mem; }
    // neighbour migration (multi-rank)
    long capacity = 0;           // entries of every SoA array of both buffers
    int mig_cap_max = 0, mig_cap = 0;
    DeviceBuf<int> mig_counts;   // [2]
    DeviceBuf<int> mig_idx[2];
    DeviceBuf<double> mig_msg[4];   // send lo/hi, recv lo/hi
    DeviceBuf<int> mig_work;
    PinnedBuf<int> mig_head;     // 8 ints
    // plasma injector (continuous injection behind the moving window) and absorbing boundaries
    bool has_injector = false;
    pic_plasma_injector inj{};
    double current_injection_position = 0.0;     // WarpXParticleContainer::m_current_injection_position
    uint64_t next_id = 0;
    DeviceBuf<int> bnd_work;     // pic_particles_boundary_workspace_ints(bnd_cap) ints
    int bnd_cap = 0;
    // fusion reactant: the particles a fusion spent (id PIC_SPENT_ID) are listed here for the compaction, capacity + 1
    DeviceBuf<int> spent_work;
    int spent_cap = 0;
    bool do_not_push = false;      // <species>.do_not_push: x and u keep their bits (pic_engine_set_species_flags)
    bool do_not_deposit = false;   // <species>.do_not_deposit: no current deposition
    std::vector<FluxInjector> flux;
};

// Laser antenna: its own particle container (LaserParticleContainer), no gather, order-agnostic deposit
struct Laser {
    pic_laser_antenna prm;
    pic_soa P;                   // borrowed device arrays, P.np particles
    long capacity;
    DeviceBuf<int> bnd_work;
    int bnd_cap = 0;
    DeviceBuf<double> w_owned;   // multi-rank: weights masked to this rank's brick
};

// Per-stage CUDA-event timing of the step driver (pic_engine_enable_timing / pic_engine_stage_ms): the events are
// recorded on the stream the stages are launched on, inside the same pic_engine_evolve calls a benchmark times.
enum { ST_FILL_EB = 0, ST_GATHER_PUSH, ST_ZERO_J, ST_DEPOSIT, ST_SYNC_J, ST_EVOLVE_B, ST_FILL_B, ST_EVOLVE_E, ST_FILL_E,
       ST_WRAP, ST_MIGRATE, ST_SORT, ST_NCI, ST_WINDOW, ST_PUSHP, ST_FILTER, ST_FLUID_GATHER_PUSH, ST_FLUID_FILL,
       ST_FLUID_ADVECT, ST_FLUID_DEPOSIT, ST_COLLISIONS, ST_FUSION, ST_FUSION_PRODUCTS, ST_FLUX_INJECTION, ST_COUNT };
static const char* const stage_names[ST_COUNT] = {"fill_boundary_eb", "gather_push", "zero_j", "deposit", "sync_current",
    "evolve_b", "fill_boundary_b", "evolve_e", "fill_boundary_e", "wrap", "migrate", "sort", "nci_filter", "move_window", "push_p", "filter_j",
    "fluid_gather_push", "fluid_fill_boundary", "fluid_advect", "fluid_deposit", "collisions", "fusion", "fusion_products", "flux_injection"};
// Cold fluid species (WarpXFluidContainer): two borrowed states of N, NUx, NUy, NUz; the advection writes one from the
// other and `cur` names the current one.
struct Fluid {
    double q, m;
    pic_fab U[2][4];
    int cur = 0;
};

// One entry of collisions.collision_names (CollisionHandler): pairwise Coulomb collisions of species isp1 with isp2, or
// (fusion) nuclear fusion of isp1 with isp2 into iprod[0], iprod[1] (-1 for proton-boron: one product species) with
// its engine-owned pair workspace.
struct Collision {
    int isp1, isp2, ndt;
    double coulomb_log;
    uint64_t seed;
    bool fusion = false;
    int iprod[2] = {-1, -1};
    int type = 0;
    double multiplier = 1.0, threshold = 0.02, target = 0.002;
    DeviceBuf<char> work;
    long pair_cap = 0;
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
    DeviceBuf<double> jdep_mem[3];
    pic_stencil st;
    pic_fab fab[9];        // Ex Ey Ez Bx By Bz jx jy jz
    std::vector<Species> species;
    bool is_synchronized = true;
    long istep = 0;
    // multi-rank
    Comm* comm = nullptr;
    int nb[3] = {1, 1, 1}, coord[3] = {0, 0, 0};
    DeviceBuf<double> hbuf[4];                   // halo send lo/hi, recv lo/hi
    // non-periodic domains
    pic_boundaries bnd{};
    bool any_pec = false, all_periodic = true;
    bool do_moving_window = false;
    int mw_dir = 2;
    double mw_v = 0.0, mw_x = 0.0;               // moving_window_v [m/s], moving_window_x
    double gamma_boost = 1.0, beta_boost = 0.0;  // warpx.gamma_boost, boost_direction = z
    bool use_nci = false;                        // particles.use_fdtd_nci_corr
    double nci_stencil[2][5];                    // [0] Ex Ey Bz, [1] Bx By Ez
    pic_fab nci_fab[6];                          // filtered copies of E, B
    DeviceBuf<double> nci_mem[6];
    double cur_time = 0.0;                       // t_new[0]
    DeviceBuf<double> shift_tmp;                 // one component-sized scratch array
    PinnedBuf<int> host_count;                   // particles removed per container and pass, one per container + 1
    std::vector<Laser> lasers;
    std::vector<Fluid> fluids;
    std::vector<Collision> collisions;
    DeviceBuf<int> coll_status;                  // a cell exceeded the collision kernel's capacity
    int n_flux = 0;                              // flux injectors of all species
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

// Low/high neighbour exchange along one axis; along a non-periodic axis the bricks at the domain faces skip the
// missing side.  A message travelling upwards (sent to hi, received from lo) is posted first on both sides: with two
// bricks per axis both neighbours are the same rank and NCCL matches sends and receives of a pair of ranks in
// posting order.
static int exchange(Engine& e, int dim, const double* s_lo, const double* s_hi, double* r_lo, double* r_hi,
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

// The four halo message buffers hold at least n doubles each.  A failed allocation leaves that buffer empty: a later
// sweep allocates again or fails cleanly.
static int grow_halo_buffers(Engine& e, size_t n) {
    for (auto& b : e.hbuf)
        if (b.bytes() < sizeof(double) * n) ENG_CALL(b.alloc(sizeof(double) * n, "pic_engine: halo buffer allocation failed"));
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
                ENG_CALL(pic_halo_pack(&fabs[c], dim, side, ng, mode, e.hbuf[side].get() + off, s));
                off += (size_t)pic_halo_slab_count(&fabs[c], dim, ng, mode);
            }
        }
        ENG_CALL(exchange(e, dim, e.hbuf[0].get(), e.hbuf[1].get(), e.hbuf[2].get(), e.hbuf[3].get(), n, (cudaStream_t)s));
        for (int side = 0; side < 2; ++side) {
            if (!has_neighbour(e, dim, side)) continue;
            size_t off = 0;
            for (int c = 0; c < nfab; ++c) {
                ENG_CALL(pic_halo_unpack(&fabs[c], dim, side, ng, mode, e.hbuf[2 + side].get() + off, s));
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
    ENG_CALL(pic_halo_pack_multi(fabs, nfab, dim, ng, mode, e.hbuf[0].get(), e.hbuf[1].get(), s));
    ENG_CALL(exchange(e, dim, e.hbuf[0].get(), e.hbuf[1].get(), e.hbuf[2].get(), e.hbuf[3].get(), n, (cudaStream_t)s));
    ENG_CALL(pic_halo_unpack_multi(fabs, nfab, dim, ng, mode, e.hbuf[2].get(), e.hbuf[3].get(), s));
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

// the move a deferred sort left out: buf[cur] -> buf[1-cur] through the permutation
static int apply_pending(Species& sp, void* s) {
    if (!sp.ord.pending()) return 0;
    ENG_CALL(pic_sort_apply_permutation(&sp.buf[sp.cur], &sp.buf[1 - sp.cur], sp.ord.pending(), s));
    sp.cur = 1 - sp.cur;
    sp.ord.moved();
    return 0;
}

static int push(Engine& e, Species& sp, double dt, int push_position, void* s) {
    double xyzmin[3]; int lo[3];
    lower_corner(e, e.ng_EB, xyzmin, lo);
    // only the default supercell kernel of PushPX carries a pending sort; PushP, order 4 and the pair kernels get the
    // particles moved first
    if (!(push_position && sp.ord.has_bins() && gather_push_carries_permutation(e.nox))) ENG_CALL(apply_pending(sp, s));
    const pic_soa& P = sp.buf[sp.cur];
    if (push_position) sp.ord.pushed();
    if (push_position && sp.has_esc()) {
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
    }
    // the main push gathers from the NCI-filtered copies (PhysicalParticleContainer.cpp:1900-1911); PushP does not
    const pic_fab* EB = (e.use_nci && push_position) ? e.nci_fab : e.fab;
    if (const int* src = sp.ord.pending()) {
        sp.ord.moved();
        sp.cur = 1 - sp.cur;
        return pic_gather_push_permuted(&P, &sp.buf[sp.cur], src, &EB[0], &EB[3], e.dinv, xyzmin, lo, sp.q, sp.m, dt, e.nox,
                                        e.galerkin, e.pusher, &sp.ord.bins(), sp.has_esc() ? &sp.esc : nullptr, s);
    }
    return pic_gather_push(&P, 0, P.np, &EB[0], &EB[3], e.dinv, xyzmin, lo, sp.q, sp.m, dt, e.nox,
                           e.galerkin, e.pusher, push_position, sp.ord.bins_if_sorted(),
                           sp.has_esc() ? &sp.esc : nullptr, s);
}

// Engine-owned copies of n field components with the shapes of src (the NCI-filtered E, B; the deposition copy of J):
// either all n are allocated or none.
static int alloc_fab_copies(const pic_fab* src, int n, pic_fab* copy, DeviceBuf<double>* mem, const char* what) {
    DeviceBuf<double> m[6];
    for (int c = 0; c < n; ++c) ENG_CALL(m[c].alloc(sizeof(double) * (size_t)fab_size(src[c]), what));
    for (int c = 0; c < n; ++c) {
        mem[c] = std::move(m[c]);
        copy[c] = src[c];
        copy[c].p = mem[c].get();
    }
    return 0;
}

// PhysicalParticleContainer::applyNCIFilter for the rank's box (one tile): E, B -> the engine's filtered copies
static int apply_nci(Engine& e, void* s) {
    if (!e.nci_mem[0]) {
        ENG_CALL(alloc_fab_copies(e.fab, 6, e.nci_fab, e.nci_mem, "pic_engine: cannot allocate the NCI-filtered field copies"));
        for (int c = 0; c < 6; ++c) cudaMemsetAsync(e.nci_fab[c].p, 0, e.nci_mem[c].bytes(), (cudaStream_t)s);
    }
    for (int c = 0; c < 6; ++c) {
        const bool exeybz = (c == 0 || c == 1 || c == 5);              // :2132-2163
        ENG_CALL(pic_apply_nci_filter(&e.fab[c], &e.nci_fab[c], e.nci_stencil[exeybz ? 0 : 1], e.box_lo, e.box_hi, e.nox, s));
    }
    return 0;
}

// A species that is not pushed (do_not_push): the move a deferred sort left out happens here instead of in the gather
// + push, and its escape list is empty -- nothing left the domain or the brick.  Its bins stay exact.
static int hold(Species& sp, void* s) {
    ENG_CALL(apply_pending(sp, s));
    if (sp.has_esc()) cudaMemsetAsync(sp.esc.count, 0, sizeof(int), (cudaStream_t)s);
    sp.ord.held();
    return 0;
}

static int push_particles_and_deposit(Engine& e, void* s) {
    if (e.solver == PIC_SOLVER_NONE) {       // gather + push with the deposition skipped (WarpXEvolve.cpp:176-182)
        for (auto& sp : e.species) {
            Stage t(e, ST_GATHER_PUSH, s);
            ENG_CALL(sp.do_not_push ? hold(sp, s) : push(e, sp, e.dt, 1, s));
        }
        return 0;
    }
    {
        Stage t(e, ST_ZERO_J, s);
        if (e.use_filter && !e.jdep_mem[0])
            ENG_CALL(alloc_fab_copies(&e.fab[6], 3, e.jdep, e.jdep_mem, "pic_engine: cannot allocate the deposition copy of J (filter)"));
        const pic_fab* Jd = e.use_filter ? e.jdep : &e.fab[6];
        for (int c = 0; c < 3; ++c)                     // J.setVal(0), MultiParticleContainer.cpp:467-478
            cudaMemsetAsync(Jd[c].p, 0, sizeof(double) * (size_t)fab_size(Jd[c]), (cudaStream_t)s);
    }
    const pic_fab* Jd = e.use_filter ? e.jdep : &e.fab[6];
    double xyzmin[3]; int lo[3];
    lower_corner(e, e.ng_J, xyzmin, lo);
    if (e.use_nci && !e.species.empty()) { Stage t(e, ST_NCI, s); ENG_CALL(apply_nci(e, s)); }
    for (auto& sp : e.species) {
        { Stage t(e, ST_GATHER_PUSH, s); ENG_CALL(sp.do_not_push ? hold(sp, s) : push(e, sp, e.dt, 1, s)); }
        if (sp.do_not_deposit) continue;     // DepositCurrent returns early (WarpXParticleContainer.cpp:370)
        const pic_soa& P = sp.buf[sp.cur];
        Stage t(e, ST_DEPOSIT, s);
        ENG_CALL(pic_deposit_esirkepov(&P, 0, P.np, Jd, e.dinv, xyzmin, lo, sp.q, e.dt, -0.5 * e.dt,
                                       e.nox, sp.ord.bins_if_sorted(), s));
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
            ENG_CALL(pic_particles_owned_weights(&L.P, own_lo, own_hi, L.w_owned.get(), s));
            dep.w = L.w_owned.get();
        }
        ENG_CALL(pic_deposit_esirkepov(&dep, 0, dep.np, Jd, e.dinv, xyzmin, lo, 1.0, e.dt, -0.5 * e.dt,
                                       e.nox, nullptr, s));
    }
    return 0;
}

// defer: leave the move to the next gather + push (sp.ord.pending())
static int sort_species(Engine& e, Species& sp, bool defer, void* s) {
    ENG_CALL(apply_pending(sp, s));
    pic_soa& in = sp.buf[sp.cur];
    sp.buf[1 - sp.cur].np = in.np;
    const int* src = nullptr;
    ENG_CALL(pic_sort_index_by_cell(&in, &e.geom, &sp.ord.bins(), sp.sort_work, &src, s));
    sp.ord.sorted(in.np, src);
    return defer ? 0 : apply_pending(sp, s);
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
    int* head = sp.mig_head.get();
    int* work = sp.mig_work.get();
    int* counts = sp.mig_counts.get();
    int* idx[2] = {sp.mig_idx[0].get(), sp.mig_idx[1].get()};
    double* msg[4] = {sp.mig_msg[0].get(), sp.mig_msg[1].get(), sp.mig_msg[2].get(), sp.mig_msg[3].get()};
    for (int n = 0; n < 8; ++n) head[n] = 0;
    head[0] = (int)P.np;
    cudaMemcpyAsync(work, head, 8 * sizeof(int), cudaMemcpyHostToDevice, s);
    const int* np_dev = work;
    pic_soa view = P;
    view.np = sp.capacity;                       // launch bound only: the kernels read the count from np_dev
    // Who can leave: the particles the push of this step listed (nothing else moved since: periodic particle boundaries
    // remove nobody, no window shift re-drew the brick) -- else every particle is classified.
    const bool listed = sp.has_esc() && sp.ord.escape_list_current() && e.all_periodic && !e.do_moving_window &&
                        !g_migrate_full_sweep;
    for (int dim = 0; dim < 3; ++dim) {
        if (spans(e, dim)) continue;
        const bool np_dim = !e.geom.periodic[dim];
        if (listed) ++g_listed_sweeps;
        if (listed)
            ENG_CALL(pic_particles_classify_listed(&view, &e.geom, dim, e.box_lo[dim], e.box_hi[dim],
                                                   np_dim ? 2 : (e.nb[dim] == 2 ? 1 : 0), counts, idx[0], idx[1], cap,
                                                   np_dev, &sp.esc, s));
        else
        ENG_CALL(pic_particles_classify(&view, &e.geom, dim, e.box_lo[dim], e.box_hi[dim],
                                        np_dim ? 2 : (e.nb[dim] == 2 ? 1 : 0), counts, idx[0], idx[1], cap, np_dev, s));
        peak_kernel<<<1, 1, 0, s>>>(work + 6, counts);
        count_launch();
        ENG_CALL(pic_migrate_pack(&view, idx[0], counts, cap, msg[0], s));
        ENG_CALL(pic_migrate_pack(&view, idx[1], counts + 1, cap, msg[1], s));
        // a missing neighbour (beyond a non-periodic face) sends nothing: its message reads "0 particles"
        for (int side = 0; side < 2; ++side)
            if (!has_neighbour(e, dim, side)) cudaMemsetAsync(msg[2 + side], 0, sizeof(double), s);
        ENG_CALL(exchange(e, dim, msg[0], msg[1], msg[2], msg[3], nmsg, s));
        ENG_CALL(pic_migrate_unpack(&view, counts, idx[0], idx[1], msg[2], msg[3], cap, sp.capacity, work, np_dev, s));
        if (listed) ENG_CALL(pic_migrate_note_appended(work, &sp.esc, s));     // arrivals may have to travel on
    }
    sp.ord.escape_list_spent();
    ENG_NCCL(g_nccl.AllReduce(work + 6, work + 6, 1, PIC_NCCL_INT32, PIC_NCCL_MAX, e.comm->comm, s));
    cudaMemcpyAsync(head, work, 8 * sizeof(int), cudaMemcpyDeviceToHost, s);
    if (cudaStreamSynchronize(s) != cudaSuccess) return fail("pic_engine: migration failed (%s)", cudaGetErrorString(cudaGetLastError()));
    const int np_new = head[0], status = head[1], seen = head[6];
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
    if (bytes > e.shift_tmp.bytes()) ENG_CALL(e.shift_tmp.alloc(bytes, "pic_engine: moving-window scratch allocation failed"));
    return pic_shift_fab(&e.fab[c], e.shift_tmp.get(), &e.geom, num_shift, e.mw_dir, 0.0 /* no external field */, s);
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
    for (auto& sp : e.species) sp.ord.cells_changed();     // every particle changed cell along dir
    *num_moved = nsb;
    return 0;
}

// One particle container of a removal pass (a species, or an antenna when sp is null) and the workspace its marks go to
struct Removal {
    Species* sp; Laser* L; int* work; int cap;
    pic_soa& P() const { return sp ? sp->buf[sp->cur] : L->P; }
};

// The removal AMReX Redistribute performs: mark(r) lists the particles of every container r to remove (work[0] = how
// many), ONE host read of the counts, then the compactions.
template <class Mark>
static int remove_marked(Engine& e, const std::vector<Removal>& rs, Mark mark, const char* pass, cudaStream_t s) {
    if (rs.empty()) return 0;
    for (size_t n = 0; n < rs.size(); ++n) {
        ENG_CALL(mark(rs[n]));
        cudaMemcpyAsync(e.host_count.get() + n, rs[n].work, sizeof(int), cudaMemcpyDeviceToHost, s);
    }
    if (cudaStreamSynchronize(s) != cudaSuccess) return fail("pic_engine: %s failed (%s)", pass, cudaGetErrorString(cudaGetLastError()));
    for (size_t n = 0; n < rs.size(); ++n) {
        const int lost = e.host_count.get()[n];
        if (lost == 0) continue;
        pic_soa& P = rs[n].P();
        ENG_CALL(pic_particles_boundary_compact(&P, rs[n].work, rs[n].cap, lost, s));
        P.np -= lost;
        if (rs[n].sp) rs[n].sp->ord.cells_changed();
    }
    return 0;
}

// mypc->ApplyBoundaryConditions() over species and lasers (MultiParticleContainer.cpp:659-664) and the removal
static int apply_particle_boundaries(Engine& e, void* stream) {
    if (e.all_periodic) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    std::vector<Removal> rs;
    for (auto& sp : e.species) rs.push_back({&sp, nullptr, sp.bnd_work.get(), sp.bnd_cap});
    for (auto& L : e.lasers) rs.push_back({nullptr, &L, L.bnd_work.get(), L.bnd_cap});
    return remove_marked(e, rs, [&](const Removal& r) { return pic_particles_boundary_mark(&r.P(), &e.geom, &e.bnd, r.work, r.cap, s); },
                         "particle boundary pass", s);
}

// WarpXFluidContainer::Evolve (Source/Fluids/WarpXFluidContainer.cpp:257-314) on a periodic domain: GatherAndPush,
// the FillBoundary of N and NU with all 2 guard nodes (ApplyBcFluidsAndComms :413-417), AdvectivePush_Muscl into the
// other state, DepositCurrent into the J the particles deposit into (filtered afterwards like theirs).
static int evolve_fluid(Engine& e, Fluid& fl, void* s) {
    pic_fab* U = fl.U[fl.cur];
    { Stage t(e, ST_FLUID_GATHER_PUSH, s); ENG_CALL(pic_fluid_gather_push(U, &e.fab[0], &e.fab[3], fl.q, fl.m, e.dt, s)); }
    { Stage t(e, ST_FLUID_FILL, s); for (int d = 0; d < 3; ++d) ENG_CALL(halo_sweep(e, U, 4, d, 2, 0, s)); }
    { Stage t(e, ST_FLUID_ADVECT, s); ENG_CALL(pic_fluid_advect(U, fl.U[1 - fl.cur], e.dx, e.dt, nullptr, s)); }
    fl.cur = 1 - fl.cur;
    Stage t(e, ST_FLUID_DEPOSIT, s);
    return pic_fluid_deposit_current(fl.U[fl.cur], e.use_filter ? e.jdep : &e.fab[6], fl.q, s);
}

// MultiParticleContainer::doCollisions -> CollisionHandler::doCollisions (Particles/Collision/CollisionHandler.cpp:85-93)
// at t_new: a collision runs when int(floor(t / dt)) % ndt == 0, with dt * ndt.  Its species need their current cells:
// one not sorted since its last position push (or with particles appended behind the bins) is sorted here first, with
// the move left to this step's gather + push like the end-of-step sort.
// The parameters pic_coulomb_collision and pic_fusion_collision share, for entry ic of the collisions
template <class Prm>
static Prm pair_params(const Collision& c, int ic, Species* const sp[2]) {
    Prm p{};
    p.q1 = sp[0]->q; p.m1 = sp[0]->m; p.q2 = sp[1]->q; p.m2 = sp[1]->m;
    p.seed = c.seed; p.collision_index = ic; p.same_species = c.isp1 == c.isp2 ? 1 : 0;
    return p;
}
// the part of a colliding species' sort workspace that is free until its next sort
static int* sort_scratch(const Species& sp) { return pic_sort_scratch(sp.sort_work, sp.ord.bins().np_binned); }

static int do_fusion(Engine& e, const Collision& c, int ic, Species* sp[2], void* s) {
    pic_fusion_collision fc = pair_params<pic_fusion_collision>(c, ic, sp);
    const bool pb = c.type == PIC_FUSION_PB_3HE4;      // one product species: six alphas per event
    Species* pr[2] = {&e.species[c.iprod[0]], pb ? nullptr : &e.species[c.iprod[1]]};
    fc.mA = pr[0]->m; fc.mB = pb ? 0.0 : pr[1]->m;
    fc.type = c.type; fc.fusion_multiplier = c.multiplier;
    fc.fusion_probability_threshold = c.threshold; fc.fusion_probability_target_value = c.target;
    {
        Stage t(e, ST_FUSION, s);
        ENG_CALL(pic_collide_nuclear_fusion(&fc, &sp[0]->buf[sp[0]->cur], &sp[0]->ord.bins(), sp[0]->ord.pending(),
                                            &sp[1]->buf[sp[1]->cur], &sp[1]->ord.bins(), sp[1]->ord.pending(), &e.geom,
                                            e.dt * c.ndt, e.istep, sort_scratch(*sp[0]), sort_scratch(*sp[1]), c.work.get(),
                                            c.pair_cap, e.coll_status.get(), s));
    }
    Stage t(e, ST_FUSION_PRODUCTS, s);
    for (Species* p : pr)                // products are appended behind the particles in place
        if (p) ENG_CALL(apply_pending(*p, s));
    long nev = 0;
    ENG_CALL(pic_fusion_create_products(&fc, &sp[0]->buf[sp[0]->cur], &sp[0]->ord.bins(), &sp[1]->buf[sp[1]->cur],
                                        &sp[1]->ord.bins(), &e.geom, e.istep, c.work.get(), c.pair_cap, &pr[0]->buf[pr[0]->cur],
                                        pr[0]->capacity, pr[0]->next_id, pb ? nullptr : &pr[1]->buf[pr[1]->cur],
                                        pb ? 0 : pr[1]->capacity, pb ? 0 : pr[1]->next_id, &nev, s));
    const long per_event = pb ? 6 : 2;
    for (Species* p : pr) {
        if (!p) continue;
        p->buf[p->cur].np += per_event * nev;
        p->next_id += (uint64_t)(per_event * nev);
        if (nev) p->ord.cells_changed();
    }
    return 0;
}

static int do_collisions(Engine& e, void* s) {
    for (size_t ic = 0; ic < e.collisions.size(); ++ic) {
        const Collision& c = e.collisions[ic];
        if (int(std::floor(e.cur_time / e.dt)) % c.ndt != 0) continue;
        Species* sp[2] = {&e.species[c.isp1], &e.species[c.isp2]};
        for (Species* p : sp)
            if (p->ord.collision_needs_sort(p->buf[p->cur].np)) {
                Stage t(e, ST_SORT, s);
                ENG_CALL(sort_species(e, *p, true, s));
            }
        if (c.fusion) { ENG_CALL(do_fusion(e, c, (int)ic, sp, s)); continue; }
        Stage t(e, ST_COLLISIONS, s);
        pic_coulomb_collision cc = pair_params<pic_coulomb_collision>(c, (int)ic, sp);
        cc.coulomb_log = c.coulomb_log;
        ENG_CALL(pic_collide_pairwise_coulomb(&cc, &sp[0]->buf[sp[0]->cur], &sp[0]->ord.bins(), sp[0]->ord.pending(),
                                              &sp[1]->buf[sp[1]->cur], &sp[1]->ord.bins(), sp[1]->ord.pending(), &e.geom,
                                              e.dt * c.ndt, e.istep, sort_scratch(*sp[0]), sort_scratch(*sp[1]),
                                              e.coll_status.get(), s));
    }
    return 0;
}

// The reactants a fusion spent leave with the particles lost at the boundaries (the reference's
// deleteInvalidParticles, BinaryCollision.H:212-218), in a pass of their own: the marks must see the compacted arrays.
static int remove_spent(Engine& e, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    std::vector<Removal> rs;
    for (auto& sp : e.species)
        if (sp.spent_work) rs.push_back({&sp, nullptr, sp.spent_work.get(), sp.spent_cap});
    return remove_marked(e, rs, [&](const Removal& r) {
        ENG_CALL(apply_pending(*r.sp, s));
        return pic_particles_mark_spent(&r.P(), r.work, r.cap, s);
    }, "spent-reactant pass", s);
}

// PhysicalParticleContainer::ContinuousFluxInjection (PhysicalParticleContainer.cpp:2531-2540), the first thing
// HandleParticlesAtBoundaries does (WarpXEvolve.cpp:535): each injector's particles of this step go behind the species'
// particles and join its escape list, so that the wrap, the particle boundaries and the migration of the step treat
// them as pushed particles.
static int flux_injection(Engine& e, long step, void* s) {
    for (auto& sp : e.species) {
        if (sp.flux.empty()) continue;
        ENG_CALL(apply_pending(sp, s));
        pic_soa& P = sp.buf[sp.cur];
        const long np0 = P.np;
        for (auto& f : sp.flux) {
            uint64_t used = 0;
            const long n = pic_add_flux_particles(&f.prm, f.index, &e.geom, e.box_lo, e.box_hi, step, e.cur_time, e.dt, &P,
                                                  sp.capacity, sp.next_id, &used, f.work.get(), (long)f.work.bytes(), s);
            if (n < 0) return 1;
            P.np += n;
            sp.next_id += used;
        }
        if (P.np == np0) continue;
        sp.ord.cells_changed();
        if (sp.has_esc()) ENG_CALL(flux_list_escapes(&sp.esc, np0, P.np - np0, s));
    }
    return 0;
}

// last: Synchronize() ends the step; defer_sort: another step of the same call follows, its push moves the sorted particles
static int one_step(Engine& e, bool last, bool defer_sort, void* s) {
    // ---- ExplicitFillBoundaryEBUpdateAux ----
    if (e.is_synchronized) {
        { Stage t(e, ST_FILL_EB, s); ENG_CALL(fill_boundary(e, 0, 6, e.ng_EB, s)); }                    // ng_alloc_EB, :487-488
        {                                                                 // PushP(-dt/2), :492-504
            Stage t(e, ST_PUSHP, s);
            for (auto& sp : e.species) if (!sp.do_not_push) ENG_CALL(push(e, sp, -0.5 * e.dt, 0, s));
        }
        e.is_synchronized = false;
    } else {
        Stage t(e, ST_FILL_EB, s);
        ENG_CALL(fill_boundary(e, 0, 6, e.ng_FG, s));                    // :515-516
    }
    // ---- mypc->doCollisions, :157-159 ----
    if (!e.collisions.empty()) ENG_CALL(do_collisions(e, s));
    // ---- OneStep_nosub ----
    ENG_CALL(push_particles_and_deposit(e, s));
    for (auto& fl : e.fluids) ENG_CALL(evolve_fluid(e, fl, s));      // myfl->Evolve, :1171-1178
    if (e.solver != PIC_SOLVER_NONE) {                                    // no J, no field update (:176-182)
        if (e.use_filter) { Stage t(e, ST_FILTER, s); ENG_CALL(pic_apply_filter_multi(e.jdep, &e.fab[6], 3, e.npass, s)); }
        { Stage t(e, ST_SYNC_J, s); ENG_CALL(sync_current(e, s)); }
        { Stage t(e, ST_EVOLVE_B, s); ENG_CALL(evolve_b(e, 0.5 * e.dt, s)); }
        { Stage t(e, ST_FILL_B, s); ENG_CALL(fill_boundary(e, 3, 6, e.ng_FS, s)); }
        { Stage t(e, ST_EVOLVE_E, s); ENG_CALL(evolve_e(e, e.dt, s)); }
        { Stage t(e, ST_FILL_E, s); ENG_CALL(fill_boundary(e, 0, 3, e.ng_FS, s)); }
        { Stage t(e, ST_EVOLVE_B, s); ENG_CALL(evolve_b(e, 0.5 * e.dt, s)); }
    }
    if (last) {                                                           // Synchronize(), :64-91
        { Stage t(e, ST_FILL_EB, s); ENG_CALL(fill_boundary(e, 0, 6, e.ng_FG, s)); }
        {
            Stage t(e, ST_PUSHP, s);
            for (auto& sp : e.species) if (!sp.do_not_push) ENG_CALL(push(e, sp, 0.5 * e.dt, 0, s));
        }
        e.is_synchronized = true;
    }
    const long step = e.istep++;
    e.cur_time += e.dt;                                                   // :232
    // ---- MoveWindow(step+1, move_j = is_synchronized), :247 ----
    int num_moved = 0;
    { Stage t(e, ST_WINDOW, s); ENG_CALL(move_window(e, e.is_synchronized, &num_moved, s)); }
    // ---- HandleParticlesAtBoundaries ----
    if (e.n_flux) { Stage t(e, ST_FLUX_INJECTION, s); ENG_CALL(flux_injection(e, step, s)); }
    {
        Stage t(e, ST_WRAP, s);
        for (auto& sp : e.species) {
            // amrex enforcePeriodic: only the particles the push of this step moved out of the domain
            // (done before the removal below, while the indices listed by the push are still valid; the
            // two act on different directions)
            if (sp.has_esc()) ENG_CALL(pic_particles_wrap_listed(&sp.buf[sp.cur], &e.geom, &sp.esc, s));
            else ENG_CALL(pic_particles_wrap_periodic(&sp.buf[sp.cur], &e.geom, s));
        }
        for (auto& L : e.lasers) ENG_CALL(pic_particles_wrap_periodic(&L.P, &e.geom, s));
        ENG_CALL(apply_particle_boundaries(e, s));
        ENG_CALL(remove_spent(e, s));
    }
    for (auto& sp : e.species) {
        if (e.comm) { Stage t(e, ST_MIGRATE, s); ENG_CALL(migrate(e, sp, s)); }
        const bool due = sp.ord.end_of_step_sort_due(e.sort_interval > 0 && (step + 1) % e.sort_interval == 0);
        if (sp.sort_work && due) { Stage t(e, ST_SORT, s); ENG_CALL(sort_species(e, sp, defer_sort, s)); }
    }
    if (e.tm.on && e.tm.recs.size() > 4096) collect_timing(e);          // bound the event pool of long runs
    return 0;
}

}  // namespace pic

using namespace pic;

// The particle-boundary scratch of a container of `capacity` particles
static int alloc_boundary_scratch(long capacity, DeviceBuf<int>& work, int* cap) {
    const long c = capacity / 16 + 65536;
    *cap = (int)(c < capacity + 1 ? c : capacity + 1);
    return work.alloc(sizeof(int) * (size_t)pic_particles_boundary_workspace_ints(*cap),
                      "pic_engine: cannot allocate the particle-boundary scratch");
}
// The pinned counts of the removal passes for the engine's containers and one more, plus a spare slot
static int alloc_host_counts_for_one_more(const Engine& e, PinnedBuf<int>& counts) {
    return counts.alloc(sizeof(int) * (e.species.size() + e.lasers.size() + 2), "pic_engine: cannot allocate pinned host memory");
}

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
    if (solver == PIC_SOLVER_NONE && !(dt > 0)) { fail("pic_engine_create: algo.maxwell_solver = none needs an explicit dt"); return nullptr; }
    if (solver == PIC_SOLVER_NONE && use_filter) { fail("pic_engine_create: algo.maxwell_solver = none takes no current filter"); return nullptr; }
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
    if (solver != PIC_SOLVER_NONE) stencil_coefficients(solver, e->dx, &e->st);
    else e->st = pic_stencil{};
    guard_cells(*e);
    return e;
}
extern "C" void pic_engine_destroy(void* h) {
    Engine* e = static_cast<Engine*>(h);
#ifndef PIC_SIMT_HOST
    if (e) for (cudaEvent_t ev : e->tm.pool) cudaEventDestroy(ev);
#endif
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
    for (auto& m : e->jdep_mem) m.release();     // new shapes
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
// Over several ranks (collective): the sum of n over the ranks, the particle count of the single box that would hold
// every brick's particles.  A new species' id counter starts there on every rank, so that the ids a species creates
// later (flux injection) are the same on any decomposition.
static int global_count(Engine& e, long n, uint64_t* out, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    DeviceBuf<double> d;
    ENG_CALL(d.alloc(sizeof(double), "pic_engine_add_species: cannot allocate the count scratch"));
    double v = (double)n;            // exact below 2^53
    cudaMemcpyAsync(d.get(), &v, sizeof(double), cudaMemcpyHostToDevice, s);
    ENG_NCCL(g_nccl.AllReduce(d.get(), d.get(), 1, PIC_NCCL_FLOAT64, PIC_NCCL_SUM, e.comm->comm, s));
    cudaMemcpyAsync(&v, d.get(), sizeof(double), cudaMemcpyDeviceToHost, s);
    if (cudaStreamSynchronize(s) != cudaSuccess) return fail("pic_engine_add_species: %s", cudaGetErrorString(cudaGetLastError()));
    *out = (uint64_t)v;
    return 0;
}

// bufA holds the particles; bufB is the sort target.  cell_start / sort_work may be NULL (no bins).
extern "C" int pic_engine_add_species(void* h, double q, double m, const pic_soa* bufA, const pic_soa* bufB,
                                      long capacity, int* cell_start, const int tile[3], void* sort_work,
                                      void* stream) {
    Engine* e = static_cast<Engine*>(h);
    PIC_REQUIRE(capacity >= bufA->np, "pic_engine_add_species: capacity %ld < np %ld", capacity, (long)bufA->np);
    PIC_REQUIRE(e->fluids.empty(), "pic_engine_add_species: runs with fluid species take no particle species yet");
    pic_bins bins{};
    bins.cell_start = cell_start;
    for (int d = 0; d < 3; ++d) {
        bins.box_lo[d] = e->box_lo[d]; bins.box_hi[d] = e->box_hi[d];
        bins.tile[d] = tile ? tile[d] : 8;
    }
    // Everything is allocated for a local species; the engine takes it only when the call succeeds.
    Species sp(q, m, bins);
    sp.capacity = capacity;
    sp.next_id = (uint64_t)bufA->np;     // ids of particles created later (fusion products) follow the initial ones
    sp.buf[0] = *bufA; sp.buf[1] = *bufB; sp.sort_work = sort_work;
    // escape list: a layer of one cell next to every domain face can leave per step at most
    const long esc_cap = capacity / 16 + 65536;
    if (sp.esc_mem.try_alloc(sizeof(int) * (size_t)(esc_cap + 1))) {
        sp.esc.count = sp.esc_mem.get(); sp.esc.idx = sp.esc_mem.get() + 1; sp.esc.capacity = (int)esc_cap;
        for (int d = 0; d < 3; ++d) {
            sp.esc.lo[d] = e->geom.periodic[d] ? e->geom.prob_lo[d] : -INFINITY;
            sp.esc.hi[d] = e->geom.periodic[d] ? e->geom.prob_hi[d] : INFINITY;
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
        const char* what = "pic_engine_add_species: cannot allocate the migration buffers";
        ENG_CALL(sp.mig_counts.alloc(2 * sizeof(int), what));
        for (auto& b : sp.mig_idx) ENG_CALL(b.alloc(sizeof(int) * (size_t)sp.mig_cap_max, what));
        for (auto& b : sp.mig_msg) ENG_CALL(b.alloc(sizeof(double) * nmsg, what));
        ENG_CALL(sp.mig_work.alloc((size_t)pic_migrate_workspace_bytes(sp.mig_cap_max), what));
        ENG_CALL(sp.mig_head.alloc(8 * sizeof(int), what));
        for (auto& b : sp.mig_msg) cudaMemsetAsync(b.get(), 0, sizeof(double) * nmsg, (cudaStream_t)stream);
        cudaMemsetAsync(sp.mig_work.get(), 0, (size_t)pic_migrate_workspace_bytes(sp.mig_cap_max), (cudaStream_t)stream);
    }
    if (!e->all_periodic) ENG_CALL(alloc_boundary_scratch(capacity, sp.bnd_work, &sp.bnd_cap));
    if (e->comm) ENG_CALL(global_count(*e, (long)bufA->np, &sp.next_id, stream));
    PinnedBuf<int> counts;
    ENG_CALL(alloc_host_counts_for_one_more(*e, counts));
    if (cell_start && sort_work) ENG_CALL(sort_species(*e, sp, false, stream));
    e->species.push_back(std::move(sp));
    e->host_count = std::move(counts);
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
        sp.ord.escape_list_spent();      // the caller moved the particles, not the push: classify every one
        if (e->comm) ENG_CALL(migrate(*e, sp, stream));
        sp.ord.cells_changed();
    }
    return 0;
}

// ---- non-periodic runs ------------------------------------------------------------------------
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
    PIC_REQUIRE(e->n_flux == 0, "pic_engine_set_boost: boosted frames take no flux injection");
    e->gamma_boost = gamma_boost; e->beta_boost = beta_boost;
    return 0;
}
// particles.use_fdtd_nci_corr (MultiParticleContainer.cpp:327, WarpX::InitNCICorrector, WarpXInitData.cpp:858-890)
extern "C" int pic_engine_set_nci_corrector(void* h, const double stencil_exeybz[5], const double stencil_bxbyez[5]) {
    Engine* e = static_cast<Engine*>(h);
    PIC_REQUIRE(e->species.empty() && e->lasers.empty(), "pic_engine_set_nci_corrector: call before adding particles");
    PIC_REQUIRE(e->solver != PIC_SOLVER_NONE, "pic_engine_set_nci_corrector: algo.maxwell_solver = none has no field solver to correct");
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
    PIC_REQUIRE(e->solver != PIC_SOLVER_NONE, "pic_engine_add_laser: algo.maxwell_solver = none deposits no current");
    double info[4];
    PIC_REQUIRE(same_boost(*e, prm->gamma_boost, prm->beta_boost), "pic_engine_add_laser: the antenna's gamma_boost / beta_boost differ from pic_engine_set_boost");
    ENG_CALL(pic_laser_antenna_info(prm, e->dx, info));
    PIC_REQUIRE(capacity >= p->np, "pic_engine_add_laser: capacity %ld < np %ld", capacity, (long)p->np);
    Laser L;
    L.prm = *prm; L.P = *p; L.capacity = capacity;
    if (!e->all_periodic) ENG_CALL(alloc_boundary_scratch(capacity, L.bnd_work, &L.bnd_cap));
    if (e->comm) ENG_CALL(L.w_owned.alloc(sizeof(double) * (size_t)(capacity > 0 ? capacity : 1),
                                          "pic_engine_add_laser: cannot allocate the weight scratch"));
    PinnedBuf<int> counts;
    ENG_CALL(alloc_host_counts_for_one_more(*e, counts));
    e->lasers.push_back(std::move(L));
    e->host_count = std::move(counts);
    return 0;
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
    if (!e->collisions.empty()) cudaMemsetAsync(e->coll_status.get(), 0, sizeof(int), (cudaStream_t)stream);
    for (int n = 0; n < numsteps; ++n) {
        const bool final_step = n == numsteps - 1;
        ENG_CALL(one_step(*e, synchronize_last && final_step, !final_step, stream));
    }
    if (!e->collisions.empty()) {        // one read per call: did a cell exceed the collision kernel's capacity?
        int st = 0;
        cudaMemcpyAsync(&st, e->coll_status.get(), sizeof(int), cudaMemcpyDeviceToHost, (cudaStream_t)stream);
        if (cudaStreamSynchronize((cudaStream_t)stream) != cudaSuccess)
            return fail("pic_engine_evolve: %s", cudaGetErrorString(cudaGetLastError()));
        PIC_REQUIRE(st == 0, "pic_engine_evolve: a collision found no scratch for a cell of more than 2048 particles");
    }
    return 0;
}

// The refusals every collision entry shares (who: the calling function); checked before the engine changes.
static int check_collision_entry(const Engine& e, const char* who, int isp1, int isp2, int ndt) {
    const int nsp = (int)e.species.size();
    PIC_REQUIRE(isp1 >= 0 && isp1 < nsp && isp2 >= 0 && isp2 < nsp, "%s: no species %d / %d", who, isp1, isp2);
    PIC_REQUIRE(ndt >= 1, "%s: ndt must be at least 1 (got %d)", who, ndt);
    PIC_REQUIRE(e.fluids.empty(), "%s: runs with fluid species take no collisions", who);
    PIC_REQUIRE(e.comm == nullptr, "%s: one rank only (collisions over several ranks are not yet checked against a "
                                   "single box)", who);
    for (int isp : {isp1, isp2}) {
        const pic_bins& b = e.species[isp].ord.bins();
        PIC_REQUIRE(e.species[isp].sort_work && b.cell_start, "%s: species %d has no cell bins", who, isp);
        for (int d = 0; d < 3; ++d)
            PIC_REQUIRE(b.tile[d] == e.species[isp1].ord.bins().tile[d], "%s: the species' bins use different tiles", who);
    }
    return 0;
}

extern "C" int pic_engine_add_collision(void* h, int isp1, int isp2, double coulomb_log, int ndt, uint64_t seed) {
    Engine* e = static_cast<Engine*>(h);
    PIC_REQUIRE(e, "pic_engine_add_collision: no engine");
    ENG_CALL(check_collision_entry(*e, "pic_engine_add_collision", isp1, isp2, ndt));
    // a Coulomb entry after a fusion on one of its species would meet the reactants that fusion spent in the same step
    // (they leave at the end of the step); the reference removes them between the two collisions
    for (const Collision& c : e->collisions)
        PIC_REQUIRE(!c.fusion || (c.isp1 != isp1 && c.isp1 != isp2 && c.isp2 != isp1 && c.isp2 != isp2),
                    "pic_engine_add_collision: species %d / %d are reactants of an earlier fusion entry; register the "
                    "Coulomb collision before the fusion", isp1, isp2);
    DeviceBuf<int> status;
    if (!e->coll_status) ENG_CALL(status.alloc(sizeof(int), "pic_engine_add_collision: cannot allocate the status word"));
    if (status) e->coll_status = std::move(status);
    e->collisions.push_back(Collision{isp1, isp2, ndt, coulomb_log, seed});
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
    PIC_REQUIRE(e->solver != PIC_SOLVER_NONE, "pic_engine_add_fluid_species: algo.maxwell_solver = none is not supported");
    PIC_REQUIRE(e->collisions.empty(), "pic_engine_add_fluid_species: runs with collisions take no fluids");
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

// One nuclearfusion entry of collisions.collision_names: see include/pic_b200.h.  Every precondition is checked before
// the engine changes; the pair workspace and the removal lists of the reactants are allocated here.
extern "C" int pic_engine_add_fusion(void* h, int isp1, int isp2, int iprodA, int iprodB, int type, double multiplier,
                                     double probability_threshold, double probability_target_value, int ndt, uint64_t seed) {
    Engine* e = static_cast<Engine*>(h);
    PIC_REQUIRE(e, "pic_engine_add_fusion: no engine");
    const int nsp = (int)e->species.size();
    PIC_REQUIRE(type == PIC_FUSION_DT_NHE4 || type == PIC_FUSION_DD_PT || type == PIC_FUSION_DD_NHE3 ||
                type == PIC_FUSION_PB_3HE4, "pic_engine_add_fusion: unknown fusion type %d", type);
    const bool pb = type == PIC_FUSION_PB_3HE4;         // one product species
    PIC_REQUIRE(pb == (iprodB == -1),
                pb ? "pic_engine_add_fusion: proton-boron fusion takes one product species (iprodB = -1)"
                   : "pic_engine_add_fusion: this reaction takes two product species");
    for (int i : {isp1, isp2, iprodA, iprodB})
        PIC_REQUIRE((pb && i == iprodB) || (i >= 0 && i < nsp), "pic_engine_add_fusion: no species %d", i);
    PIC_REQUIRE(iprodA != iprodB, "pic_engine_add_fusion: the two products must be different species");
    for (int i : {iprodA, iprodB})
        PIC_REQUIRE(i != isp1 && i != isp2, "pic_engine_add_fusion: a product species (%d) cannot be a reactant", i);
    PIC_REQUIRE(multiplier > 0.0 && probability_threshold > 0.0 && probability_target_value > 0.0,
                "pic_engine_add_fusion: the multiplier, threshold and target value must be positive");
    ENG_CALL(check_collision_entry(*e, "pic_engine_add_fusion", isp1, isp2, ndt));
    Collision c{isp1, isp2, ndt, 0.0, seed};
    c.fusion = true; c.iprod[0] = iprodA; c.iprod[1] = iprodB; c.type = type;
    c.multiplier = multiplier; c.threshold = probability_threshold; c.target = probability_target_value;
    c.pair_cap = e->species[isp1].capacity + (isp1 == isp2 ? 0 : e->species[isp2].capacity);
    const long nbins = pic_bins_count(e->box_lo, e->box_hi, e->species[isp1].ord.bins().tile);
    const char* what = "pic_engine_add_fusion: cannot allocate the fusion workspace";
    ENG_CALL(c.work.alloc((size_t)pic_fusion_workspace_bytes(c.pair_cap, nbins), what));
    DeviceBuf<int> status, spent[2];
    if (!e->coll_status) ENG_CALL(status.alloc(sizeof(int), what));
    for (int k = 0; k < 2; ++k) {
        const Species& sp = e->species[k ? isp2 : isp1];
        if (sp.spent_work || (k == 1 && isp1 == isp2)) continue;
        ENG_CALL(spent[k].alloc(sizeof(int) * (size_t)pic_particles_boundary_workspace_ints((int)(sp.capacity + 1)), what));
    }
    if (status) e->coll_status = std::move(status);
    for (int k = 0; k < 2; ++k)
        if (spent[k]) {
            Species& sp = e->species[k ? isp2 : isp1];
            sp.spent_work = std::move(spent[k]);
            sp.spent_cap = (int)(sp.capacity + 1);
        }
    e->collisions.push_back(std::move(c));
    return 0;
}

// The id the next particle species isp creates (fusion products, injected plasma) receives; a restart sets it from the
// checkpoint so that new ids never repeat old ones.  The setter refuses a counter below the species' particle count.
extern "C" uint64_t pic_engine_species_next_id(void* h, int isp) {
    Engine* e = static_cast<Engine*>(h);
    return (e && isp >= 0 && isp < (int)e->species.size()) ? e->species[isp].next_id : 0;
}
extern "C" int pic_engine_set_species_next_id(void* h, int isp, uint64_t next_id) {
    Engine* e = static_cast<Engine*>(h);
    PIC_REQUIRE(e && isp >= 0 && isp < (int)e->species.size(), "pic_engine_set_species_next_id: no species %d", isp);
    Species& sp = e->species[isp];
    PIC_REQUIRE(next_id >= (uint64_t)sp.buf[sp.cur].np, "pic_engine_set_species_next_id: %llu is below the %ld particles",
                (unsigned long long)next_id, (long)sp.buf[sp.cur].np);
    sp.next_id = next_id;
    return 0;
}

// One NFluxPerCell source of species isp (include/pic_b200.h); refused before the engine changes.
extern "C" int pic_engine_add_flux_injector(void* h, int isp, const pic_flux_injector* inj) {
    Engine* e = static_cast<Engine*>(h);
    PIC_REQUIRE(e && inj, "pic_engine_add_flux_injector: null argument");
    PIC_REQUIRE(isp >= 0 && isp < (int)e->species.size(), "pic_engine_add_flux_injector: no species %d", isp);
    PIC_REQUIRE(!e->do_moving_window, "pic_engine_add_flux_injector: runs with a moving window take no flux injection");
    PIC_REQUIRE(!(e->gamma_boost > 1.0), "pic_engine_add_flux_injector: boosted frames take no flux injection");
    const long bytes = pic_flux_workspace_bytes(inj, &e->geom);
    if (bytes < 0) return 1;
    FluxInjector f;
    f.prm = *inj;
    f.index = e->n_flux;
    ENG_CALL(f.work.alloc((size_t)bytes, "pic_engine_add_flux_injector: cannot allocate the injection workspace"));
    e->species[isp].flux.push_back(std::move(f));
    ++e->n_flux;
    return 0;
}

extern "C" int pic_engine_set_species_flags(void* h, int isp, int do_not_push, int do_not_deposit) {
    Engine* e = static_cast<Engine*>(h);
    PIC_REQUIRE(e && isp >= 0 && isp < (int)e->species.size(), "pic_engine_set_species_flags: no species %d", isp);
    e->species[isp].do_not_push = do_not_push != 0;
    e->species[isp].do_not_deposit = do_not_deposit != 0;
    return 0;
}
