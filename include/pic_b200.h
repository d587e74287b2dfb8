/* pic_b200.h -- C ABI of the PIC step engine (CUDA, sm_90a / H100).
 *
 * Every entry point replaces ONE host-side call site of ECP-WarpX/WarpX's explicit
 * electromagnetic PIC step (reference paths are relative to the ECP-WarpX/WarpX tree).  WarpX has no
 * plugin registry for this path: the seam is the argument set of each call site, which
 * decays to raw device pointers + index metadata.  These are those argument sets, as POD.
 *
 * Conventions (identical to the reference, SURVEY.md Appendix A):
 *   - all arithmetic is fp64 (WarpX_PRECISION=DOUBLE); indices are global level-0 indices;
 *   - arrays are Fortran ordered (i fastest), exactly amrex::Array4 / FArrayBox layout;
 *   - memory is BORROWED: no entry point allocates persistent memory or frees anything
 *     (WarpX callees never own MultiFab / ParticleTile storage);
 *   - all launches are asynchronous on `stream` (a cudaStream_t passed as void*), like
 *     kernels on amrex::Gpu::gpuStream(); the caller synchronises (PhysicalParticleContainer.cpp:2076);
 *   - errors: WarpX aborts (WARPX_ABORT_WITH_MESSAGE -> amrex::Abort).  Default here is the same:
 *     print to stderr and abort().  Tests switch to return codes with pic_set_error_mode().
 */
#ifndef PIC_B200_H_
#define PIC_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------
 * Data descriptors
 * ---------------------------------------------------------------------------------------- */

/* One component of a MultiFab on one box == amrex::FArrayBox / Array4<Real>
 * (Source/FieldSolver/FiniteDifferenceSolver/EvolveB.cpp:143-148).
 * p points at element (lo[0],lo[1],lo[2]); element (i,j,k) lives at
 * p[(i-lo[0]) + (j-lo[1])*nx + (k-lo[2])*nx*ny], nx = hi[0]-lo[0]+1, ny = hi[1]-lo[1]+1. */
typedef struct pic_fab {
    double* p;
    int lo[3];     /* smallest allocated index  (= valid lo - ng)            */
    int hi[3];     /* largest  allocated index, inclusive (= valid hi + ng)  */
    int ng[3];     /* guard cells per side (MultiFab::nGrowVect)             */
    int stag[3];   /* amrex::IndexType: 1 = NODE, 0 = CELL                   */
} pic_fab;

/* Particle struct-of-arrays of one tile == ParticleContainerPureSoA<PIdx::nattribs,0>
 * with PIdx {x,y,z,w,ux,uy,uz} (Source/Particles/NamedComponentParticleContainer.H:23-40)
 * + the 64-bit idcpu.  u = gamma*v in m/s; w = physical particles per macro-particle. */
typedef struct pic_soa {
    double* x; double* y; double* z; double* w;
    double* ux; double* uy; double* uz;
    uint64_t* idcpu;
    long np;
} pic_soa;

/* Stencil coefficients == FiniteDifferenceSolver::m_stencil_coefs_{x,y,z}
 * (FiniteDifferenceSolver.cpp:30-103).  Yee: c[0] = 1/dx (CartesianYeeAlgorithm.H:37-42).
 * CKC: {1/d, alpha, beta1, beta2, gamma/d} (CartesianCKCAlgorithm.H:84-101).
 * PIC_SOLVER_NONE: algo.maxwell_solver = none (the step driver only gathers and pushes, WarpXEvolve.cpp:176-182). */
enum { PIC_SOLVER_YEE = 0, PIC_SOLVER_CKC = 1, PIC_SOLVER_NONE = 2 };
typedef struct pic_stencil {
    int algo;
    double cx[5]; double cy[5]; double cz[5];
} pic_stencil;

/* Particle pusher selection == ParticlePusherAlgo (Utils/WarpXAlgorithmSelection.H). */
enum { PIC_PUSHER_BORIS = 0, PIC_PUSHER_VAY = 1, PIC_PUSHER_HC = 2 };

/* Cell bins of a cell-sorted particle tile == amrex::DenseBins as built by
 * SortParticlesForDeposition / the shared-memory deposition path
 * (Source/Particles/WarpXParticleContainer.cpp:493-540, MultiParticleContainer.cpp:615-624;
 * the reference's bins are likewise grouped by a tile of WarpX::shared_tilesize cells,
 * Source/WarpX.cpp:126,133).
 * Cells of the rank's valid box [box_lo, box_hi] are numbered SUPERCELL-MAJOR: the box is cut
 * into supercells of tile[0] x tile[1] x tile[2] cells (partial supercells at the high ends are
 * padded), supercell t = ti + ntx*(tj + nty*tk), and inside a supercell
 * l = li + tile[0]*(lj + tile[1]*lk); bin id = t*tile[0]*tile[1]*tile[2] + l.
 * Particles of bin b are [cell_start[b], cell_start[b+1]).  All particles of one supercell are
 * therefore contiguous.  pic_bins_count() gives the (padded) number of bins.
 * Optional everywhere (NULL = particle order unknown -> order-agnostic kernels). */
typedef struct pic_bins {
    const int* cell_start;  /* pic_bins_count()+1 entries, device              */
    int box_lo[3];          /* first cell of the box                           */
    int box_hi[3];          /* last cell of the box, inclusive                 */
    int tile[3];            /* supercell size in cells (8,8,8 is what the kernels are tuned for) */
    long np_binned;         /* particles [0, np_binned) are covered by cell_start; particles appended
                               later (neighbour migration) are processed order-agnostically     */
} pic_bins;

/* Optional by-product of the position push: the indices of the particles whose NEW position lies
 * outside [lo, hi] in some direction -- exactly the particles amrex enforcePeriodic will shift at
 * the end of the step (set lo/hi to -/+inf in non-periodic directions).  Lets
 * pic_particles_wrap_listed touch only those particles instead of re-reading every position.
 * count is a device int the caller zeroes before the push; when more than `capacity` particles
 * are found, count still holds the true number and the consumer falls back to a full sweep. */
typedef struct pic_escape_list {
    int* idx;               /* capacity entries, device                        */
    int* count;             /* one int, device                                 */
    int capacity;
    double lo[3], hi[3];
} pic_escape_list;

/* Domain description for the periodic / neighbour guard-cell operations
 * (amrex::Geometry + Periodicity). */
typedef struct pic_geom {
    int n_cell[3];          /* global number of cells                          */
    double prob_lo[3];
    double prob_hi[3];
    int periodic[3];
} pic_geom;

/* Boundary types per domain face == WarpX::field_boundary_lo/hi (FieldBoundaryType) and
 * particle_boundary_lo/hi (ParticleBoundaryType), Source/Utils/WarpXAlgorithmSelection.H;
 * parsed from boundary.field_lo/hi, boundary.particle_lo/hi (Source/Utils/WarpXUtil.cpp:470-540).
 * A periodic field face implies a periodic particle face.  Supported subset: periodic / PEC fields,
 * periodic / absorbing / reflecting particles. */
enum { PIC_FIELD_PERIODIC = 0, PIC_FIELD_PEC = 1 };
enum { PIC_PARTICLE_PERIODIC = 0, PIC_PARTICLE_ABSORBING = 1, PIC_PARTICLE_REFLECTING = 2 };
typedef struct pic_boundaries {
    int field_lo[3], field_hi[3];
    int particle_lo[3], particle_hi[3];
} pic_boundaries;

/* Laser antenna with the Gaussian profile == LaserParticleContainer (Source/Particles/
 * LaserParticleContainer.cpp:84-270: position, direction, polarization, wavelength, e_max) +
 * GaussianLaserProfile (Source/Laser/LaserProfilesImpl/LaserProfileGaussian.cpp:32-86:
 * profile_waist, profile_duration, profile_t_peak, profile_focal_distance, phi0; the
 * spatio-temporal couplings zeta, beta, phi2 are 0).  All parameters are lab-frame values, as in the
 * deck.  gamma_boost > 1 (warpx.gamma_boost, with beta_boost = sqrt(1 - 1/gamma_boost^2),
 * Source/Utils/WarpXUtil.cpp:114-121): the simulation frame moves along nvec (the reference asserts
 * boost_direction == nvec, LaserParticleContainer.cpp:183-190); the library moves the antenna plane to
 * Z0/gamma_boost (:191-197), evaluates the profile at the lab time of the plane (:573-579), divides the
 * mobility by gamma_boost (:775) and lets the antenna drift with -beta_boost c nvec (:908-915).
 * gamma_boost <= 1 (0 included) = lab frame. */
typedef struct pic_laser_antenna {
    double position[3];     /* a point of the antenna plane                    */
    double nvec[3];         /* plane normal = propagation direction (normalised by the library) */
    double p_X[3];          /* main polarisation vector (normalised by the library)             */
    double wavelength, e_max;
    double waist, duration, t_peak, focal_distance, phi0;
    double gamma_boost, beta_boost;
} pic_laser_antenna;

/* Plasma injector of one species: NUniformPerCell positions (InjectorPositionRegular,
 * Source/Initialization/InjectorPosition.H:67-108), constant density, momentum at rest
 * (<species>.injection_style / num_particles_per_cell_each_dim / xmin..zmax / profile = constant /
 * momentum_distribution_type = at_rest / do_continuous_injection of Source/Initialization/PlasmaInjector.cpp).
 * gamma_boost > 1: frame boosted along +z; bound_lo/hi and density stay lab-frame values, the library
 * tests the bounds at z_lab = gamma (z + beta c t), scales the density by gamma and gives every particle
 * uz = -gamma beta c (PhysicalParticleContainer.cpp:138-148,1209-1247). */
typedef struct pic_plasma_injector {
    int ppc[3];
    double bound_lo[3], bound_hi[3];   /* xmin,ymin,zmin / xmax,ymax,zmax (+-inf when unset) */
    double density;
    int do_continuous_injection;
    double gamma_boost, beta_boost;
} pic_plasma_injector;

/* Gaussian particle beam of one species (<species>.injection_style = "gaussian_beam",
 * Source/Initialization/PlasmaInjector.cpp:222-246 + momentum_distribution_type = gaussian / constant / at_rest,
 * InjectorMomentum.H:60-90).  Every value is a lab-frame value, as in the deck.  rms = x_rms, y_rms, z_rms;
 * cut = x_cut.. in units of rms (unset: DBL_MAX, the reference's default, PlasmaInjector.H:108-110);
 * bound_lo/hi = xmin..zmax (+-inf when unset); u_m / u_th = bulk momentum and spread in units of c
 * (u_th = 0: constant / at_rest); do_focusing with focal_distance = <species>.focal_distance.
 * Random numbers: a counter-based Philox4x64-10 keyed by seed (not AMReX's stream), see
 * pic_add_gaussian_beam.  gamma_boost > 1: frame boosted along +z (MapParticletoBoostedFrame, forward
 * propagation, transverse positions unchanged); gamma_boost <= 1 = lab frame. */
typedef struct pic_gaussian_beam {
    double x_m[3], rms[3], cut[3];
    double bound_lo[3], bound_hi[3];
    double q_tot;
    long npart;
    int do_symmetrize, symmetrization_order;    /* order 4 or 8 */
    int do_focusing;
    double focal_distance;
    double u_m[3], u_th[3];
    uint64_t seed;
    double gamma_boost, beta_boost;
} pic_gaussian_beam;

enum { PIC_ERR_ABORT = 0, PIC_ERR_RETURN = 1 };
void pic_set_error_mode(int mode);
const char* pic_last_error(void);
/* Kernel-variant defaults from the environment: PIC_FDTD_MODE, PIC_DEPOSIT_MODE, PIC_GATHER_MODE (values as the
 * pic_set_*_mode calls).  The Python loader calls it once after dlopen. */
void pic_apply_env_defaults(void);
const char* pic_version(void);

/* ------------------------------------------------------------------------------------------
 * Maxwell solver  (replaces FiniteDifferenceSolver::EvolveB / EvolveE)
 * ---------------------------------------------------------------------------------------- */

/* FiniteDifferenceSolver::EvolveBCartesian<T_Algo> (EvolveB.cpp:122-186), called from
 * WarpX::EvolveB (WarpXPushFieldsEM.cpp:904-907).  B[c] += dt * curl-part over the valid
 * points of each staggered component.  B = {Bx,By,Bz}, E = {Ex,Ey,Ez}. */
int pic_evolve_b(const pic_fab B[3], const pic_fab E[3], const pic_stencil* st, double dt,
                 void* stream);

/* FiniteDifferenceSolver::EvolveECartesian<T_Algo> (EvolveE.cpp:120-216), called from
 * WarpX::EvolveE (WarpXPushFieldsEM.cpp:958-962).  E += c^2 dt (curl B - mu0 J). */
int pic_evolve_e(const pic_fab E[3], const pic_fab B[3], const pic_fab J[3],
                 const pic_stencil* st, double dt, void* stream);
/* How the Yee kernels read their source field, a bit mask: bit 0 (default on) = EvolveB, bit 1 = EvolveE through
 * bulk-asynchronous copies (cp.async.bulk, completion on an mbarrier) that stage the rows a CTA needs into a
 * shared-memory ring, plane after plane (csrc/fdtd_bulk.cu); bit clear = plain read-only loads (csrc/fdtd.cu).
 * CKC's EvolveB and arrays whose base is not 16-byte aligned always take the plain kernels.  Same arithmetic either way. */
void pic_set_fdtd_mode(int mode);
long pic_fdtd_bulk_launches(void);   /* launches of the bulk-staged kernels so far (tests: the path really ran) */

/* ------------------------------------------------------------------------------------------
 * Particles  (replaces PhysicalParticleContainer::PushPX / PushP and
 *             WarpXParticleContainer::DepositCurrent)
 * ---------------------------------------------------------------------------------------- */

/* PhysicalParticleContainer::PushPX (PhysicalParticleContainer.cpp:2549-2786): per particle
 * doGatherShapeN (Gather/FieldGather.H:36-424), doParticleMomentumPush (Pusher/PushSelector.H:38-102),
 * UpdatePosition (Pusher/UpdatePosition.H:24-45).  xyzmin/lo describe the guard-grown tile box
 * (:2575-2601).  push_position = 0 gives PushP (:2368-2513; momentum only).
 * nox = 1..4 (algo.particle_shape); the supercell kernel behind `bins` serves orders 1..3, order 4
 * always takes the order-agnostic kernel.
 * bins may be NULL; escaped may be NULL (it is only written when push_position != 0). */
int pic_gather_push(const pic_soa* p, long offset, long np,
                    const pic_fab E[3], const pic_fab B[3],
                    const double dinv[3], const double xyzmin[3], const int lo[3],
                    double q, double m, double dt,
                    int nox, int galerkin, int pusher, int push_position,
                    const pic_bins* bins, const pic_escape_list* escaped, void* stream);

/* PushPX that also carries out a pending cell sort: particle `pos` of the binned order is read from
 * in[src[pos]] (src, cell_start of `bins` from pic_sort_index_by_cell on `in`; bins->np_binned = in->np),
 * pushed, and written to out[pos] together with its weight and id; `in` is left as it was.  `escaped` lists
 * indices of `out`.  Same arithmetic per particle as pic_sort_apply_permutation followed by pic_gather_push on
 * `out`.  Served by the default supercell kernel only: orders 1..3 and PIC_GATHER_TILE, anything else is an error
 * (apply the permutation, then call pic_gather_push). */
int pic_gather_push_permuted(const pic_soa* in, const pic_soa* out, const int* src,
                             const pic_fab E[3], const pic_fab B[3],
                             const double dinv[3], const double xyzmin[3], const int lo[3],
                             double q, double m, double dt, int nox, int galerkin, int pusher,
                             const pic_bins* bins, const pic_escape_list* escaped, void* stream);

/* Which kernel the cell-sorted (bins != NULL) gather uses.  PIC_GATHER_TILE (default): one particle per lane.
 * PIC_GATHER_PAIRS: a lane takes two particles of one cell and feeds both from one set of shared-memory loads
 * (half the loads per particle); applies where the stencils of all particles of a cell coincide -- order 3 or 1
 * with the Galerkin gather on the Yee grid -- other configurations keep the default kernel.  Same results
 * (each particle's own accumulation order is unchanged).  PIC_GATHER_PAIRS_WIDE: the same kernel without the
 * 128-register cap (254 registers, one CTA per SM).  Experiments until measured. */
enum { PIC_GATHER_TILE = 0, PIC_GATHER_PAIRS = 1, PIC_GATHER_PAIRS_WIDE = 2,
       PIC_GATHER_PAIRS_192 = 3 /* the pair kernel with 192 threads per CTA: 168 registers, no spills, 12 warps per SM */ };
void pic_set_gather_mode(int mode);

/* WarpXParticleContainer::DepositCurrent (WarpXParticleContainer.cpp:352-827) ->
 * doEsirkepovDepositionShapeN<nox> (Deposition/CurrentDeposition.H:642-907).
 * J = {jx,jy,jz} is ADDED to (the caller zeroes J, MultiParticleContainer.cpp:467-478).
 * xyzmin/lo describe the ng_J-grown tile box (WarpXParticleContainer.cpp:424-479).
 * bins may be NULL (-> order-agnostic kernel with global fp64 atomics, the reference's
 * GPU strategy); with bins the shared-memory tile kernel is used. */
int pic_deposit_esirkepov(const pic_soa* p, long offset, long np,
                          const pic_fab J[3],
                          const double dinv[3], const double xyzmin[3], const int lo[3],
                          double q, double dt, double relative_time, int nox,
                          const pic_bins* bins, void* stream);

/* Which kernel serves pic_deposit_esirkepov when bins are given (tuning / A-B measurements):
 * PIC_DEPOSIT_RUNS (default): warp-segmented register reduction + fp64 L2 reductions;
 * PIC_DEPOSIT_TILE: the same reduction staged through a shared-memory J block per supercell;
 * PIC_DEPOSIT_RUNS2: PIC_DEPOSIT_RUNS with two stencil lines per lane (fewer shared-memory reads per
 *   particle; orders 1 and 3 -- order 2 falls back to PIC_DEPOSIT_RUNS);
 * PIC_DEPOSIT_RUNS_SLOTRED / PIC_DEPOSIT_RUNS2_SLOTRED: the particle slots of a warp pass send their own
 *   partial sums to L2 instead of being summed by shuffles first.
 * PIC_DEPOSIT_RUNS4 / PIC_DEPOSIT_RUNS4_SLOTRED: four lines per lane (order 3 only; 168 registers).
 * PIC_DEPOSIT_RUNS_SLAB: PIC_DEPOSIT_RUNS retiring into a per-warp shared-memory J slab (lone strays too), added to
 *   J with coalesced L2 reductions at a rebase and at the end of the warp's particles (orders 1..3).
 * Modes 2..6 are experiments until measured; all pass the same parity tests.
 * Analogous to WarpX's runtime switch warpx.do_shared_mem_current_deposition
 * (Source/WarpX.cpp:126, Docs/source/usage/parameters.rst:2608-2623). */
enum { PIC_DEPOSIT_RUNS = 0, PIC_DEPOSIT_TILE = 1, PIC_DEPOSIT_RUNS2 = 2, PIC_DEPOSIT_RUNS_SLOTRED = 3,
       PIC_DEPOSIT_RUNS2_SLOTRED = 4, PIC_DEPOSIT_RUNS4 = 5, PIC_DEPOSIT_RUNS4_SLOTRED = 6, PIC_DEPOSIT_CELLS = 7,
       PIC_DEPOSIT_CELLS2 = 8, PIC_DEPOSIT_CELLS2_WIDE = 9 /* lane per cell with two producer warps (3 / 2 CTAs per SM) */,
       PIC_DEPOSIT_CELLS3 = 10, PIC_DEPOSIT_CELLS3_WIDE = 11 /* the same, producers and consumers decoupled by mbarriers */,
       PIC_DEPOSIT_RUNS_SLAB = 12 };
void pic_set_deposit_mode(int mode);

/* ------------------------------------------------------------------------------------------
 * Guard cells  (replaces ablastr::utils::communication::FillBoundary / SumBoundary)
 * ---------------------------------------------------------------------------------------- */

/* FillBoundary along one dimension when the box spans the whole periodic domain in that
 * dimension (self-neighbour): guards <- periodic image of valid points
 * (WarpXComm.cpp:699-827 -> Communication.cpp:71-115).  Other dimensions are covered over
 * their full allocated extent so that sweeping dim = 0,1,2 fills edges and corners. */
int pic_fill_boundary_local(const pic_fab* f, int dim, int ng, const pic_geom* g, void* stream);

/* SumBoundary along one dimension for a self-neighbour box: valid points accumulate the
 * periodic images of guard points (and the duplicate nodal point)
 * (WarpXComm.cpp:1386-1424 -> WarpXSumGuardCells.cpp:17-24 -> Communication.cpp:148-175). */
int pic_sum_boundary_local(const pic_fab* f, int dim, int src_ng, const pic_geom* g, void* stream);
/* pic_fill_boundary_local (mode 0) / pic_sum_boundary_local (mode 1, ng = src_ng) of up to 8 components with one
 * launch (the step driver's form: one launch per axis sweep of an exchange). */
int pic_boundary_local_multi(const pic_fab* fabs, int nfab, int dim, int ng, int mode, const pic_geom* g, void* stream);

/* Bilinear (binomial) filter of one component: dst(i,j,k) = sum of the (1,2,1)/4 kernel applied
 * npass[d] times along each direction d, over every allocated point of dst (valid + guards),
 * src zero-padded outside its allocation.  src and dst must not alias; the caller copies dst
 * back over src as WarpX::ApplyFilterJ does.
 * Replaces BilinearFilter::ComputeStencils + Filter::ApplyStencil (Source/Filter/BilinearFilter.cpp:
 * 64-88, Source/Filter/Filter.cpp:37-133) as called from WarpXComm.cpp:1357-1374. */
int pic_apply_filter(const pic_fab* src, const pic_fab* dst, const int npass[3], void* stream);
/* The same for up to three components in ONE launch (Jx, Jy, Jz of WarpX::ApplyFilterJ): for npass = (1,1,1) a
 * streaming kernel that walks every column along z with the last three xy-filtered planes in registers (same nesting of
 * the sums, same bits as pic_apply_filter).  The step driver deposits into its own scratch copies of J and filters
 * from there INTO the caller's J arrays, so there is no copy back. */
int pic_apply_filter_multi(const pic_fab* src, const pic_fab* dst, int nfab, const int npass[3], void* stream);

/* Godfrey's NCI corrector (particles.use_fdtd_nci_corr; SURVEY.md section 8f rank 3).
 * _table_index / _stencil: NCIGodfreyFilter::ComputeStencils (Source/Filter/NCIGodfreyFilter.cpp:49-139) --
 *   index = clamp(int(tab_length * cdtodz), 0, tab_length - 2); the four coefficients are interpolated between
 *   line_lo = table[index] and line_hi = table[index + 1] of the caller's copy of the reference's tables
 *   (Source/Utils/NCIGodfreyTables.H: galerkin / momentum x Ex_Ey_Bz / Bx_By_Ez, tab_length = 101), then combined
 *   into stencil_z[5] with coefficient 0 halved, i.e. the contents of Filter::m_stencil_2.  A WarpX build skips
 *   these two and passes the m_stencil_2 it already holds.
 * pic_apply_nci_filter: PhysicalParticleContainer::applyNCIFilter (Source/Particles/PhysicalParticleContainer.cpp:
 *   2097-2169) for one component: dst = the 5-point z filter of src over the tile box [tile_lo, tile_hi] (cells)
 *   grown by `grow` = the particle shape order and converted to the component's index type; src zero-padded
 *   outside its allocation (Filter::DoFilter, Source/Filter/Filter.cpp:92-133).  Ex, Ey, Bz take the Ex_Ey_Bz
 *   stencil, Bx, By, Ez the other (:2132-2163).  The gather then reads dst instead of src. */
int pic_nci_godfrey_table_index(double cdtodz, int tab_length);
void pic_nci_godfrey_stencil(const double line_lo[4], const double line_hi[4], int index, int tab_length,
                             double cdtodz, double stencil_z[5]);
int pic_apply_nci_filter(const pic_fab* src, const pic_fab* dst, const double stencil_z[5], const int tile_lo[3],
                         const int tile_hi[3], int grow, void* stream);

/* Neighbour (multi-GPU) versions: pack the slab that the neighbour on `side` (0 = low,
 * 1 = high) of dimension `dim` needs, and unpack what it sent.  mode 0 = copy (FillBoundary),
 * mode 1 = sum (SumBoundary).  pic_halo_slab_count returns the number of doubles. */
long pic_halo_slab_count(const pic_fab* f, int dim, int ng, int mode);
int pic_halo_pack(const pic_fab* f, int dim, int side, int ng, int mode, double* buf, void* stream);
int pic_halo_unpack(const pic_fab* f, int dim, int side, int ng, int mode, const double* buf,
                    void* stream);
/* All components of one exchange (e.g. Ex Ey Ez Bx By Bz) and both sides in ONE launch: buf_lo /
 * buf_hi hold the slabs for the low / high neighbour concatenated in component order (nfab <= 8).
 * The multi calls also take mode 2 = SumBoundary AND the FillBoundary that follows it (WarpXSumGuardCells.H:
 * SumBoundary then FillBoundary of J / rho) as ONE exchange between two ranks along a periodic axis: each side packs
 * its whole overlap zone (ng valid layers, the shared node, ng guards) and adds what it receives; needs
 * 2 ng + nodal <= box width. */
int pic_halo_pack_multi(const pic_fab* fabs, int nfab, int dim, int ng, int mode, double* buf_lo,
                        double* buf_hi, void* stream);
int pic_halo_unpack_multi(const pic_fab* fabs, int nfab, int dim, int ng, int mode, const double* buf_lo,
                          const double* buf_hi, void* stream);

/* ------------------------------------------------------------------------------------------
 * Particle housekeeping  (replaces AMReX Redistribute periodic wrap and
 *                         SortParticlesByBin / SortParticlesForDeposition)
 * ---------------------------------------------------------------------------------------- */

/* amrex enforcePeriodic as applied by ParticleContainer::Redistribute
 * (WarpXEvolve.cpp:550-559 -> MultiParticleContainer.cpp:650-656; AMReX 24.10 @62c2a81
 * AMReX_ParticleUtil.H, un-vendored dependency). */
int pic_particles_wrap_periodic(const pic_soa* p, const pic_geom* g, void* stream);

/* Same result, but only the particles listed by the preceding pic_gather_push are visited
 * (full sweep if the list overflowed).  Valid when every particle was inside the domain before
 * that push, i.e. when this function (or pic_particles_wrap_periodic) ended the previous step. */
int pic_particles_wrap_listed(const pic_soa* p, const pic_geom* g, const pic_escape_list* escaped, void* stream);

/* Neighbour migration, step 1 (replaces the locate/partition phase of AMReX
 * ParticleContainer::Redistribute, WarpXEvolve.cpp:550-559): indices of the particles whose cell
 * along `dim` lies below cell_lo (-> idx_lo) or above cell_hi (-> idx_hi) after the periodic wrap.
 * With `both_up` = 1 (two ranks along a periodic dim: both neighbours are the same rank) everything
 * goes to idx_hi; `both_up` = 2 marks a NON-periodic dim (no wrap-around ownership: below cell_lo -> low
 * neighbour, above cell_hi -> high neighbour).  counts[0], counts[1] (device ints, zeroed here) receive the list lengths; lists hold at
 * most `capacity` entries each (counts keep counting: the caller checks for overflow). */
int pic_particles_classify(const pic_soa* p, const pic_geom* g, int dim, int cell_lo, int cell_hi,
                           int both_up, int* counts, int* idx_lo, int* idx_hi, int capacity,
                           const int* np_dev /* NULL: p->np; else the count lives on the device and
                                                p->np is only an upper bound for the launch */,
                           void* stream);

/* The same classification over a CANDIDATE list instead of every particle: `candidates` is the list the preceding
 * pic_gather_push wrote with lo/hi set to the rank's brick (every particle that left the brick is in it; the periodic
 * wrap has been applied since).  Entries that point behind the current particle count are dropped (set to -1: a tail
 * particle that an earlier sweep moved into a hole is reached through the hole's entry).  When the list overflowed
 * (count > capacity) every particle is visited, as pic_particles_classify does.  After pic_migrate_unpack,
 * pic_migrate_note_appended adds the particles that sweep appended behind the old count (`work` = the unpack's
 * workspace), so that the next axis sweep forwards arrivals that have to travel on (edges, corners).  Arrivals that
 * filled holes need no entry: the holes are candidates already. */
int pic_particles_classify_listed(const pic_soa* p, const pic_geom* g, int dim, int cell_lo, int cell_hi,
                                  int both_up, int* counts, int* idx_lo, int* idx_hi, int capacity,
                                  const int* np_dev, const pic_escape_list* candidates, void* stream);
int pic_migrate_note_appended(const void* work, const pic_escape_list* candidates, void* stream);
/* how many axis sweeps of this process classified from the candidate list (tests: the list path really ran) */
long pic_engine_listed_sweeps(void);
/* how many J exchanges of this process ran as the fused sum + refresh (halo mode 2) */
long pic_engine_fused_sum_exchanges(void);

/* Neighbour migration, steps 2 and 3 (pack / unpack phases of Redistribute).  A message is
 * pic_migrate_message_doubles(cap) doubles: header (true particle count) + 8 rows of cap doubles
 * (x y z w ux uy uz id) -- a FIXED size, so the send/recv pair needs no count exchange.
 * pic_migrate_unpack drops the arrivals (msg_lo from the low, msg_hi from the high neighbour) into
 * the holes left by the particles listed in idx_lo/idx_hi, appends the rest, or moves tail
 * particles into the remaining holes; work[0] receives the new particle count, work[1] a status
 * (bit 0: a list or message overflowed `cap`; bit 1: `capacity` exceeded; bits are OR-ed into
 * work[1], the caller clears it).  The count before migration is p->np, or *np_dev when given
 * (np_dev may point at work[0] of the previous sweep: the sweeps of a step chain on the device and
 * the host reads the count once). */
long pic_migrate_message_doubles(int cap);
long pic_migrate_workspace_bytes(int cap);
int pic_migrate_pack(const pic_soa* p, const int* idx, const int* count, int cap, double* msg, void* stream);
int pic_migrate_unpack(const pic_soa* p, const int* counts, const int* idx_lo, const int* idx_hi,
                       const double* msg_lo, const double* msg_hi, int cap, long capacity,
                       void* work, const int* np_dev /* NULL: p->np */, void* stream);

/* Counting sort of the particles by cell over the valid box [box_lo,box_hi]
 * (WarpX: mypc->SortParticlesByBin, WarpXEvolve.cpp:575-580).  `in` is permuted into `out`;
 * bins->cell_start (pic_bins_count()+1 ints) receives the bins.  work must hold
 * pic_sort_workspace_bytes(). */
long pic_bins_count(const int box_lo[3], const int box_hi[3], const int tile[3]);
long pic_sort_workspace_bytes(long np, long nbins);
int pic_sort_particles_by_cell(const pic_soa* in, const pic_soa* out, const pic_geom* g,
                               const pic_bins* bins /* cell_start is written */,
                               void* work, void* stream);
/* The same sort in two halves.  pic_sort_index_by_cell moves nothing: it writes cell_start and the permutation
 * (*src points into `work`: particle src[pos] of `in` belongs at position pos).  pic_sort_apply_permutation writes
 * out[pos] = in[src[pos]] for the seven arrays and the id; pic_gather_push_permuted does that move inside the push. */
int pic_sort_index_by_cell(const pic_soa* in, const pic_geom* g, const pic_bins* bins /* cell_start is written */,
                           void* work, const int** src, void* stream);
int pic_sort_apply_permutation(const pic_soa* in, const pic_soa* out, const int* src, void* stream);
/* np ints of the sort workspace that only pic_sort_index_by_cell writes: free for other uses until the next sort
 * (np = the particle count of the last pic_sort_index_by_cell on `work`). */
int* pic_sort_scratch(void* work, long np);

/* ------------------------------------------------------------------------------------------
 * Non-periodic domains: PEC walls, moving window, laser antenna, continuous injection, particle
 * boundaries (SURVEY.md 8f rank 3 -- what BASELINE.json's config 4, the laser-wakefield deck, adds
 * to the periodic step).  Boxes must span the domain along a non-periodic direction.
 * ---------------------------------------------------------------------------------------- */

/* PEC::ApplyPECtoEfield (is_E = 1) / ApplyPECtoBfield (is_E = 0), Source/BoundaryConditions/WarpX_PEC.cpp:
 * 456-612, called at the end of WarpX::EvolveE / EvolveB (Source/FieldSolver/WarpXPushFieldsEM.cpp:926,990
 * -> Source/BoundaryConditions/WarpXFieldBoundaries.cpp:51-159).  Acts on the valid points of each
 * component grown by ng_fieldgather: tangential E / normal B vanish on the wall and are odd across
 * it, the other components are even. */
int pic_apply_pec_field(const pic_fab F[3], int is_E, const pic_geom* g, const pic_boundaries* b,
                        const int ng_fieldgather[3], void* stream);

/* PEC::ApplyReflectiveBoundarytoJfield (WarpX_PEC.cpp:702-880), called at the end of
 * WarpX::SyncCurrentAndRho (Source/Evolve/WarpXEvolve.cpp:629-652): current deposited beyond a PEC /
 * reflecting face is folded back as an image current, the guards receive the image of the interior. */
int pic_apply_pec_current(const pic_fab J[3], const pic_geom* g, const pic_boundaries* b, void* stream);

/* WarpX::shiftMF (Source/Utils/WarpXMovingWindow.cpp:478-604) for one component: the data move by
 * num_shift cells against `dir`, `external_field` enters from the face the window moves into.
 * tmp: scratch with as many doubles as the fab (borrowed). */
int pic_shift_fab(const pic_fab* f, double* tmp, const pic_geom* g, int num_shift, int dir,
                  double external_field, void* stream);

/* Laser antenna (LaserParticleContainer, Source/Particles/LaserParticleContainer.cpp).
 * _info: out = {S_X, S_Y, mobility, weight} (ComputeSpacing :727-761, ComputeWeightMobility :763-781).
 * _particles: InitData (:369-560) -- HOST arrays x y z w receive one +w/-w pair per antenna cell inside
 *   the box (the reference builds host vectors and hands them to AddNParticles); returns the particle
 *   count (call with x = NULL to size), -1 when `capacity` is too small.  Momenta start at 0.
 * _push: one step at time t = start of the step (Evolve :614-626): plane coordinates, Gaussian
 *   amplitude (LaserProfileGaussian.cpp:100-162), u and x update (:860-951).  The antenna then
 *   deposits through pic_deposit_esirkepov with q = 1 (:88). */
int pic_laser_antenna_info(const pic_laser_antenna* prm, const double dx[3], double out[4]);
long pic_laser_antenna_particles(const pic_laser_antenna* prm, const double dx[3], const double box_lo[3],
                                 const double box_hi[3], double* x, double* y, double* z, double* w,
                                 long capacity);
int pic_laser_antenna_push(const pic_laser_antenna* prm, const double dx[3], const pic_soa* p, double t,
                           double dt, void* stream);

/* PhysicalParticleContainer::AddPlasma (Source/Particles/PhysicalParticleContainer.cpp:924-1333) for
 * the injector described by pic_plasma_injector, restricted to the RealBox [part_lo, part_hi] (the
 * whole domain at start-up, the slab uncovered by the moving window for ContinuousInjection, :2518-2527).
 * Particles are appended on the device after p->np, in the order the reference creates them, with
 * ids first_id, first_id+1, ...  cell_size = Geometry::CellSize() (NULL: (prob_hi - prob_lo) / n_cell;
 * a moving window translates the domain but keeps the cell size it started with).  box_lo/box_hi =
 * the cells of this rank's box (the tile whose RealBox must contain a particle, :1141-1156; NULL = the
 * whole domain).  t = WarpX::gett_new(0), used only in a boosted frame (:956).  p = NULL only counts.
 * Returns how many were (would be) added, -1 on error. */
long pic_add_plasma(const pic_plasma_injector* inj, const pic_geom* g, const double cell_size[3],
                    const int box_lo[3], const int box_hi[3], const double part_lo[3], const double part_hi[3],
                    const pic_soa* p, long capacity, uint64_t first_id, double t, void* stream);

/* PhysicalParticleContainer::AddGaussianBeam (Source/Particles/PhysicalParticleContainer.cpp:503-677) +
 * CheckAndAddParticle (:830-853) + MapParticletoBoostedFrame (:456-500) + the Redistribute of InitData (:450-454)
 * for the beam described by b.  Draw i (0 <= i < npart, npart /= symmetrization_order with do_symmetrize) takes
 * the Philox4x64-10 blocks 2i and 2i+1 keyed by seed (pic_philox4x64) and turns them into 8 normals
 * (pic_gaussian_beam_normals); the first six are x, y, z, ux, uy, uz.  A draw inside the bounds and the cuts
 * gives 1, 4 or 8 particles (the images of do_symmetrize, in the reference's order) of weight
 * q_tot / (npart charge) / images; in a boosted frame they are mapped to it at t0 = WarpX::gett_new(0).
 * Redistribute: positions are wrapped along periodic axes of g (oracle semantics, amrex::enforcePeriodic)
 * and particles outside a non-periodic face (x < prob_lo or x > prob_hi) are dropped.  The particles whose
 * position then lies in [own_lo, own_hi) (+-inf at the domain's faces) are appended on the device after
 * p->np, in creation order; the id of a particle is its index in the creation list of a single box
 * (AddNParticles, WarpXParticleContainer.cpp:163-240), whatever the decomposition.  Deterministic: a count
 * pass, a scan, a write pass, no atomics.  p = NULL only counts.  Synchronises `stream` (the count is read
 * back); borrows device scratch of 16 bytes per 64 draws for the duration of the call.  Every precondition
 * (npart >= 1, rms >= 0, symmetrization order 4 or 8, 0 < beta_boost < 1 when boosted, a non-zero bulk
 * momentum when focusing, capacity) is checked before anything is written: a failed call leaves p as it was.
 * Returns the number of particles appended (or that would be), -1 on error. */
long pic_add_gaussian_beam(const pic_gaussian_beam* b, double charge, const pic_geom* g, const double own_lo[3],
                           const double own_hi[3], const pic_soa* p, long capacity, double t0, void* stream);

/* The random numbers of pic_add_gaussian_beam, for checking the generator.  pic_philox4x64: out[4 j + c] = word c
 * of Philox4x64-10 block first_block + j, keyed by (seed, 0), block j taking the counter (j + 1, 0, 0, 0) -- the
 * stream of numpy.random.Philox(key=seed) after advance(j).  pic_gaussian_beam_normals: out[8 j + c] = normal c
 * of draw first_draw + j (Box-Muller on the 53-bit uniforms of the draw's two blocks, warpx_b200.workloads).
 * out: device memory. */
int pic_philox4x64(uint64_t seed, long first_block, long nblocks, uint64_t* out, void* stream);
int pic_gaussian_beam_normals(uint64_t seed, long first_draw, long ndraws, double* out, void* stream);

/* w_out[ip] = w[ip] for particles inside [own_lo, own_hi), 0 elsewhere.  Used for containers that are
 * replicated on every rank (laser antennas): each rank deposits only what lies in its own box. */
int pic_particles_owned_weights(const pic_soa* p, const double own_lo[3], const double own_hi[3], double* w_out,
                                void* stream);

/* WarpXParticleContainer::ApplyBoundaryConditions (Source/Particles/WarpXParticleContainer.cpp:1574-1638,
 * ParticleBoundaries_K.H:21-75) + the removal AMReX Redistribute performs.  _mark reflects at
 * reflecting faces and lists the particles lost at absorbing faces: work[0] = number lost (device int;
 * work has pic_particles_boundary_workspace_ints(cap) ints).  After reading work[0] the caller
 * calls _compact, which moves tail particles into the holes; the new count is np - n_lost. */
long pic_particles_boundary_workspace_ints(int cap);
int pic_particles_boundary_mark(const pic_soa* p, const pic_geom* g, const pic_boundaries* b, int* work,
                                int cap, void* stream);
int pic_particles_boundary_compact(const pic_soa* p, int* work, int cap, int n_lost, void* stream);

/* ------------------------------------------------------------------------------------------
 * NCCL transport (one process per GPU).  Replaces the MPI layer under
 * ablastr::utils::communication::FillBoundary / SumBoundary (Source/ablastr/utils/Communication.cpp:
 * 71-175) and AMReX ParticleContainer::Redistribute (Source/Evolve/WarpXEvolve.cpp:550-559).
 * NCCL is bound at run time (libnccl.so.2 of the host process).  Bootstrap: rank 0 obtains the
 * 128-byte id, the host broadcasts it out of band (MPI_Bcast in WarpX), every rank creates.
 * ---------------------------------------------------------------------------------------- */
int pic_comm_unique_id(unsigned char out[128]);
void* pic_comm_create(const unsigned char id[128], int nranks, int rank);   /* collective; NULL on failure */
void pic_comm_destroy(void* comm);

/* ------------------------------------------------------------------------------------------
 * C++ step driver (periodic, one brick per rank): WarpX::Evolve / OneStep_nosub expressed through
 * the entry points above (csrc/engine.cu cites the reference lines of every stage).  Memory is
 * borrowed: fabs = Ex Ey Ez Bx By Bz jx jy jz with at least pic_engine_guards() guard cells;
 * bufA/bufB = the two particle buffers of a species (the counting sort permutes one into the
 * other), every SoA array with `capacity` entries.  With pic_engine_set_comm (before the species
 * are added) the guard-cell exchanges and the particle migration run over NCCL on the same stream:
 * the brick grid is nb[0] x nb[1] x nb[2], rank = cx + nb[0]*(cy + nb[1]*cz), box = that brick.
 * ---------------------------------------------------------------------------------------- */
void* pic_engine_create(const pic_geom* geom, const int box_lo[3], const int box_hi[3], int nox,
                        int galerkin, int pusher, int solver, double cfl, double dt /* <=0: cfl*max_dt */,
                        int sort_interval, int use_filter /* warpx.use_filter */,
                        const int filter_npass[3] /* warpx.filter_npass_each_dir; NULL = 1 1 1 */);
void pic_engine_destroy(void* engine);
double pic_engine_dt(void* engine);
void pic_engine_guards(void* engine, int out[12] /* ng_EB[3] ng_J[3] ng_FieldGather[3] ng_FieldSolver[3] */);
/* Per-stage timing of pic_engine_evolve: CUDA events recorded on the launching stream around every stage of
 * the step (the instrumentation a WarpX run gets from its TinyProfiler regions, WarpXEvolve.cpp BL_PROFILE).
 * enable_timing(1) resets the sums; stage_ms fills total milliseconds and call counts of the
 * pic_engine_stage_count() stages named by pic_engine_stage_name(n) (it waits for the recorded events). */
int pic_engine_enable_timing(void* engine, int on);
int pic_engine_stage_count(void);
const char* pic_engine_stage_name(int n);
int pic_engine_stage_ms(void* engine, double ms[], long calls[]);
int pic_engine_set_fields(void* engine, const pic_fab fabs[9]);
int pic_engine_set_comm(void* engine, void* comm, const int nb[3]);
/* The engine's decomposition as a guard-cell context (an engine created only for this needs pic_engine_create,
 * pic_engine_set_boundaries for non-periodic axes and pic_engine_set_comm; with one rank no communicator):
 *   pic_halo_copy  <- ablastr::utils::communication::FillBoundary(mf, ng, ..., period)
 *                     (Source/ablastr/utils/Communication.cpp:71-115; WarpX::FillBoundaryE/B, WarpXComm.cpp:699-827)
 *   pic_halo_add   <- ablastr::utils::communication::SumBoundary(mf, icomp, ncomp, src_ng, dst_ng, ..., period)
 *                     (:148-175; WarpXSumGuardCells.cpp:17-24 passes dst_ng = all guards)
 * for nfab components of this rank's box (all with at least ng / src_ng / dst_ng allocated guard cells): axis sweeps
 * with local copies where the box spans a periodic axis, pack -> ncclSend/ncclRecv -> unpack(+add) elsewhere; guard
 * cells beyond a non-periodic domain face have no image and keep their values (pic_halo_add: their own deposits;
 * along a non-periodic direction src_ng must equal dst_ng, as in every SumBoundary WarpX issues). */
int pic_halo_copy(void* engine, const pic_fab* fabs, int nfab, const int ng[3], void* stream);
int pic_halo_add(void* engine, const pic_fab* fabs, int nfab, const int src_ng[3], const int dst_ng[3], void* stream);
/* Non-periodic runs (one rank; call in this order, before pic_engine_set_fields / add_species):
 *   set_boundaries     boundary.field_lo/hi + boundary.particle_lo/hi (PEC walls, absorbing / reflecting particles);
 *   set_moving_window  warpx.do_moving_window / moving_window_dir / moving_window_v [c] (grows the guard
 *                      cells like guardCellManager::Init, GuardCellManager.cpp:103-115 -- query pic_engine_guards after);
 *   set_boost          warpx.gamma_boost with boost_direction = z: the window and the injection front move with the
 *                      boosted velocities (WarpXMovingWindow.cpp:108-133,156); injectors and antennas added afterwards
 *                      take the engine's gamma_boost / beta_boost; prob_lo/hi are the caller's boosted-frame values
 *                      (ConvertLabParamsToBoost, Source/Utils/WarpXUtil.cpp:180-262);
 *   set_injector       the plasma injector of species isp (its particles must have been created by
 *                      pic_add_plasma over the whole domain, ids 0..np-1); with do_continuous_injection
 *                      the moving window refills the uncovered slab (WarpXMovingWindow.cpp:388-438);
 *   add_laser          a Gaussian antenna whose particles (pic_laser_antenna_particles, momenta 0) the
 *                      caller has uploaded into p (capacity >= p->np).
 * pic_engine_time = t_new[0]; pic_engine_prob_domain = the (moving) problem domain, out = lo[3] hi[3]. */
int pic_engine_set_boundaries(void* engine, const pic_boundaries* b);
int pic_engine_set_moving_window(void* engine, int dir, double v_over_c);
int pic_engine_set_boost(void* engine, double gamma_boost, double beta_boost);
/* particles.use_fdtd_nci_corr: the two z stencils (see pic_nci_godfrey_stencil).  Grows the guard cells of E and B
 * along z (GuardCellManager.cpp:87-90,319-330): call before pic_engine_set_fields, query pic_engine_guards after.
 * The engine owns the six filtered copies the gather of the main push reads (the half pushes of the first and
 * last step, PushP, gather from the unfiltered fields like the reference). */
int pic_engine_set_nci_corrector(void* engine, const double stencil_exeybz[5], const double stencil_bxbyez[5]);
int pic_engine_set_injector(void* engine, int isp, const pic_plasma_injector* inj);
int pic_engine_add_laser(void* engine, const pic_laser_antenna* prm, const pic_soa* p, long capacity);
long pic_engine_laser_np(void* engine, int ilaser);
double pic_engine_time(void* engine);
int pic_engine_set_step(void* engine, long istep, double time);   /* restart: WarpX::InitFromCheckpoint, Diagnostics/WarpXIO.cpp */
void pic_engine_prob_domain(void* engine, double out[6]);
int pic_engine_add_species(void* engine, double q, double m, const pic_soa* bufA, const pic_soa* bufB,
                           long capacity, int* cell_start, const int tile[3], void* sort_work, void* stream);
int pic_engine_species_buffer(void* engine, int isp, long* np);
int pic_engine_evolve(void* engine, int numsteps, int synchronize_last, void* stream);
/* WarpX::HandleParticlesAtBoundaries (Source/Evolve/WarpXEvolve.cpp:533-564) as one call, for a host that keeps its own
 * step loop: periodic wrap, ApplyBoundaryConditions on the non-periodic faces + removal (WarpXParticleContainer.cpp:
 * 1574-1638), RedistributeLocal(1) -- every particle that left this rank's brick goes to the neighbour that owns it
 * (at most one brick per call and direction).  Species / antennas registered with the engine; read the new counts
 * with pic_engine_species_buffer / pic_engine_laser_np.  Cell bins are stale afterwards. */
int pic_engine_redistribute(void* engine, void* stream);

/* ------------------------------------------------------------------------------------------
 * Reduced diagnostics used as parity metrics
 * ---------------------------------------------------------------------------------------- */

/* Sum of squares over the unique (periodicity-aware) valid points of one component ==
 * MultiFab::norm2(0, periodicity)^2 as used by FieldEnergy
 * (Source/Diagnostics/ReducedDiags/FieldEnergy.cpp:120-144).  out: 1 double, device. */
int pic_sum_squares_unique(const pic_fab* f, const pic_geom* g, double* out, void* stream);

/* ParticleEnergy reduced diagnostic of one species (Source/Diagnostics/ReducedDiags/ParticleEnergy.cpp:
 * 86-170 with Algorithms::KineticEnergy, Source/Particles/Algorithms/KineticEnergy.H:31-46):
 * out[0] = sum w m u^2 / (1 + gamma) [J], out[1] = sum w.  out: 2 doubles, device. */
int pic_particle_energy(const pic_soa* p, double mass, double* out, void* stream);

/* The `rho` diagnostic (not on the per-step path of the FDTD loop).
 * pic_deposit_charge: WarpXParticleContainer::DepositCharge (Source/Particles/WarpXParticleContainer.cpp:
 *   890-1216) -> doChargeDepositionShapeN<nox> (Source/Particles/Deposition/ChargeDeposition.H:37-157);
 *   rho is ADDED to; xyzmin / lo describe the tile box grown by rho's guard cells.
 * pic_apply_pec_rho: PEC::ApplyReflectiveBoundarytoRhofield (Source/BoundaryConditions/WarpX_PEC.cpp:624-699),
 *   applied per container before the containers are summed (WarpXParticleContainer.cpp:1277-1283). */
int pic_deposit_charge(const pic_soa* p, long offset, long np, const pic_fab* rho, const double dinv[3],
                       const double xyzmin[3], const int lo[3], double q, int nox, void* stream);
int pic_apply_pec_rho(const pic_fab* rho, const pic_geom* g, const pic_boundaries* b, void* stream);

/* ------------------------------------------------------------------------------------------
 * Cold relativistic fluid species (WarpXFluidContainer, Source/Fluids/WarpXFluidContainer.cpp), 3D Cartesian,
 * periodic domains, lab frame.  A fluid's state U is four all-nodal components {N, NUx, NUy, NUz} on the run's
 * cell box with 2 guard nodes (AllocateLevelMFs :142-164).  Products and sums are rounded as the reference's
 * CPU build rounds them (no multiply-add contraction).
 * pic_fluid_gather_push:     GatherAndPush :967-1238 without external fields or boost: at the valid nodes with
 *   N > 0, E and B interpolated to the node (ablastr::coarsen::sample::Interp), U pushed with Higuera-Cary,
 *   N U written back.  E / B guards must be filled (one guard node).
 * pic_fluid_advect:          AdvectivePush_Muscl :421-893 from U_in into U_out (valid nodes only; two arrays:
 *   one fused kernel reads neighbours while others are written).  The 2 guard nodes of U_in must be filled
 *   (the FillBoundary of ApplyBcFluidsAndComms :413-417).  counters: NULL, or 2 device words that count the
 *   nodes whose edges are zero (N <= 0) and the directions the positivity limiter reset.
 * pic_fluid_deposit_current: DepositCurrent :1276-1398: J += the Yee-point average of q N U / gamma of the
 *   two (or one) nodes it lies between, at the points this box owns (every index in [box_lo, box_hi]: each
 *   point shared by bricks or periodic images is added once; J's SumBoundary completes the copies).
 * pic_fluid_deposit_charge:  DepositCharge :1240-1273: rho += q N at the owned nodes.  rho: nodal, same box. */
int pic_fluid_gather_push(const pic_fab U[4], const pic_fab E[3], const pic_fab B[3], double q, double m,
                          double dt, void* stream);
int pic_fluid_advect(const pic_fab U_in[4], const pic_fab U_out[4], const double dx[3], double dt,
                     unsigned long long* counters, void* stream);
int pic_fluid_deposit_current(const pic_fab U[4], const pic_fab J[3], double q, void* stream);
int pic_fluid_deposit_charge(const pic_fab* N, const pic_fab* rho, double q, void* stream);
/* The C++ driver's fluid species (fluids.species_names): pic_engine_evolve runs WarpXFluidContainer::Evolve
 * (:257-314) for every fluid after the particle species' push and deposit (myfl->Evolve, Source/Evolve/
 * WarpXEvolve.cpp:1171-1178): gather + push, FillBoundary of N and NU, advection into the other state, current deposit.
 * stateA: the initial state on the engine's box (2 guard nodes), stateB: a second state of the same shape; both are
 * borrowed.  One rank, periodic faces, no moving window, no boost, no particle species or antennas; refused calls
 * leave the engine unchanged.  pic_engine_fluid_state: which state of fluid i is current (0 = A, 1 = B), -1 if none. */
int pic_engine_add_fluid_species(void* h, double q, double m, const pic_fab stateA[4], const pic_fab stateB[4]);
int pic_engine_fluid_state(void* h, int i);

/* ------------------------------------------------------------------------------------------
 * Binary Coulomb collisions (collisions.collision_names, <name>.type = pairwisecoulomb), 3D Cartesian.
 * One collision of species 1 with species 2 (the same species when same_species):
 * PairWiseCoulombCollisionFunc (Source/Particles/Collision/BinaryCollision/Coulomb/PairWiseCoulombCollisionFunc.H)
 * with its CoulombLog (<= 0: computed per pair) and the run's collision index and random seed.
 * ---------------------------------------------------------------------------------------- */
typedef struct pic_coulomb_collision {
    double q1, m1, q2, m2;
    double coulomb_log;     /* <name>.CoulombLog; <= 0: computed from the cell's Debye length              */
    uint64_t seed;          /* key of the Philox4x64-10 streams                                            */
    int collision_index;    /* position in collisions.collision_names; part of every stream's counter      */
    int same_species;       /* 1: intra-species (species 2 arguments ignored)                              */
} pic_coulomb_collision;

/* BinaryCollision::doCollisionsWithinTile (BinaryCollision/BinaryCollision.H:234-750) over the box of the bins, dt =
 * the collision's dt (dt * ndt, CollisionHandler.cpp:85-93): per cell, density (and temperature,
 * Coulomb/ComputeTemperature.H), ShuffleFisherYates, the independent pair chains of ElasticCollisionPerez
 * (Coulomb/ElasticCollisionPerez.H:57-148) and UpdateMomentumPerezElastic (Coulomb/UpdateMomentumPerezElastic.H).
 * The bins must be current (np_binned == np); src1 / src2: the pending permutation of pic_sort_index_by_cell (slot ->
 * storage index), NULL when the particles lie in bin order.  Both species' bins describe the same box and tiles.
 * Only ux, uy, uz change; positions, weights, ids, cell_start and src keep their bits.  The result depends on the
 * particles of each cell by id, the seed, the collision index, `step` and the global cell, not on storage order
 * (csrc/collision.cu states the random-stream layout).  scratch1 / scratch2: one device int per particle of each
 * species (e.g. pic_sort_scratch of its sort workspace), used only by cells of more than 2048 colliding particles;
 * with NULL such cells are left unchanged and *status (device int, zeroed by the caller) becomes non-zero. */
int pic_collide_pairwise_coulomb(const pic_coulomb_collision* c, const pic_soa* p1, const pic_bins* b1, const int* src1,
                                 const pic_soa* p2, const pic_bins* b2, const int* src2, const pic_geom* g, double dt,
                                 long step, int* scratch1, int* scratch2, int* status, void* stream);
/* One entry of collisions.collision_names for the step driver (CollisionHandler, Source/Particles/Collision/
 * CollisionHandler.cpp:26-93): species isp1 with isp2 (the same index: intra-species), <name>.CoulombLog,
 * <name>.ndt >= 1, the random seed.  Collisions run after ExplicitFillBoundaryEBUpdateAux and before the push
 * (WarpXEvolve.cpp:141-159), at the steps with int(floor(t / dt)) % ndt == 0, with dt * ndt.  A colliding species is
 * sorted by cell before its collision whenever its bins are stale.  Species without bins, indices out of range,
 * ndt < 1, runs with fluid species, runs over several ranks (not yet checked against a single box) and a species that
 * is a reactant of an earlier pic_engine_add_fusion entry are refused before the engine changes. */
int pic_engine_add_collision(void* engine, int isp1, int isp2, double coulomb_log, int ndt, uint64_t seed);

/* ------------------------------------------------------------------------------------------
 * Nuclear fusion (collisions.collision_names, <name>.type = nuclearfusion), 3D Cartesian:
 * NuclearFusionFunc (Source/Particles/Collision/BinaryCollision/NuclearFusion/NuclearFusionFunc.H) with
 * SingleNuclearFusionEvent.H, BoschHaleFusionCrossSection.H or ProtonBoronFusionCrossSection.H, and the products of
 * ParticleCreationFunc.H:170-225 (TwoProductFusionInitializeMomentum.H, ProtonBoronFusionInitializeMomentum.H).
 * D + He3 is not supported.
 * ---------------------------------------------------------------------------------------- */
enum { PIC_FUSION_DT_NHE4 = 0,   /* D + T  -> n + He4, 17.5893 MeV   (DeuteriumTritiumToNeutronHelium)  */
       PIC_FUSION_DD_PT = 1,     /* D + D  -> p + T,   4.032667 MeV  (DeuteriumDeuteriumToProtonTritium) */
       PIC_FUSION_DD_NHE3 = 2,   /* D + D  -> n + He3, 3.268911 MeV  (DeuteriumDeuteriumToNeutronHelium) */
       PIC_FUSION_PB_3HE4 = 3 }; /* p + B11 -> 3 He4 through alpha + 8Be*, 5.55610759 + 3.12600414 MeV
                                  * (ProtonBoronToAlphas); one product species, mB unused */

/* Particle id of a reactant whose weight the fusion used up (BinaryCollisionUtils.H:140-162 sets
 * amrex::ParticleIdCpus::Invalid): later pairs skip it, later fusion entries of the step leave it out (the engine refuses
 * a Coulomb entry that would follow a fusion on a shared species), and the step removes it
 * where it removes the particles lost at absorbing faces. */
#define PIC_SPENT_ID 0xFFFFFFFFFFFFFFFFull

typedef struct pic_fusion_collision {
    double q1, m1, q2, m2;       /* reactants 1 and 2 (species 2 = species 1 when same_species)              */
    double mA, mB;               /* product species A and B, in the order of <name>.product_species          */
    int type;                    /* PIC_FUSION_*                                                             */
    double fusion_multiplier;                /* <name>.fusion_multiplier (default 1)                        */
    double fusion_probability_threshold;     /* <name>.fusion_probability_threshold (default 0.02)          */
    double fusion_probability_target_value;  /* <name>.fusion_probability_target_value (default 0.002)      */
    uint64_t seed;               /* key of the Philox4x64-10 streams                                         */
    int collision_index;         /* position in collisions.collision_names                                   */
    int same_species;
} pic_fusion_collision;

/* Device workspace of one fusion collision whose reactants hold at most np1 + np2 particles (np1 when same_species)
 * over `nbins` bins: per-pair records at the cell's own slots, per-bin pair and event counts, their scan. */
long pic_fusion_workspace_bytes(long pair_capacity, long nbins);

/* The event pass: BinaryCollision::doCollisionsWithinTile (BinaryCollision/BinaryCollision.H:383-472 intra-species,
 * :613-730 inter-species) with NuclearFusionFunc::Executor (NuclearFusionFunc.H:127-234) over the box of the bins, dt =
 * the collision's dt.  Per cell: the live particles (id != PIC_SPENT_ID) of each species in ascending id order,
 * ShuffleFisherYates, the pair chains with SingleNuclearFusionEvent; an event takes w_min / multiplier_eff from both
 * reactants and marks a reactant left with weight <= DBL_MIN spent.  Only w and ids change.  The pairs and the
 * per-bin event counts go to `work` (pic_fusion_workspace_bytes(pair_capacity, bins)) for
 * pic_fusion_create_products.  Bins, permutations, scratch and *status as for pic_collide_pairwise_coulomb. */
int pic_collide_nuclear_fusion(const pic_fusion_collision* c, const pic_soa* p1, const pic_bins* b1, const int* src1,
                               const pic_soa* p2, const pic_bins* b2, const int* src2, const pic_geom* g, double dt,
                               long step, int* scratch1, int* scratch2, void* work, long pair_capacity, int* status,
                               void* stream);

/* The product pass (ParticleCreationFunc.H:120-230 with TwoProductFusionInitializeMomentum): an exclusive scan of the
 * event counts, ONE host read of the total (synchronises `stream`), then event e of the call -- cell-major, pair order
 * inside the cell -- writes product A at slots pA->np + 2e, + 1 and product B at pB->np + 2e, + 1: the first of each
 * pair at reactant 1's position, the second at reactant 2's, weight w / 2, ids next_id + 2e (+ 1), momenta isotropic
 * in the centre-of-momentum frame.  The reactants and bins are those of the event pass, unchanged since.  *n_events
 * receives the number of events; the caller adds 2 n_events to both products' counts.  When a product would exceed
 * its capacity nothing is written and the call fails naming the product and the capacity needed.
 * PIC_FUSION_PB_3HE4 (ParticleCreationFunc.H:170-200 with ProtonBoronFusionInitializeMomentum): pB may be NULL and
 * is not touched; event e writes six alphas into pA: alpha k = 0, 1, 2 at slots pA->np + 6e + 2k (reactant 1's
 * position) and + 1 (reactant 2's), weight w / 2, ids next_idA + 6e + 2k (+ 1), the two of each k with one momentum;
 * the caller adds 6 n_events to pA's count. */
int pic_fusion_create_products(const pic_fusion_collision* c, const pic_soa* p1, const pic_bins* b1, const pic_soa* p2,
                               const pic_bins* b2, const pic_geom* g, long step, void* work, long pair_capacity,
                               const pic_soa* pA, long capA, uint64_t next_idA, const pic_soa* pB, long capB,
                               uint64_t next_idB, long* n_events, void* stream);

/* Lists the particles whose id is PIC_SPENT_ID for pic_particles_boundary_compact: work and cap as for
 * pic_particles_boundary_mark, work[0] = how many. */
int pic_particles_mark_spent(const pic_soa* p, int* work, int cap, void* stream);

/* One fusion entry of collisions.collision_names for the step driver: reactants isp1, isp2 (the same index:
 * intra-species), products iprodA, iprodB (PIC_FUSION_* order; iprodB = -1 for PIC_FUSION_PB_3HE4 and only for it,
 * whose alphas all go to iprodA), type, multiplier, probability threshold and target,
 * ndt, seed.  It shares the collision index and the schedule of pic_engine_add_collision.  The event pass runs in the
 * `fusion` stage, the product pass in `fusion_products`; the spent reactants are removed in the step's particle
 * boundary stage.  Refused before the engine changes: indices out of range, reactants without bins, a product equal
 * to a reactant or to the other product, ndt < 1, a bad type or parameter, fluid species, several ranks. */
int pic_engine_add_fusion(void* engine, int isp1, int isp2, int iprodA, int iprodB, int type, double multiplier,
                          double probability_threshold, double probability_target_value, int ndt, uint64_t seed);
/* The id counter of species isp: the id the next particle it creates receives (fusion products, flux injection; ids
 * next_id, next_id + 1, ...).  It starts at the species' initial particle count -- over several ranks the sum of the
 * ranks' counts, which makes pic_engine_add_species a collective call there; a checkpoint carries it.  The setter
 * refuses a value below the species' current count. */
uint64_t pic_engine_species_next_id(void* engine, int isp);
int pic_engine_set_species_next_id(void* engine, int isp, uint64_t next_id);

/* ------------------------------------------------------------------------------------------
 * Flux injection through a plane (<species>.injection_style = NFluxPerCell), 3D Cartesian, lab frame, a constant
 * flux and momentum_distribution_type = gaussianflux: PlasmaInjector::setupNFluxPerCell
 * (Source/Initialization/PlasmaInjector.cpp:295-385) and PhysicalParticleContainer::AddPlasmaFlux
 * (Source/Particles/PhysicalParticleContainer.cpp:1336-1810); csrc/flux_injection.cu states the random streams and ids.
 * ---------------------------------------------------------------------------------------- */
typedef struct pic_flux_injector {
    double num_ppc;              /* <species>.num_particles_per_cell (real, > 0)                                   */
    double surface_flux_pos;     /* <species>.surface_flux_pos [m]                                                 */
    int normal_axis;             /* <species>.flux_normal_axis: 0 = x, 1 = y, 2 = z                                */
    int direction;               /* <species>.flux_direction: +1 or -1                                             */
    double flux;                 /* <species>.flux [m^-2 s^-1] (flux_profile = constant); <= 0 injects nothing     */
    double tmin, tmax;           /* <species>.flux_tmin / flux_tmax [s]; < 0: unset                                */
    double bound_lo[3], bound_hi[3];   /* xmin,ymin,zmin / xmax,ymax,zmax (+-inf when unset)                      */
    double u_m[3], u_th[3];      /* ux_m.. / ux_th.. in units of c (InjectorMomentumGaussianFlux)                  */
    uint64_t seed;               /* key of the Philox4x64-10 streams                                               */
} pic_flux_injector;

/* Device workspace of pic_add_flux_particles for injector inj on the domain g (any box of it); -1 and an error for an
 * injector the library refuses (normal axis, direction, num_ppc, u_th, more than 2^31 particles per call). */
long pic_flux_workspace_bytes(const pic_flux_injector* inj, const pic_geom* g);

/* One step of PhysicalParticleContainer::ContinuousFluxInjection (PhysicalParticleContainer.cpp:2531-2540) ->
 * AddPlasmaFlux (:1336-1810) for the box [box_lo, box_hi] of the domain g, at t = t_new (after cur_time += dt):
 * nothing outside (tmin < 0 || t >= tmin) && (tmax < 0 || t < tmax).  The box owns the plane when box_lo <= pos < box_hi
 * along the normal for direction > 0, box_lo < pos <= box_hi for direction < 0 (find_overlap_flux,
 * AddPlasmaUtilities.cpp:45-109); each of its plane cells that overlaps the bounds draws int(num_ppc + Random)
 * particles, at surface_flux_pos along the normal and uniform over the cell across it (InjectorPositionRandomPlane,
 * InjectorPosition.H:33-63), with the Gaussian-flux normal momentum (SampleGaussianFluxDistribution.H, its sign flipped
 * for direction < 0) and normal transverse momenta (InjectorMomentum.H:98-156), weight flux dx dy dz / num_ppc /
 * dx[normal] dt (AddPlasmaUtilities.H:214-234), each then moved over t_fract = Random dt (UpdatePosition).  Particles
 * outside the box or the bounds (inclusive) are dropped.  They are appended after p->np (the caller adds the return
 * value to its count); ids first_id + cell (floor(num_ppc) + 1) + p for particle p of global plane cell cell, and
 * *ids_used receives the ids the call used up on every box (0 outside the window).  step and injector_index are part
 * of every random stream's counter.  work: pic_flux_workspace_bytes(inj, g) bytes (4 bytes per particle slot of the
 * plane).  The particles are appended in slot order (cell-major, then p) without the dropped ones.  ONE host read of
 * the count (synchronises `stream`); when p->np + the count would exceed capacity nothing is written and the call
 * fails.  Returns the number appended, -1 on error. */
long pic_add_flux_particles(const pic_flux_injector* inj, int injector_index, const pic_geom* g, const int box_lo[3],
                            const int box_hi[3], long step, double t, double dt, const pic_soa* p, long capacity,
                            uint64_t first_id, uint64_t* ids_used, void* work, long work_bytes, void* stream);

/* One <species>.injection_style = NFluxPerCell source of species isp for the step driver: every step injects first in
 * HandleParticlesAtBoundaries (Source/Evolve/WarpXEvolve.cpp:535), in the `flux_injection` stage, before the periodic
 * wrap, the particle boundaries, the removal of spent reactants and the migration, which treat the injected particles
 * like pushed ones; on bricks the brick that owns the plane cell creates them.  The species' id counter advances by
 * the plane's cells times (floor(num_ppc) + 1) every injecting step.  The injector's index (the order of the calls)
 * is part of its streams' counter.  Refused before the engine changes: a bad index or injector, a moving window, a
 * boosted frame (pic_engine_set_boost refuses an engine with flux injectors). */
int pic_engine_add_flux_injector(void* engine, int isp, const pic_flux_injector* inj);

/* <species>.do_not_push / <species>.do_not_deposit of species isp for the step driver (0 or 1 each; both 0 is the
 * default).  do_not_push replaces the early returns of WarpXParticleContainer::PushX (WarpXParticleContainer.cpp:1478)
 * and PhysicalParticleContainer::PushP (PhysicalParticleContainer.cpp:2375) and the skipped gather + push of
 * PhysicalParticleContainer::Evolve (:1948-2053): the species' positions and momenta keep their bits, in the main
 * push, in the half pushes of u at the start and end of a run, and with algo.maxwell_solver = none; it is still sorted,
 * collided, fused and wrapped.  do_not_deposit replaces the early return of DepositCurrent
 * (WarpXParticleContainer.cpp:370): the species is pushed but adds nothing to J (Simulation.rho_numpy leaves it out
 * as MultiParticleContainer::GetChargeDensity does, MultiParticleContainer.cpp:576,598).  A bad index is refused. */
int pic_engine_set_species_flags(void* engine, int isp, int do_not_push, int do_not_deposit);

/* Number of kernels launched by this library since load (bench.py's gpu_launches). */
long pic_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* PIC_B200_H_ */
