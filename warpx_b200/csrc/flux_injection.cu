// Flux injection through a plane (<species>.injection_style = NFluxPerCell with momentum_distribution_type =
// gaussianflux and a constant flux) over the rank's box, lab frame.
//
// Restates (paths relative to Source/ of ECP-WarpX/WarpX):
//   plane_of_box    <- find_overlap_flux                           Particles/AddPlasmaUtilities.cpp:45-109
//   count_kernel    <- AddPlasmaFlux, the counting ParallelForRNG  Particles/PhysicalParticleContainer.cpp:1472-1530
//   create_kernel   <- AddPlasmaFlux, the creating ParallelForRNG  :1570-1790, with
//                      InjectorPositionRandomPlane                 Initialization/InjectorPosition.H:33-63
//                      InjectorMomentumGaussianFlux                Initialization/InjectorMomentum.H:98-156
//                      generateGaussianFluxDist (gaussian_flux)    Initialization/SampleGaussianFluxDistribution.H
//                      compute_scale_fac_area_plane (the weight)   Particles/AddPlasmaUtilities.H:214-234
//                      UpdatePosition over t_fract                 Particles/Pusher/UpdatePosition.H
//   the dropped particles: the Redistribute of AddPlasmaFlux's temporary container (:1801-1806), here a keep flag per
//   particle slot whose scan leaves them out.
//
// Determinism: a particle is a function of (seed, injector index, step, global plane cell, its index p in the cell) and
// nothing else -- not of the decomposition or the thread mapping:
//   * random streams: Philox4x64-10 keyed by (seed, 0), counter (j + 1, step, global plane cell,
//     2^63 | 2^61 | injector index << 32 | tag) for block j (binary_collision.cuh's Stream, amrex::Random in (0, 1]).
//     Tag 0 draws the cell's count, int(num_ppc + Random) held to floor(num_ppc) + 1; tag 1 + p is particle p's sequential stream: the two
//     transverse position uniforms (in increasing axis order), the normal momentum (gaussian_flux), the two transverse
//     momenta (random_normal, in increasing axis order), then t_fract.  Bit 61 keeps these streams apart from the
//     collision (2^63 | index << 32 | tag, index < 2^29) and fusion-product (2^63 | 2^62 | ...) streams;
//   * amrex::RandomNormal(mean, stddev) is random_normal: Box-Muller on two consecutive uniforms, the cosine branch;
//   * global plane cell: i0 + n0 i1 over the domain's cells along the two transverse axes (t0 < t1);
//   * positions across the plane: prob_lo + (global cell index + r) dx -- getCellCoords of the reference on a single box
//     (its overlap corner is then prob_lo and its cell index global), the same bits on any decomposition (a box's own
//     overlap corner, prob_lo + shifted dx, would round differently from box to box);
//   * ids: first_id + cell (floor(num_ppc) + 1) + p, the same on any decomposition; a call inside the injection window
//     uses up n0 n1 (floor(num_ppc) + 1) ids, whether or not this box owns the plane;
//   * output order: slot order (cell-major, then p) without the particles a box drops (outside its RealBox or the
//     species' bounds, flux <= 0).  keep_kernel decides, per slot, whether it holds a kept particle (the count and the
//     position draws); an in-place exclusive scan of those flags gives every kept particle its output slot and, with
//     ONE host read, the total; create_kernel writes the particles.  No atomics, no second host read;
//   * the file is compiled without FMA contraction and keeps the reference's expression order.
#include "binary_collision.cuh"
#include <cub/device/device_scan.cuh>
#include <algorithm>
#include <cmath>

namespace pic {
namespace flux {

using coll::Stream;
constexpr uint64_t FLUX_TAG = 1ull << 61;
constexpr int THREADS = 128;

// amrex::RandomNormal(mean, stddev, engine) of this project: Box-Muller on two consecutive uniforms, the cosine branch
__host__ __device__ __forceinline__ double random_normal(double mean, double stddev, Stream& rng) {
    const double u1 = rng.uniform();
    const double u2 = rng.uniform();
    return mean + stddev * (sqrt(-2.0 * log(u1)) * cos(2.0 * coll::PI * u2));
}

// generateGaussianFluxDist: u with p(u) ~ u exp(-(u - u_m)^2 / 2 u_th^2), u > 0
__host__ __device__ __forceinline__ double gaussian_flux(double u_m, double u_th, Stream& rng) {
    double u = 0.0;
    const double abs_u_m = fabs(u_m);
    if (u_th == 0.0) {
        u = u_m;
    } else if (abs_u_m < 0.6 * u_th) {
        const double umsign = copysign(1.0, u_m);
        const double approx_u_th = u_th / sqrt(1.0 - abs_u_m / u_th);
        const double reject_prefactor = (abs_u_m / u_th) / (2.0 * u_th * u_th);
        bool reject = true;
        while (reject) {
            double xrand = 1.0 - rng.uniform();
            u = approx_u_th * sqrt(2.0 * log(1.0 / xrand));
            xrand = rng.uniform();
            if (xrand < exp(-reject_prefactor * (u - umsign * u_th) * (u - umsign * u_th))) reject = false;
        }
    } else {
        bool reject = true;
        const double approx_u_m = u_m + u_th * u_th / abs_u_m;
        const double inv_um = 1.0 / abs_u_m;
        while (reject) {
            u = -1.0;
            while (u < 0) u = random_normal(approx_u_m, u_th, rng);
            const double xrand = rng.uniform();
            if (xrand < u * inv_um * exp(1.0 - u * inv_um)) reject = false;
        }
    }
    return u;
}

// The box's share of the plane (find_overlap_flux with part_realbox = the problem domain)
struct Plane {
    int axis, t0, t1;      // normal axis, transverse axes (t0 < t1)
    int n0, n1;            // the box's plane cells along t0, t1
    int g0, g1;            // global index of its first plane cell along t0, t1 (`shifted`)
    double corner[3];      // prob_lo across the plane, the plane itself along the normal
    double tile_lo[3], tile_hi[3];
};

struct Args {
    SoaView P;                 // pointers start at the old np
    uint64_t* id;
    Plane pl;
    long gn0;                  // global plane cells along t0
    int slots;                 // floor(num_ppc) + 1
    double dx[3], bound_lo[3], bound_hi[3], u_m[3], u_th[3];
    double um_n, uth_n;        // u_m, u_th along the normal
    double num_ppc, flux, weight, dt;
    int direction;
    uint64_t seed, step, tag, first_id;
    int* keep;                 // per slot: 1 when it holds a kept particle; scanned in place into the output slots
};

__device__ __forceinline__ uint64_t global_cell(const Args& a, int i0, int i1) {
    return (uint64_t)(a.pl.g0 + i0) + (uint64_t)a.gn0 * (uint64_t)(a.pl.g1 + i1);
}

// InjectorPositionRandomPlane + getCellCoords: the first two uniforms of the particle's stream for the transverse axes
// in increasing order, 0 along the normal.  The components are selected with the axis as a value (no local arrays
// indexed at run time).
__device__ __forceinline__ void position(const Args& a, int i0, int i1, Stream& rng, double pos[3]) {
    const double ra = rng.uniform(), rb = rng.uniform();
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const bool first = d == a.pl.t0;
        const double r = d == a.pl.axis ? 0.0 : (first ? ra : rb);
        const int iv = d == a.pl.axis ? 0 : (first ? a.pl.g0 + i0 : a.pl.g1 + i1);
        pos[d] = a.pl.corner[d] + (iv + r) * a.dx[d];
    }
}

// One thread per particle slot (cell, p < floor(num_ppc) + 1): keep[slot] = 1 when p is below the cell's count and the
// particle is not dropped.  The cell's count, int(num_ppc + Random), is 0 when the cell does not overlap the species'
// bounds; it is held to the slots (num_ppc + Random can round up to floor(num_ppc) + 2 when num_ppc lies just below an
// integer).  A particle is dropped outside the box's RealBox or the bounds (both inclusive) or with flux <= 0.
__global__ void __launch_bounds__(THREADS) keep_kernel(Args a, long nslots) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nslots) return;
    const long c = t / a.slots;
    const int p = (int)(t % a.slots);
    const int i0 = (int)(c % a.pl.n0), i1 = (int)(c / a.pl.n0);
    bool overlaps = true;           // InjectorPosition::overlapsWith(getCellCoords(r = 0), getCellCoords(r = 1))
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const int iv = d == a.pl.axis ? 0 : (d == a.pl.t0 ? a.pl.g0 + i0 : a.pl.g1 + i1);
        const double lo = a.pl.corner[d] + (iv + 0.0) * a.dx[d];
        const double hi = a.pl.corner[d] + (iv + 1.0) * a.dx[d];
        overlaps = overlaps && a.bound_lo[d] <= hi && a.bound_hi[d] >= lo;
    }
    int keep = 0;
    if (overlaps) {
        const uint64_t gcell = global_cell(a, i0, i1);
        Stream cnt(a.seed, a.step, gcell, a.tag);
        const int n = min(static_cast<int>(a.num_ppc + cnt.uniform()), a.slots);
        if (p < n) {
            Stream rng(a.seed, a.step, gcell, a.tag | (uint64_t)(1 + p));
            double pos[3];
            position(a, i0, i1, rng, pos);
            bool ok = true;
#pragma unroll
            for (int d = 0; d < 3; ++d) ok = ok && a.pl.tile_lo[d] <= pos[d] && pos[d] <= a.pl.tile_hi[d];  // containsInclusive
#pragma unroll
            for (int d = 0; d < 3; ++d) ok = ok && pos[d] <= a.bound_hi[d] && pos[d] >= a.bound_lo[d];      // insideBoundsInclusive
            keep = (ok && !(a.flux <= 0)) ? 1 : 0;
        }
    }
    a.keep[t] = keep;
}

// One thread per particle slot: a kept particle goes to its scanned output slot, keep[t] (keep[t + 1] - keep[t] = 1).
// The stream repeats keep_kernel's position draws, then draws the momenta and t_fract.
__global__ void __launch_bounds__(THREADS) create_kernel(Args a, long nslots) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nslots) return;
    const long ip = a.keep[t];
    if (a.keep[t + 1] == ip) return;
    const long c = t / a.slots;
    const int p = (int)(t % a.slots);
    const int i0 = (int)(c % a.pl.n0), i1 = (int)(c / a.pl.n0);
    const uint64_t gcell = global_cell(a, i0, i1);
    a.id[ip] = a.first_id + gcell * (uint64_t)a.slots + (uint64_t)p;
    a.P.w[ip] = a.weight;
    Stream rng(a.seed, a.step, gcell, a.tag | (uint64_t)(1 + p));
    double pos[3], u[3];
    position(a, i0, i1, rng, pos);
    const int ax = a.pl.axis;
    double un = gaussian_flux(a.um_n, a.uth_n, rng);
    if (a.direction < 0) un = -un;
#pragma unroll
    for (int d = 0; d < 3; ++d) u[d] = d == ax ? un : random_normal(a.u_m[d], a.u_th[d], rng);
#pragma unroll
    for (int d = 0; d < 3; ++d) u[d] *= C_LIGHT;
    a.P.ux[ip] = u[0]; a.P.uy[ip] = u[1]; a.P.uz[ip] = u[2];
    const double t_fract = rng.uniform() * a.dt;
    const double inv_gamma = 1.0 / sqrt(1.0 + (u[0] * u[0] + u[1] * u[1] + u[2] * u[2]) * INV_C2);
    a.P.x[ip] = pos[0] + u[0] * inv_gamma * t_fract;
    a.P.y[ip] = pos[1] + u[1] * inv_gamma * t_fract;
    a.P.z[ip] = pos[2] + u[2] * inv_gamma * t_fract;
}

// the particles [first, first + n) join the escape list (count keeps the true number beyond the capacity)
__global__ void list_kernel(int* __restrict__ idx, const int* __restrict__ count, int cap, long first, long n) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long k = *count + t;
    if (t < n && k < cap) idx[k] = (int)(first + t);
}
__global__ void list_count_kernel(int* count, long n) { *count += (int)n; }

static size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

static size_t scan_bytes(long n) {
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, bytes, (int*)nullptr, (int*)nullptr, (int)n);
    return bytes;
}

// the workspace for up to `slots` particle slots: the keep flags, scanned in place (slots + 1 ints), and the scan's
// temporary storage
struct Work {
    int* keep;
    void* temp;
    size_t temp_bytes;
};

static Work carve(void* base, long slots, size_t* total = nullptr) {
    Work w;
    char* p = static_cast<char*>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) { char* q = p ? p + off : nullptr; off += align256(bytes); return q; };
    w.keep = (int*)take((size_t)(slots + 1) * 4);
    w.temp_bytes = scan_bytes(slots + 1);
    w.temp = take(w.temp_bytes);
    if (total) *total = off;
    return w;
}

static void axes(int axis, int& t0, int& t1) { t0 = axis == 0 ? 1 : 0; t1 = axis == 2 ? 1 : 2; }

static long plane_cells(const pic_flux_injector* f, const pic_geom* g) {
    int t0, t1;
    axes(f->normal_axis, t0, t1);
    return (long)g->n_cell[t0] * g->n_cell[t1];
}

static int check_injector(const char* what, const pic_flux_injector* f, const pic_geom* g) {
    PIC_REQUIRE(f && g, "%s: null argument", what);
    PIC_REQUIRE(f->normal_axis >= 0 && f->normal_axis < 3, "%s: flux_normal_axis must be x, y or z (0, 1, 2), got %d", what,
                f->normal_axis);
    PIC_REQUIRE(f->direction == 1 || f->direction == -1, "%s: flux_direction must be -1 or +1, got %d", what, f->direction);
    PIC_REQUIRE(f->num_ppc > 0.0 && std::isfinite(f->num_ppc) && f->num_ppc < 1.0e6,
                "%s: num_particles_per_cell must be positive and below 1e6", what);
    for (int d = 0; d < 3; ++d)
        PIC_REQUIRE(f->u_th[d] >= 0.0 && std::isfinite(f->u_th[d]) && std::isfinite(f->u_m[d]),
                    "%s: u_th must be finite and non-negative, u_m finite", what);
    PIC_REQUIRE(plane_cells(f, g) * (long)(std::floor(f->num_ppc) + 1) < 2147483647L,
                "%s: one call of this injector could create more than 2^31 particles", what);
    return 0;
}

// find_overlap_flux for the box [box_lo, box_hi]; false when the box does not own the plane or has no plane cell
static bool plane_of_box(const pic_flux_injector* f, const pic_geom* g, const int box_lo[3], const int box_hi[3], Plane& pl) {
    double dx[3];
    for (int d = 0; d < 3; ++d) dx[d] = (g->prob_hi[d] - g->prob_lo[d]) / g->n_cell[d];
    pl.axis = f->normal_axis;
    axes(pl.axis, pl.t0, pl.t1);
    int nov[3];
    for (int d = 0; d < 3; ++d) {
        pl.tile_lo[d] = g->prob_lo[d] + dx[d] * box_lo[d];          // RealBox(tile_box, dx, prob_lo)
        pl.tile_hi[d] = g->prob_lo[d] + dx[d] * (box_hi[d] + 1);
        if (d == pl.axis) {
            const double pos = f->surface_flux_pos;
            if (f->direction > 0 ? (pos < pl.tile_lo[d] || pos >= pl.tile_hi[d]) : (pos <= pl.tile_lo[d] || pos > pl.tile_hi[d]))
                return false;
            pl.corner[d] = pos;
            nov[d] = 1;
            continue;
        }
        const double part_lo = g->prob_lo[d], part_hi = g->prob_hi[d];
        double ov_lo, ov_hi;
        if (pl.tile_lo[d] <= part_hi) {
            const double adj = std::floor((pl.tile_lo[d] - part_lo) / dx[d]);
            ov_lo = part_lo + std::max(adj, 0.0) * dx[d];
        } else return false;
        if (pl.tile_hi[d] >= part_lo) {
            const double adj = std::floor((part_hi - pl.tile_hi[d]) / dx[d]);
            ov_hi = part_hi - std::max(adj, 0.0) * dx[d];
        } else return false;
        nov[d] = int(std::round((ov_hi - ov_lo) / dx[d]));
        pl.corner[d] = g->prob_lo[d];
        const int shifted = static_cast<int>(std::round((ov_lo - g->prob_lo[d]) / dx[d]));
        if (d == pl.t0) pl.g0 = shifted; else pl.g1 = shifted;
    }
    pl.n0 = nov[pl.t0]; pl.n1 = nov[pl.t1];
    return pl.n0 > 0 && pl.n1 > 0;
}

}  // namespace flux

// The particles [first, first + n) of a species join its escape list: the wrap and the migration of the step visit
// them like the particles the push listed.
int flux_list_escapes(const pic_escape_list* e, long first, long n, void* stream) {
    if (n <= 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    flux::list_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(e->idx, e->count, e->capacity, first, n);
    flux::list_count_kernel<<<1, 1, 0, s>>>(e->count, n);
    count_launch(2);
    return check_launch("flux_list_escapes") ? 0 : 1;
}

}  // namespace pic

using namespace pic;

extern "C" long pic_flux_workspace_bytes(const pic_flux_injector* inj, const pic_geom* g) {
    if (flux::check_injector("pic_flux_workspace_bytes", inj, g)) return -1;
    const long cells = flux::plane_cells(inj, g);
    size_t total = 0;
    flux::carve(nullptr, cells * (long)(std::floor(inj->num_ppc) + 1), &total);
    return (long)total;
}

extern "C" long pic_add_flux_particles(const pic_flux_injector* inj, int injector_index, const pic_geom* g,
                                       const int box_lo[3], const int box_hi[3], long step, double t, double dt,
                                       const pic_soa* p, long capacity, uint64_t first_id, uint64_t* ids_used,
                                       void* work, long work_bytes, void* stream) {
    const char* what = "pic_add_flux_particles";
    if (flux::check_injector(what, inj, g)) return -1;
    if (!(box_lo && box_hi && p && ids_used && work)) { fail("%s: null argument", what); return -1; }
    if (!(p->idcpu && p->w)) { fail("%s: the species needs ids and weights", what); return -1; }
    if (!(dt > 0.0) || step < 0 || injector_index < 0) { fail("%s: needs dt > 0, step >= 0 and injector_index >= 0", what); return -1; }
    const long cells = flux::plane_cells(inj, g);
    const int slots = (int)std::floor(inj->num_ppc) + 1;
    const long cap = cells * slots;
    size_t need = 0;
    flux::carve(nullptr, cap, &need);
    if ((size_t)work_bytes < need) { fail("%s: the workspace has %ld bytes, needs %zu", what, work_bytes, need); return -1; }
    *ids_used = 0;
    // ContinuousFluxInjection (PhysicalParticleContainer.cpp:2531-2540): the injection window
    if (!((inj->tmin < 0 || t >= inj->tmin) && (inj->tmax < 0 || t < inj->tmax))) return 0;
    *ids_used = (uint64_t)cap;
    flux::Args a;
    if (!flux::plane_of_box(inj, g, box_lo, box_hi, a.pl)) return 0;
    const long nslots = (long)a.pl.n0 * a.pl.n1 * slots;
    flux::Work w = flux::carve(work, cap);
    cudaStream_t s = (cudaStream_t)stream;
    a.gn0 = g->n_cell[a.pl.t0];
    a.slots = slots;
    for (int d = 0; d < 3; ++d) {
        a.dx[d] = (g->prob_hi[d] - g->prob_lo[d]) / g->n_cell[d];
        a.bound_lo[d] = inj->bound_lo[d]; a.bound_hi[d] = inj->bound_hi[d];
        a.u_m[d] = inj->u_m[d]; a.u_th[d] = inj->u_th[d];
    }
    a.um_n = inj->u_m[a.pl.axis]; a.uth_n = inj->u_th[a.pl.axis];
    a.num_ppc = inj->num_ppc; a.flux = inj->flux; a.dt = dt; a.direction = inj->direction;
    double scale_fac = a.dx[0] * a.dx[1] * a.dx[2] / inj->num_ppc;     // compute_scale_fac_area_plane
    scale_fac /= a.dx[a.pl.axis];
    a.weight = inj->flux * scale_fac * dt;
    a.seed = inj->seed; a.step = (uint64_t)step; a.first_id = first_id;
    a.tag = flux::FLUX_TAG | ((uint64_t)(uint32_t)injector_index << 32);
    a.keep = w.keep;
    const unsigned blocks = (unsigned)((nslots + flux::THREADS - 1) / flux::THREADS);
    cudaMemsetAsync(w.keep + nslots, 0, sizeof(int), s);
    flux::keep_kernel<<<blocks, flux::THREADS, 0, s>>>(a, nslots);
    count_launch();
    cub::DeviceScan::ExclusiveSum(w.temp, w.temp_bytes, w.keep, w.keep, (int)(nslots + 1), s);     // in place
    count_launch();
    int total = 0;
    cudaMemcpyAsync(&total, w.keep + nslots, sizeof(int), cudaMemcpyDeviceToHost, s);
    if (cudaStreamSynchronize(s) != cudaSuccess) { fail("%s: %s", what, cudaGetErrorString(cudaGetLastError())); return -1; }
    if (p->np + total > capacity) {
        fail("%s: %ld + %d injected particles exceed the capacity %ld", what, (long)p->np, total, capacity);
        return -1;
    }
    if (total == 0) return 0;
    a.P = make_soa(*p, p->np);
    a.id = p->idcpu + p->np;
    flux::create_kernel<<<blocks, flux::THREADS, 0, s>>>(a, nslots);
    count_launch();
    return check_launch(what) ? (long)total : -1;
}
