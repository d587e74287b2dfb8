// Particle housekeeping between steps: periodic wrap and counting sort by cell.
//
// Replaces what WarpX::HandleParticlesAtBoundaries obtains from AMReX
// (Source/Evolve/WarpXEvolve.cpp:533-581): ParticleContainer::Redistribute's periodic shift
// (amrex::enforcePeriodic, AMReX 24.10 AMReX_ParticleUtil.H -- un-vendored dependency) and
// mypc->SortParticlesByBin (counting sort into cell bins, MultiParticleContainer.cpp:615-624).
#include "pic_common.cuh"
#include "bins.cuh"
#include <cub/device/device_scan.cuh>

namespace pic {

struct WrapGeom { double lo[3], hi[3], len[3]; int periodic[3]; };

__device__ __forceinline__ double wrap1(double v, double lo, double hi, double len) {
    if (v > hi) {
        while (v > hi) v -= len;
        if (v < lo) v = lo;          // clamp round-off
    } else if (v < lo) {
        while (v < lo) v += len;
        if (v > hi) v = hi;
    }
    return v;
}

__global__ void wrap_kernel(SoaView P, long np, WrapGeom g) {
    const long ip = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (ip >= np) return;
    // only particles outside the domain are rewritten (the others cost a read, not a read+write)
    if (g.periodic[0]) { const double v = P.x[ip], w = wrap1(v, g.lo[0], g.hi[0], g.len[0]); if (w != v) P.x[ip] = w; }
    if (g.periodic[1]) { const double v = P.y[ip], w = wrap1(v, g.lo[1], g.hi[1], g.len[1]); if (w != v) P.y[ip] = w; }
    if (g.periodic[2]) { const double v = P.z[ip], w = wrap1(v, g.lo[2], g.hi[2], g.len[2]); if (w != v) P.z[ip] = w; }
}

// the particles pic_gather_push listed (pic_escape_list); full grid-stride sweep if the list overflowed
__global__ void wrap_listed_kernel(SoaView P, long np, WrapGeom g, const int* __restrict__ idx,
                                   const int* __restrict__ count, int cap) {
    const long tid = (long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long)gridDim.x * blockDim.x;
    const int n = *count;
    auto wrap_one = [&](long ip) {
        if (g.periodic[0]) { const double v = P.x[ip], w = wrap1(v, g.lo[0], g.hi[0], g.len[0]); if (w != v) P.x[ip] = w; }
        if (g.periodic[1]) { const double v = P.y[ip], w = wrap1(v, g.lo[1], g.hi[1], g.len[1]); if (w != v) P.y[ip] = w; }
        if (g.periodic[2]) { const double v = P.z[ip], w = wrap1(v, g.lo[2], g.hi[2], g.len[2]); if (w != v) P.z[ip] = w; }
    };
    if (n <= cap) { for (long t = tid; t < n; t += stride) wrap_one(idx[t]); }
    else { for (long ip = tid; ip < np; ip += stride) wrap_one(ip); }
}

struct SortGeom { double plo[3], dinv[3]; };

// Warp-aggregated histogram / slot allocation: particles are nearly sorted already, so the lanes of a
// warp mostly hit the same few bins; one atomic per distinct bin per warp instead of one per lane.
__device__ __forceinline__ int warp_aggregated_add(int* counters, int bin, bool active, int* rank_out) {
    const unsigned peers = __match_any_sync(__activemask(), active ? bin : -1 - (int)(threadIdx.x & 31));
    const int lane = threadIdx.x & 31;
    const int leader = __ffs(peers) - 1;
    const int rank = __popc(peers & ((1u << lane) - 1u));
    int base = 0;
    if (active && lane == leader) base = atomicAdd(&counters[bin], __popc(peers));
    base = __shfl_sync(peers, base, leader);
    *rank_out = rank;
    return base;
}

__global__ void sort_count_kernel(SoaView P, long np, BinsView b, SortGeom sg, int* __restrict__ keys,
                                  int* __restrict__ counts) {
    const long ip = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = ip < np;
    int bin = 0;
    if (active) {
        int ci = (int)floor((P.x[ip] - sg.plo[0]) * sg.dinv[0]) - b.box_lo[0];
        int cj = (int)floor((P.y[ip] - sg.plo[1]) * sg.dinv[1]) - b.box_lo[1];
        int ck = (int)floor((P.z[ip] - sg.plo[2]) * sg.dinv[2]) - b.box_lo[2];
        ci = min(max(ci, 0), b.n[0] - 1); cj = min(max(cj, 0), b.n[1] - 1); ck = min(max(ck, 0), b.n[2] - 1);
        bin = (int)bin_of_cell(b, ci, cj, ck);
        keys[ip] = bin;
    }
    int rank;
    warp_aggregated_add(counts, bin, active, &rank);
}

// the slot of every particle in the binned order, as the permutation src[slot] = particle
__global__ void sort_index_kernel(long np, const int* __restrict__ keys, const int* __restrict__ cell_start,
                                  int* __restrict__ fill, int* __restrict__ src) {
    const long ip = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = ip < np;
    const int bin = active ? keys[ip] : 0;
    int rank;
    const int base = warp_aggregated_add(fill, bin, active, &rank);
    if (active) src[cell_start[bin] + base + rank] = (int)ip;
}

// out[pos] = in[src[pos]]: coalesced stores; the loads follow src, which is monotone except where particles changed cell
__global__ void sort_apply_kernel(SoaView in, SoaView out, const uint64_t* __restrict__ id_in,
                                  uint64_t* __restrict__ id_out, long np, const int* __restrict__ src) {
    const long pos = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pos >= np) return;
    const int ip = src[pos];
    out.x[pos] = in.x[ip]; out.y[pos] = in.y[ip]; out.z[pos] = in.z[ip]; out.w[pos] = in.w[ip];
    out.ux[pos] = in.ux[ip]; out.uy[pos] = in.uy[ip]; out.uz[pos] = in.uz[ip];
    if (id_in && id_out) id_out[pos] = id_in[ip];
}

// which particles leave the rank's brick along one axis (cell index of the wrapped position).
// Neighbour ownership is periodic: cells just above cell_hi (or wrapped to the bottom of the domain when this brick is
// the last one) belong to the high neighbour.  both_up: 1 = two ranks along a periodic dim (both neighbours are the same
// rank); 2 = non-periodic dim (ownership does not wrap: above the brick -> high neighbour, below -> low neighbour).
__device__ __forceinline__ void classify_one(long ip, const double* __restrict__ pos, double plo, double dinv, int ncell,
                                             int cell_lo, int cell_hi, int both_up, int* __restrict__ counts,
                                             int* __restrict__ idx_lo, int* __restrict__ idx_hi, int capacity) {
    int c = (int)floor((pos[ip] - plo) * dinv);
    c = min(max(c, 0), ncell - 1);
    if (c >= cell_lo && c <= cell_hi) return;
    const int width = cell_hi - cell_lo + 1;
    const int up_lo = (cell_hi + 1) % ncell;                       // first cell of the high neighbour
    const bool up = both_up == 2 ? (c > cell_hi) : (both_up || (c >= up_lo && c < up_lo + width));
    if (up) { const int n = atomicAdd(&counts[1], 1); if (n < capacity) idx_hi[n] = (int)ip; }
    else    { const int n = atomicAdd(&counts[0], 1); if (n < capacity) idx_lo[n] = (int)ip; }
}

__global__ void classify_kernel(const double* __restrict__ pos, long np_host, const int* __restrict__ np_dev,
                                double plo, double dinv, int ncell,
                                int cell_lo, int cell_hi, int both_up, int* __restrict__ counts,
                                int* __restrict__ idx_lo, int* __restrict__ idx_hi, int capacity) {
    const long ip = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long np = np_dev ? (long)*np_dev : np_host;
    if (ip >= np) return;
    classify_one(ip, pos, plo, dinv, ncell, cell_lo, cell_hi, both_up, counts, idx_lo, idx_hi, capacity);
}

// candidates only (the list of the push, extended by pic_migrate_note_appended); every particle if the list overflowed
__global__ void classify_listed_kernel(const double* __restrict__ pos, long np_host, const int* __restrict__ np_dev,
                                       double plo, double dinv, int ncell, int cell_lo, int cell_hi, int both_up,
                                       int* __restrict__ counts, int* __restrict__ idx_lo, int* __restrict__ idx_hi,
                                       int capacity, int* __restrict__ cand, const int* __restrict__ cand_count, int cand_cap) {
    const long tid = (long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long)gridDim.x * blockDim.x;
    const long np = np_dev ? (long)*np_dev : np_host;
    const int n = *cand_count;
    if (n <= cand_cap) {
        for (long t = tid; t < n; t += stride) {
            const int ip = cand[t];
            if (ip < 0) continue;
            if (ip >= np) { cand[t] = -1; continue; }
            classify_one(ip, pos, plo, dinv, ncell, cell_lo, cell_hi, both_up, counts, idx_lo, idx_hi, capacity);
        }
    } else {
        for (long ip = tid; ip < np; ip += stride)
            classify_one(ip, pos, plo, dinv, ncell, cell_lo, cell_hi, both_up, counts, idx_lo, idx_hi, capacity);
    }
}

// one CTA: the particles the last unpack appended, [np_old, np_new), become candidates of the next axis sweep
__global__ void note_appended_kernel(const int* __restrict__ work, int* __restrict__ cand, int* __restrict__ cand_count,
                                     int cand_cap) {
    const int np_old = work[4], np_new = work[5];
    const int base = *cand_count;
    __syncthreads();
    if (base > cand_cap || np_new <= np_old) return;
    const int n = np_new - np_old;
    if (base + n > cand_cap) { if (threadIdx.x == 0) *cand_count = cand_cap + 1; return; }    // overflow: full sweeps from here
    for (int t = threadIdx.x; t < n; t += blockDim.x) cand[base + t] = np_old + t;
    if (threadIdx.x == 0) *cand_count = base + n;
}

static size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }
static size_t scan_temp_bytes(long n) {
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, bytes, (int*)nullptr, (int*)nullptr, (int)n);
    return bytes;
}

}  // namespace pic

using namespace pic;

extern "C" int pic_particles_wrap_periodic(const pic_soa* p, const pic_geom* g, void* stream) {
    if (p->np == 0) return 0;
    WrapGeom wg;
    for (int d = 0; d < 3; ++d) {
        wg.lo[d] = g->prob_lo[d]; wg.hi[d] = g->prob_hi[d]; wg.len[d] = g->prob_hi[d] - g->prob_lo[d];
        wg.periodic[d] = g->periodic[d];
    }
    wrap_kernel<<<(unsigned)((p->np + 255) / 256), 256, 0, (cudaStream_t)stream>>>(make_soa(*p, 0), p->np, wg);
    count_launch();
    return check_launch("pic_particles_wrap_periodic") ? 0 : 1;
}

extern "C" int pic_particles_wrap_listed(const pic_soa* p, const pic_geom* g, const pic_escape_list* e, void* stream) {
    if (p->np == 0) return 0;
    PIC_REQUIRE(e && e->idx && e->count, "pic_particles_wrap_listed: no escape list");
    WrapGeom wg;
    for (int d = 0; d < 3; ++d) {
        wg.lo[d] = g->prob_lo[d]; wg.hi[d] = g->prob_hi[d]; wg.len[d] = g->prob_hi[d] - g->prob_lo[d];
        wg.periodic[d] = g->periodic[d];
    }
    wrap_listed_kernel<<<NUM_SMS * 8, 256, 0, (cudaStream_t)stream>>>(make_soa(*p, 0), p->np, wg, e->idx, e->count, e->capacity);
    count_launch();
    return check_launch("pic_particles_wrap_listed") ? 0 : 1;
}

extern "C" int pic_particles_classify(const pic_soa* p, const pic_geom* g, int dim, int cell_lo, int cell_hi,
                                      int both_up, int* counts, int* idx_lo, int* idx_hi, int capacity,
                                      const int* np_dev, void* stream) {
    PIC_REQUIRE(dim >= 0 && dim < 3, "pic_particles_classify: bad dimension");
    cudaStream_t s = (cudaStream_t)stream;
    cudaMemsetAsync(counts, 0, 2 * sizeof(int), s);
    if (p->np == 0) return 0;
    const double* pos = dim == 0 ? p->x : (dim == 1 ? p->y : p->z);
    const double dinv = 1.0 / ((g->prob_hi[dim] - g->prob_lo[dim]) / g->n_cell[dim]);
    classify_kernel<<<(unsigned)((p->np + 255) / 256), 256, 0, s>>>(pos, p->np, np_dev, g->prob_lo[dim], dinv, g->n_cell[dim],
                                                                  cell_lo, cell_hi, both_up, counts, idx_lo, idx_hi, capacity);
    count_launch();
    return check_launch("pic_particles_classify") ? 0 : 1;
}

extern "C" int pic_particles_classify_listed(const pic_soa* p, const pic_geom* g, int dim, int cell_lo, int cell_hi,
                                             int both_up, int* counts, int* idx_lo, int* idx_hi, int capacity,
                                             const int* np_dev, const pic_escape_list* cand, void* stream) {
    PIC_REQUIRE(dim >= 0 && dim < 3, "pic_particles_classify_listed: bad dimension");
    PIC_REQUIRE(cand && cand->idx && cand->count, "pic_particles_classify_listed: no candidate list");
    cudaStream_t s = (cudaStream_t)stream;
    cudaMemsetAsync(counts, 0, 2 * sizeof(int), s);
    if (p->np == 0) return 0;
    const double* pos = dim == 0 ? p->x : (dim == 1 ? p->y : p->z);
    const double dinv = 1.0 / ((g->prob_hi[dim] - g->prob_lo[dim]) / g->n_cell[dim]);
    classify_listed_kernel<<<NUM_SMS * 8, 256, 0, s>>>(pos, p->np, np_dev, g->prob_lo[dim], dinv, g->n_cell[dim], cell_lo, cell_hi,
                                                   both_up, counts, idx_lo, idx_hi, capacity, cand->idx, cand->count,
                                                   cand->capacity);
    count_launch();
    return check_launch("pic_particles_classify_listed") ? 0 : 1;
}

extern "C" int pic_migrate_note_appended(const void* work, const pic_escape_list* cand, void* stream) {
    PIC_REQUIRE(work && cand && cand->idx && cand->count, "pic_migrate_note_appended: no workspace / candidate list");
    note_appended_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>((const int*)work, cand->idx, cand->count, cand->capacity);
    count_launch();
    return check_launch("pic_migrate_note_appended") ? 0 : 1;
}

extern "C" long pic_bins_count(const int box_lo[3], const int box_hi[3], const int tile[3]) {
    pic_bins b;
    for (int d = 0; d < 3; ++d) { b.box_lo[d] = box_lo[d]; b.box_hi[d] = box_hi[d]; b.tile[d] = tile[d]; }
    b.cell_start = nullptr;
    return bins_count(make_bins(b));
}

extern "C" long pic_sort_workspace_bytes(long np, long nbins) {
    return (long)(2 * align256((size_t)np * 4) + 2 * align256((size_t)(nbins + 1) * 4) + align256(scan_temp_bytes(nbins + 1)));
}

extern "C" int pic_sort_index_by_cell(const pic_soa* in, const pic_geom* g, const pic_bins* bins, void* work,
                                      const int** src_out, void* stream) {
    const long np = in->np;
    BinsView bv = make_bins(*bins);
    const long nbins = bins_count(bv);
    PIC_REQUIRE(nbins + 1 < (1L << 31) && np < (1L << 31), "pic_sort_index_by_cell: too many bins/particles for int32");
    cudaStream_t s = (cudaStream_t)stream;
    char* w = (char*)work;
    int* src = (int*)w; w += align256((size_t)np * 4);
    int* keys = (int*)w; w += align256((size_t)np * 4);
    int* counts = (int*)w; w += align256((size_t)(nbins + 1) * 4);
    int* fill = (int*)w; w += align256((size_t)(nbins + 1) * 4);
    void* temp = w;
    size_t temp_bytes = scan_temp_bytes(nbins + 1);
    int* cell_start = const_cast<int*>(bins->cell_start);
    cudaMemsetAsync(counts, 0, (size_t)(nbins + 1) * 4, s);
    cudaMemsetAsync(fill, 0, (size_t)(nbins + 1) * 4, s);
    SortGeom sg;
    for (int d = 0; d < 3; ++d) {
        sg.plo[d] = g->prob_lo[d];
        sg.dinv[d] = 1.0 / ((g->prob_hi[d] - g->prob_lo[d]) / g->n_cell[d]);
    }
    if (np > 0) {
        sort_count_kernel<<<(unsigned)((np + 255) / 256), 256, 0, s>>>(make_soa(*in, 0), np, bv, sg, keys, counts);
        count_launch();
    }
    cub::DeviceScan::ExclusiveSum(temp, temp_bytes, counts, cell_start, (int)(nbins + 1), s);
    count_launch();
    if (np > 0) {
        sort_index_kernel<<<(unsigned)((np + 255) / 256), 256, 0, s>>>(np, keys, cell_start, fill, src);
        count_launch();
    }
    *src_out = src;
    return check_launch("pic_sort_index_by_cell") ? 0 : 1;
}

// the per-particle int array of the sort workspace that only pic_sort_index_by_cell uses (its bin keys): free between
// sorts, np entries for the np of the last index
extern "C" int* pic_sort_scratch(void* work, long np) {
    return reinterpret_cast<int*>(static_cast<char*>(work) + align256((size_t)np * 4));
}

extern "C" int pic_sort_apply_permutation(const pic_soa* in, const pic_soa* out, const int* src, void* stream) {
    const long np = in->np;
    PIC_REQUIRE(out->np == np, "pic_sort_apply_permutation: in/out sizes differ");
    PIC_REQUIRE(in->x != out->x, "pic_sort_apply_permutation: in-place permutation is not supported");
    if (np == 0) return 0;
    sort_apply_kernel<<<(unsigned)((np + 255) / 256), 256, 0, (cudaStream_t)stream>>>(make_soa(*in, 0), make_soa(*out, 0),
        in->idcpu, out->idcpu, np, src);
    count_launch();
    return check_launch("pic_sort_apply_permutation") ? 0 : 1;
}

extern "C" int pic_sort_particles_by_cell(const pic_soa* in, const pic_soa* out, const pic_geom* g,
                                          const pic_bins* bins, void* work, void* stream) {
    PIC_REQUIRE(out->np == in->np, "pic_sort_particles_by_cell: in/out sizes differ");
    PIC_REQUIRE(in->x != out->x, "pic_sort_particles_by_cell: in-place sort is not supported");
    const int* src = nullptr;
    if (int rc = pic_sort_index_by_cell(in, g, bins, work, &src, stream)) return rc;
    return pic_sort_apply_permutation(in, out, src, stream);
}
