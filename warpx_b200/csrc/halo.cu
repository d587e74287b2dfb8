// Guard-cell operations: FillBoundary (copy) and SumBoundary (add), one dimension at a time.
//
// Replaces ablastr::utils::communication::FillBoundary / SumBoundary as called by
// WarpX::FillBoundaryE/B (Source/Parallelization/WarpXComm.cpp:699-827) and
// WarpX::SumBoundaryJ -> WarpXSumGuardCells (WarpXComm.cpp:1386-1424, WarpXSumGuardCells.cpp:17-24;
// wrappers Source/ablastr/utils/Communication.cpp:71-115, :148-175).  AMReX exchanges all 26
// neighbours at once; here the exchange is done as three axis sweeps (x, y, z), each slab
// spanning the full allocated extent of the other two axes so that edges and corners propagate.
//   * self-neighbour (box spans the periodic domain along the axis): one local kernel;
//   * real neighbour (multi-GPU): pack -> NCCL send/recv (host side) -> unpack(+add).
// All kernels are pure HBM streams with i (contiguous) innermost.
#include "pic_common.cuh"

namespace pic {

struct Slab {
    int dim;
    int n[3];        // iteration extents (n[dim] = number of layers)
    int start[3];    // first index (global) in each direction for the slab being written / read
};

__device__ __forceinline__ void decode(long t, const int n[3], int& a, int& b, int& c) {
    a = (int)(t % n[0]);
    b = (int)((t / n[0]) % n[1]);
    c = (int)(t / ((long)n[0] * n[1]));
}

// guards <- periodic image of valid points (shift by +-N along dim)
__global__ void fill_local_kernel(FabView F, int dim, int N, int vl, int vh, int ng, Slab sl, long total) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total) return;
    int a, b, c;
    decode(t, sl.n, a, b, c);
    int idx[3] = {sl.start[0] + a, sl.start[1] + b, sl.start[2] + c};
    // layers 0..ng-1 -> low guards vl-ng .. vl-1 ; layers ng..2ng-1 -> high guards vh+1 .. vh+ng
    const int layer = (dim == 0) ? a : ((dim == 1) ? b : c);
    int src[3] = {idx[0], idx[1], idx[2]};
    if (layer < ng) { idx[dim] = vl - ng + layer; src[dim] = idx[dim] + N; }
    else { idx[dim] = vh + 1 + (layer - ng); src[dim] = idx[dim] - N; }
    F(idx[0], idx[1], idx[2]) = F(src[0], src[1], src[2]);
}

// valid points accumulate the periodic images of guard points (and the nodal duplicate)
__global__ void sum_local_kernel(FabView F, int dim, int N, int vl, int vh, int src_ng, int nodal,
                                 Slab sl, long total) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total) return;
    int a, b, c;
    decode(t, sl.n, a, b, c);
    int idx[3] = {sl.start[0] + a, sl.start[1] + b, sl.start[2] + c};
    const int layer = (dim == 0) ? a : ((dim == 1) ? b : c);   // 0 .. src_ng (0 only when nodal)
    const int g = nodal ? layer : layer + 1;
    int lo_i[3] = {idx[0], idx[1], idx[2]}, hi_i[3] = {idx[0], idx[1], idx[2]};
    if (g == 0) {
        // nodal duplicate: both copies get v(vl) + v(vh)
        lo_i[dim] = vl; hi_i[dim] = vh;
        const double s = F(lo_i[0], lo_i[1], lo_i[2]) + F(hi_i[0], hi_i[1], hi_i[2]);
        F(lo_i[0], lo_i[1], lo_i[2]) = s;
        F(hi_i[0], hi_i[1], hi_i[2]) = s;
        return;
    }
    // low guard vl-g folds onto vl-g+N ; high guard vh+g folds onto vh+g-N
    int tgt[3] = {idx[0], idx[1], idx[2]};
    lo_i[dim] = vl - g; tgt[dim] = vl - g + N;
    F(tgt[0], tgt[1], tgt[2]) += F(lo_i[0], lo_i[1], lo_i[2]);
    hi_i[dim] = vh + g; tgt[dim] = vh + g - N;
    F(tgt[0], tgt[1], tgt[2]) += F(hi_i[0], hi_i[1], hi_i[2]);
}

// mode 0 copy / 1 sum; dir 0 pack (fab -> buf) / 1 unpack (buf -> fab, adding when mode = 1)
__global__ void slab_kernel(FabView F, double* __restrict__ buf, Slab sl, long total, int dir, int add) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total) return;
    int a, b, c;
    decode(t, sl.n, a, b, c);
    const int i = sl.start[0] + a, j = sl.start[1] + b, k = sl.start[2] + c;
    if (dir == 0) buf[t] = F(i, j, k);
    else if (add) F(i, j, k) += buf[t];
    else F(i, j, k) = buf[t];
}

// all components of an exchange in ONE launch per direction (pack) / per direction (unpack):
// side = side0 + blockIdx.y, the x-grid walks the concatenated slabs of up to PIC_HALO_MAX_FABS components
constexpr int HALO_MAX = 8;
struct MultiSlab {
    FabView v[HALO_MAX];
    Slab sl[2][HALO_MAX];      // [side][component]
    long off[HALO_MAX + 1];    // offsets of the components inside one side's buffer
    int n;
};
__global__ void multi_slab_kernel(MultiSlab m, double* __restrict__ buf_lo, double* __restrict__ buf_hi,
                                  int dir, int add, int side0) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= m.off[m.n]) return;
    const int side = side0 + blockIdx.y;
    int f = 0;
#pragma unroll
    for (int q = 1; q < HALO_MAX; ++q) if (q < m.n && t >= m.off[q]) f = q;
    const Slab& sl = m.sl[side][f];
    const long tl = t - m.off[f];
    int a, b, c;
    decode(tl, sl.n, a, b, c);
    const int i = sl.start[0] + a, j = sl.start[1] + b, k = sl.start[2] + c;
    double* buf = side ? buf_hi : buf_lo;
    const FabView& F = m.v[f];
    if (dir == 0) buf[t] = F(i, j, k);
    else if (add) F(i, j, k) += buf[t];
    else F(i, j, k) = buf[t];
}

// The local (self-neighbour) sweeps of up to HALO_MAX components in ONE launch: the x-grid walks the concatenated
// slabs; every thread does what fill_local_kernel / sum_local_kernel do for its component.
struct MultiLocal {
    FabView v[HALO_MAX];
    Slab sl[HALO_MAX];
    long off[HALO_MAX + 1];
    int vl[HALO_MAX], vh[HALO_MAX], nodal[HALO_MAX];
    int n, dim, N, ng;
};
__global__ void multi_local_kernel(MultiLocal m, int mode) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= m.off[m.n]) return;
    int f = 0;
#pragma unroll
    for (int q = 1; q < HALO_MAX; ++q) if (q < m.n && t >= m.off[q]) f = q;
    const Slab& sl = m.sl[f];
    const FabView& F = m.v[f];
    const int dim = m.dim, N = m.N, vl = m.vl[f], vh = m.vh[f];
    int a, b, c;
    decode(t - m.off[f], sl.n, a, b, c);
    int idx[3] = {sl.start[0] + a, sl.start[1] + b, sl.start[2] + c};
    const int layer = (dim == 0) ? a : ((dim == 1) ? b : c);
    if (mode == 0) {            // fill_local_kernel
        const int ng = m.ng;
        int src[3] = {idx[0], idx[1], idx[2]};
        if (layer < ng) { idx[dim] = vl - ng + layer; src[dim] = idx[dim] + N; }
        else { idx[dim] = vh + 1 + (layer - ng); src[dim] = idx[dim] - N; }
        F(idx[0], idx[1], idx[2]) = F(src[0], src[1], src[2]);
        return;
    }
    // sum_local_kernel
    const int g = m.nodal[f] ? layer : layer + 1;
    int lo_i[3] = {idx[0], idx[1], idx[2]}, hi_i[3] = {idx[0], idx[1], idx[2]};
    if (g == 0) {
        lo_i[dim] = vl; hi_i[dim] = vh;
        const double s2 = F(lo_i[0], lo_i[1], lo_i[2]) + F(hi_i[0], hi_i[1], hi_i[2]);
        F(lo_i[0], lo_i[1], lo_i[2]) = s2;
        F(hi_i[0], hi_i[1], hi_i[2]) = s2;
        return;
    }
    int tgt[3] = {idx[0], idx[1], idx[2]};
    lo_i[dim] = vl - g; tgt[dim] = vl - g + N;
    F(tgt[0], tgt[1], tgt[2]) += F(lo_i[0], lo_i[1], lo_i[2]);
    hi_i[dim] = vh + g; tgt[dim] = vh + g - N;
    F(tgt[0], tgt[1], tgt[2]) += F(hi_i[0], hi_i[1], hi_i[2]);
}

static void full_extent(const pic_fab& f, Slab& sl) {
    for (int d = 0; d < 3; ++d) { sl.start[d] = f.lo[d]; sl.n[d] = f.hi[d] - f.lo[d] + 1; }
}

// index range along `dim` of the slab exchanged with the neighbour on `side`
static void slab_range(const pic_fab& f, int dim, int side, int ng, int mode, int unpack, int& first, int& count) {
    const int lc = vlo(f, dim);                          // first cell
    const int hc = vhi(f, dim) - f.stag[dim];            // last cell
    const int st = f.stag[dim];
    if (mode == 0) {           // copy: send valid layers, receive into guards
        count = ng;
        if (!unpack) first = side ? (hc + 1 - ng) : (lc + st);
        else first = side ? (hc + 1 + st) : (lc - ng);
    } else if (mode == 1) {    // sum: send guards (+ shared node), add into valid
        count = ng + st;
        if (!unpack) first = side ? (hc + 1) : (lc - ng);
        else first = side ? (hc + 1 - ng) : lc;
    } else {                   // sum and refresh in one exchange (PIC_HALO_SUM_REFRESH): both ranks send the whole
        // overlap zone of the face -- ng valid layers, the shared node, ng guards -- and add what they receive to their
        // own partial sums; a + b = b + a bit for bit, so valid points hold SumBoundary's result and the guards the
        // copies FillBoundary would bring.  Needs 2 ng + st <= box width (a point shared by two ranks only): the
        // same bound SumBoundary's source width has.
        count = 2 * ng + st;
        first = side ? (hc + 1 - ng) : (lc - ng);
    }
}

}  // namespace pic

using namespace pic;

extern "C" int pic_fill_boundary_local(const pic_fab* f, int dim, int ng, const pic_geom* g, void* stream) {
    if (ng == 0) return 0;
    const int N = g->n_cell[dim];
    const int vl = vlo(*f, dim), vh = vhi(*f, dim);
    PIC_REQUIRE(g->periodic[dim], "pic_fill_boundary_local: dimension %d is not periodic", dim);
    PIC_REQUIRE(vh - vl + 1 - f->stag[dim] == N, "pic_fill_boundary_local: box does not span the domain in dim %d", dim);
    PIC_REQUIRE(ng <= f->ng[dim] && ng <= N, "pic_fill_boundary_local: ng=%d exceeds allocated guards", ng);
    Slab sl; full_extent(*f, sl); sl.dim = dim; sl.n[dim] = 2 * ng;
    // Along a non-periodic direction the guards beyond the domain face have no periodic image: AMReX
    // FillBoundary leaves (guard of dim) x (guard beyond that face) untouched, so the slab covers
    // only the valid indices there.  (Periodic directions keep the full allocated extent.)
    for (int d = 0; d < 3; ++d)
        if (d != dim && !g->periodic[d]) { sl.start[d] = vlo(*f, d); sl.n[d] = vhi(*f, d) - vlo(*f, d) + 1; }
    const long total = (long)sl.n[0] * sl.n[1] * sl.n[2];
    fill_local_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        make_view(*f), dim, N, vl, vh, ng, sl, total);
    count_launch();
    return check_launch("pic_fill_boundary_local") ? 0 : 1;
}

extern "C" int pic_sum_boundary_local(const pic_fab* f, int dim, int src_ng, const pic_geom* g, void* stream) {
    const int N = g->n_cell[dim];
    const int vl = vlo(*f, dim), vh = vhi(*f, dim);
    const int nodal = f->stag[dim];
    PIC_REQUIRE(g->periodic[dim], "pic_sum_boundary_local: dimension %d is not periodic", dim);
    PIC_REQUIRE(vh - vl + 1 - nodal == N, "pic_sum_boundary_local: box does not span the domain in dim %d", dim);
    PIC_REQUIRE(src_ng <= f->ng[dim] && 2 * src_ng + 1 <= N, "pic_sum_boundary_local: src_ng=%d too large", src_ng);
    Slab sl; full_extent(*f, sl); sl.dim = dim; sl.n[dim] = src_ng + nodal;
    const long total = (long)sl.n[0] * sl.n[1] * sl.n[2];
    if (total == 0) return 0;
    sum_local_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        make_view(*f), dim, N, vl, vh, src_ng, nodal, sl, total);
    count_launch();
    return check_launch("pic_sum_boundary_local") ? 0 : 1;
}

// pic_fill_boundary_local (mode 0, ng guard layers) / pic_sum_boundary_local (mode 1, ng = src_ng) of nfab
// components with one launch.
extern "C" int pic_boundary_local_multi(const pic_fab* fabs, int nfab, int dim, int ng, int mode, const pic_geom* g,
                                        void* stream) {
    PIC_REQUIRE(nfab >= 1 && nfab <= HALO_MAX, "pic_boundary_local_multi: 1..%d components", HALO_MAX);
    PIC_REQUIRE(dim >= 0 && dim < 3 && (mode == 0 || mode == 1), "pic_boundary_local_multi: bad arguments");
    PIC_REQUIRE(g->periodic[dim], "pic_boundary_local_multi: dimension %d is not periodic", dim);
    if (mode == 0 && ng == 0) return 0;
    MultiLocal m;
    m.n = nfab; m.dim = dim; m.N = g->n_cell[dim]; m.ng = ng;
    m.off[0] = 0;
    for (int f = 0; f < nfab; ++f) {
        const pic_fab& F = fabs[f];
        const int vl = vlo(F, dim), vh = vhi(F, dim), nodal = F.stag[dim];
        PIC_REQUIRE(vh - vl + 1 - nodal == m.N, "pic_boundary_local_multi: box does not span the domain in dim %d", dim);
        PIC_REQUIRE(ng <= F.ng[dim] && (mode == 0 ? ng <= m.N : 2 * ng + 1 <= m.N), "pic_boundary_local_multi: ng=%d too large", ng);
        m.v[f] = make_view(F); m.vl[f] = vl; m.vh[f] = vh; m.nodal[f] = nodal;
        Slab& sl = m.sl[f];
        full_extent(F, sl); sl.dim = dim;
        if (mode == 0) {
            sl.n[dim] = 2 * ng;
            for (int d = 0; d < 3; ++d)          // see pic_fill_boundary_local
                if (d != dim && !g->periodic[d]) { sl.start[d] = vlo(F, d); sl.n[d] = vhi(F, d) - vlo(F, d) + 1; }
        } else {
            sl.n[dim] = ng + nodal;
        }
        m.off[f + 1] = m.off[f] + (long)sl.n[0] * sl.n[1] * sl.n[2];
    }
    for (int f = nfab; f < HALO_MAX; ++f) m.off[f + 1] = m.off[nfab];
    const long total = m.off[nfab];
    if (total == 0) return 0;
    multi_local_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(m, mode);
    count_launch();
    return check_launch("pic_boundary_local_multi") ? 0 : 1;
}

extern "C" long pic_halo_slab_count(const pic_fab* f, int dim, int ng, int mode) {
    long n = 1;
    for (int d = 0; d < 3; ++d) if (d != dim) n *= (f->hi[d] - f->lo[d] + 1);
    return n * (mode == 0 ? ng : (mode == 1 ? ng + f->stag[dim] : 2 * ng + f->stag[dim]));
}

// cells of the box along dim
static int box_cells(const pic_fab& f, int dim) { return vhi(f, dim) - vlo(f, dim) + 1 - f.stag[dim]; }

static int slab_launch(const pic_fab* f, int dim, int side, int ng, int mode, double* buf, int unpack, void* stream) {
    PIC_REQUIRE(dim >= 0 && dim < 3 && (side == 0 || side == 1) && (mode == 0 || mode == 1), "pic_halo: bad arguments");
    PIC_REQUIRE(ng >= 0 && ng <= f->ng[dim], "pic_halo: ng=%d exceeds allocated guards", ng);
    // a wider slab would reach through the valid points into the guards of the other face
    PIC_REQUIRE(ng <= box_cells(*f, dim), "pic_halo: ng=%d exceeds the %d cells of the box", ng, box_cells(*f, dim));
    Slab sl; full_extent(*f, sl); sl.dim = dim;
    int first, count;
    slab_range(*f, dim, side, ng, mode, unpack, first, count);
    sl.start[dim] = first; sl.n[dim] = count;
    const long total = (long)sl.n[0] * sl.n[1] * sl.n[2];
    if (total == 0) return 0;
    slab_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        make_view(*f), buf, sl, total, unpack, mode);
    count_launch();
    return check_launch("pic_halo_pack/unpack") ? 0 : 1;
}

static int multi_launch(const pic_fab* fabs, int nfab, int dim, int ng, int mode, double* buf_lo, double* buf_hi,
                        int unpack, void* stream) {
    PIC_REQUIRE(nfab >= 1 && nfab <= HALO_MAX, "pic_halo_*_multi: 1..%d components", HALO_MAX);
    PIC_REQUIRE(dim >= 0 && dim < 3 && mode >= 0 && mode <= 2, "pic_halo_*_multi: bad arguments");
    MultiSlab m;
    m.n = nfab;
    m.off[0] = 0;
    bool overlap = false;      // the two sides' slabs share points of some component
    for (int f = 0; f < nfab; ++f) {
        const int cells = box_cells(fabs[f], dim);
        PIC_REQUIRE(ng >= 0 && ng <= fabs[f].ng[dim], "pic_halo_*_multi: ng=%d exceeds allocated guards", ng);
        PIC_REQUIRE(mode == 2 || ng <= cells, "pic_halo_*_multi: ng=%d exceeds the %d cells of the box", ng, cells);
        PIC_REQUIRE(mode != 2 || 2 * ng + fabs[f].stag[dim] <= cells,
                    "pic_halo_*_multi: the box is too thin for the fused sum + refresh (ng=%d)", ng);
        m.v[f] = make_view(fabs[f]);
        long cnt = 0;
        int first[2], count[2];
        for (int side = 0; side < 2; ++side) {
            Slab& sl = m.sl[side][f];
            full_extent(fabs[f], sl); sl.dim = dim;
            slab_range(fabs[f], dim, side, ng, mode, unpack, first[side], count[side]);
            sl.start[dim] = first[side]; sl.n[dim] = count[side];
            cnt = (long)sl.n[0] * sl.n[1] * sl.n[2];
        }
        if (count[0] > 0 && count[1] > 0 && first[0] + count[0] > first[1]) overlap = true;
        m.off[f + 1] = m.off[f] + cnt;
    }
    for (int f = nfab; f < HALO_MAX; ++f) m.off[f + 1] = m.off[nfab];
    const long total = m.off[nfab];
    if (total == 0) return 0;
    const unsigned gx = (unsigned)((total + 255) / 256);
    if (unpack && overlap) {
        // Thin boxes (SumBoundary with cells <= 2 ng + stag - 1): a point in both slabs gets the adds of both sides.
        // One launch per side, low then high, so that no two threads of a launch update the same point and the
        // order of the two adds is fixed.
        for (int side = 0; side < 2; ++side)
            multi_slab_kernel<<<dim3(gx, 1, 1), 256, 0, (cudaStream_t)stream>>>(m, buf_lo, buf_hi, unpack, mode, side);
        count_launch(2);
    } else {
        multi_slab_kernel<<<dim3(gx, 2, 1), 256, 0, (cudaStream_t)stream>>>(m, buf_lo, buf_hi, unpack, mode, 0);
        count_launch();
    }
    return check_launch("pic_halo_pack/unpack_multi") ? 0 : 1;
}

// Pack the low-side and high-side slabs of nfab components (concatenated in component order, each
// pic_halo_slab_count() doubles) into buf_lo / buf_hi with one launch; unpack likewise.
extern "C" int pic_halo_pack_multi(const pic_fab* fabs, int nfab, int dim, int ng, int mode, double* buf_lo,
                                   double* buf_hi, void* stream) {
    return multi_launch(fabs, nfab, dim, ng, mode, buf_lo, buf_hi, 0, stream);
}
extern "C" int pic_halo_unpack_multi(const pic_fab* fabs, int nfab, int dim, int ng, int mode, const double* buf_lo,
                                     const double* buf_hi, void* stream) {
    return multi_launch(fabs, nfab, dim, ng, mode, const_cast<double*>(buf_lo), const_cast<double*>(buf_hi), 1, stream);
}

extern "C" int pic_halo_pack(const pic_fab* f, int dim, int side, int ng, int mode, double* buf, void* stream) {
    return slab_launch(f, dim, side, ng, mode, buf, 0, stream);
}
extern "C" int pic_halo_unpack(const pic_fab* f, int dim, int side, int ng, int mode, const double* buf, void* stream) {
    return slab_launch(f, dim, side, ng, mode, const_cast<double*>(buf), 1, stream);
}
