// Godfrey's numerical-Cherenkov corrector (particles.use_fdtd_nci_corr): a 5-point filter along z applied
// to a COPY of E and B that the field gather reads instead of the fields themselves.
//
// Replaces (paths relative to Source/ of ECP-WarpX/WarpX):
//   pic_nci_godfrey_table_index / pic_nci_godfrey_stencil
//        <- NCIGodfreyFilter::ComputeStencils                      Filter/NCIGodfreyFilter.cpp:49-139
//   pic_apply_nci_filter
//        <- PhysicalParticleContainer::applyNCIFilter              Particles/PhysicalParticleContainer.cpp:2097-2169
//           -> Filter::ApplyStencil(FArrayBox) -> Filter::DoFilter Filter/Filter.cpp:78-133 with slen = {1,1,5}
// The coefficient tables (Utils/NCIGodfreyTables.H) are fitted data of the reference and stay with the
// caller: a WarpX build hands over the two stencils it already holds (m_stencil_2 of
// nci_godfrey_filter_exeybz / _bxbyez), a stand-alone run passes the two table lines around c dt / dz.
//
// One thread per destination point, i fastest: 9 source planes per point, all but one served by L2
// (the planes of a 256^2 face are 0.5 MB each), 16 B/point of HBM traffic.  The eight mirrored reads of
// DoFilter are summed in the reference's order (on the device the final multiply-add may contract to an FMA).
// The body is __host__ __device__ (harness_launch.cuh) and is compared with the oracle on the host.
#include "pic_common.cuh"
#include "harness_launch.cuh"

namespace pic {

struct NciArgs {
    FabView S, D;
    int lo[3], n[3];                 // destination region (index space of the component)
    int slo[3], shi[3];              // allocated range of the source (zero padding beyond it)
    double sz[5];                    // m_stencil_2: coefficient 0 already halved
    long total;
};

PIC_HD void nci_body(long t, const NciArgs& a) {
    const int i = a.lo[0] + (int)(t % a.n[0]);
    const int j = a.lo[1] + (int)((t / a.n[0]) % a.n[1]);
    const int k = a.lo[2] + (int)(t / ((long)a.n[0] * a.n[1]));
    const bool in_ij = i >= a.slo[0] && i <= a.shi[0] && j >= a.slo[1] && j <= a.shi[1];
    double d = 0.0;
    for (int i2 = 0; i2 < 5; ++i2) {
        // s0[0] * s1[0] * s2[i2] with s0 = s1 = {1/2} (NCIGodfreyFilter.cpp:113-129)
        const double sss = 0.5 * 0.5 * a.sz[i2];
        const int km = k - i2, kp = k + i2;
        const double m = (in_ij && km >= a.slo[2] && km <= a.shi[2]) ? a.S.p[a.S.off(i, j, km)] : 0.0;   // src_zeropad, Filter.cpp:103-107
        const double p = (in_ij && kp >= a.slo[2] && kp <= a.shi[2]) ? a.S.p[a.S.off(i, j, kp)] : 0.0;
        d += sss * (m + m + m + m + p + p + p + p);                                                       // :112-119 (i0 = i1 = 0)
    }
    a.D.p[a.D.off(i, j, k)] = d;
}
__global__ void nci_kernel(NciArgs a) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < a.total) nci_body(t, a);
}

}  // namespace pic

using namespace pic;

extern "C" int pic_nci_godfrey_table_index(double cdtodz, int tab_length) {
    int index = static_cast<int>(tab_length * cdtodz);
    index = index < tab_length - 2 ? index : tab_length - 2;
    index = index > 0 ? index : 0;
    return index;
}

extern "C" void pic_nci_godfrey_stencil(const double line_lo[4], const double line_hi[4], int index, int tab_length,
                                        double cdtodz, double stencil_z[5]) {
    const double weight_right = cdtodz - double(index) / double(tab_length);
    double pre[4];
    for (int i = 0; i < 4; ++i) pre[i] = (1.0 - weight_right) * line_lo[i] + weight_right * line_hi[i];
    stencil_z[0] =  (256 + 128 * pre[0] + 96 * pre[1] + 80 * pre[2] + 70 * pre[3]) / 256;
    stencil_z[1] = -(       64 * pre[0] + 64 * pre[1] + 60 * pre[2] + 56 * pre[3]) / 256;
    stencil_z[2] =  (                     16 * pre[1] + 24 * pre[2] + 28 * pre[3]) / 256;
    stencil_z[3] = -(                                    4 * pre[2] +  8 * pre[3]) / 256;
    stencil_z[4] =  (                                                  1 * pre[3]) / 256;
    stencil_z[0] /= 2.0;             // "Due to the way Filter::DoFilter() is written, coefficient 0 has to be /2"
}

extern "C" int pic_apply_nci_filter(const pic_fab* src, const pic_fab* dst, const double stencil_z[5],
                                    const int tile_lo[3], const int tile_hi[3], int grow, void* stream) {
    PIC_REQUIRE(src && dst && src->p && dst->p && src->p != dst->p, "pic_apply_nci_filter: src and dst must be two different arrays");
    NciArgs a;
    a.S = make_view(*src); a.D = make_view(*dst);
    a.total = 1;
    for (int d = 0; d < 3; ++d) {
        PIC_REQUIRE(src->stag[d] == dst->stag[d], "pic_apply_nci_filter: staggering mismatch");
        a.lo[d] = tile_lo[d] - grow;                                   // amrex::grow(box, nox), converted to the index type
        const int hi = tile_hi[d] + grow + dst->stag[d];
        PIC_REQUIRE(a.lo[d] >= dst->lo[d] && hi <= dst->hi[d], "pic_apply_nci_filter: the grown tile box leaves the destination array along %d", d);
        a.n[d] = hi - a.lo[d] + 1;
        PIC_REQUIRE(a.n[d] > 0, "pic_apply_nci_filter: empty tile box");
        a.slo[d] = src->lo[d]; a.shi[d] = src->hi[d];
        a.total *= a.n[d];
    }
    for (int i = 0; i < 5; ++i) a.sz[i] = stencil_z[i];
    PIC_LAUNCH(nci_kernel, nci_body, a, a.total, stream);
    return launched_ok("pic_apply_nci_filter") ? 0 : 1;
}
