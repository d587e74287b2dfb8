// What the binary collisions (collision.cu: pairwise Coulomb, fusion.cu: nuclear fusion) share: the reference's
// constants, the per-cell Philox random stream of their determinism contract, the amrex::min / max they restate and
// the cell-walking helpers over the two species' bins.  Args is each file's own argument block; it provides b1 (the
// bins), gn (global cells along x, y) and the species' permutations src1 / src2.
#ifndef PIC_BINARY_COLLISION_CUH_
#define PIC_BINARY_COLLISION_CUH_
#include "pic_common.cuh"
#include "bins.cuh"
#include "philox.cuh"

namespace pic {
namespace coll {

constexpr double PI = 3.14159265358979323846;      // MathConst::pi, Source/ablastr/constant.H
constexpr double HBAR = 1.054571817e-34;            // PhysConst::hbar
constexpr double DBL_MIN_ = 2.2250738585072014e-308;  // std::numeric_limits<double>::min()
constexpr double TWO_M53 = 1.0 / 9007199254740992.0;

// one random stream: consecutive 64-bit words of the blocks j = 0, 1, ... of counter (j + 1, c1, c2, c3)
struct Stream {
    uint64_t seed, c1, c2, c3, block;
    uint64_t w0, w1, w2, w3;
    int left;
    __host__ __device__ __forceinline__ Stream(uint64_t s, uint64_t a, uint64_t b, uint64_t c)
        : seed(s), c1(a), c2(b), c3(c | (1ull << 63)), block(0), w0(0), w1(0), w2(0), w3(0), left(0) {}
    __host__ __device__ __forceinline__ uint64_t next() {
        if (left == 0) {
            uint64_t o[4];
            philox4x64_10_counter(seed, block + 1, c1, c2, c3, o);
            w0 = o[0]; w1 = o[1]; w2 = o[2]; w3 = o[3];
            ++block; left = 4;
        }
        const uint64_t r = w0;
        w0 = w1; w1 = w2; w2 = w3;
        --left;
        return r;
    }
    __host__ __device__ __forceinline__ double uniform() { return (double)((next() >> 11) + 1) * TWO_M53; }
    __host__ __device__ __forceinline__ int random_int(int n) { return (int)(((double)(next() >> 11) * TWO_M53) * n); }
};

__host__ __device__ __forceinline__ double dmax(double a, double b) { return (a < b) ? b : a; }   // std::max
__host__ __device__ __forceinline__ double dmin(double a, double b) { return (b < a) ? b : a; }   // std::min

template <int G> __device__ __forceinline__ void group_sync() {
    if constexpr (G == 32) __syncwarp(); else __syncthreads();
}

// global cell index of the stream counter
template <class Args>
__device__ __forceinline__ uint64_t global_cell(const Args& a, long bin) {
    int tc[3], lc[3];
    const long tv = (long)a.b1.tile[0] * a.b1.tile[1] * a.b1.tile[2];
    tile_coords(a.b1, (int)(bin / tv), tc);
    const int l = (int)(bin % tv);
    lc[0] = l % a.b1.tile[0]; lc[1] = (l / a.b1.tile[0]) % a.b1.tile[1]; lc[2] = l / (a.b1.tile[0] * a.b1.tile[1]);
    return (uint64_t)(tc[0] * a.b1.tile[0] + lc[0] + a.b1.box_lo[0]) +
        (uint64_t)a.gn[0] * ((uint64_t)(tc[1] * a.b1.tile[1] + lc[1] + a.b1.box_lo[1]) +
                             (uint64_t)a.gn[1] * (uint64_t)(tc[2] * a.b1.tile[2] + lc[2] + a.b1.box_lo[2]));
}

// storage index of slot e of the cell (species 1 at [0, n1), species 2 after)
template <class Args>
__device__ __forceinline__ int storage_index(const Args& a, int e, int n1, long cs1, long cs2) {
    const bool two = e >= n1;
    const long slot = two ? cs2 + (e - n1) : cs1 + e;
    const int* src = two ? a.src2 : a.src1;
    return src ? src[slot] : (int)slot;
}

}  // namespace coll
}  // namespace pic
#endif
