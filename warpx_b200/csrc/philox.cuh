// Philox4x64-10 of Random123 (Salmon et al., SC'11): 10 rounds, multipliers M0/M1, Weyl key increments W0/W1.
// The project's replacement of AMReX's per-thread random stream: a draw is a pure function of (key, counter), so every
// decomposition, thread mapping and the numpy restatements see the same numbers.  The counter (c0, c1, c2, c3) and key
// (k0, k1) follow numpy.random.Philox: numpy's block after advance(j) with counter (0, 0, 0, 0) is c = (j + 1, 0, 0, 0).
#ifndef PIC_PHILOX_CUH_
#define PIC_PHILOX_CUH_
#include <stdint.h>

namespace pic {

__host__ __device__ __forceinline__ uint64_t mulhi64(uint64_t a, uint64_t b) {
#ifdef __CUDA_ARCH__
    return __umul64hi(a, b);
#else
    return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}

__host__ __device__ __forceinline__ void philox4x64_10_counter(uint64_t k0, uint64_t c0, uint64_t c1, uint64_t c2,
                                                              uint64_t c3, uint64_t out[4]) {
    const uint64_t M0 = 0xD2E7470EE14C6C93ull, M1 = 0xCA5A826395121157ull;
    const uint64_t W0 = 0x9E3779B97F4A7C15ull, W1 = 0xBB67AE8584CAA73Bull;
    uint64_t k1 = 0;
    for (int r = 0; r < 10; ++r) {
        if (r > 0) { k0 += W0; k1 += W1; }
        const uint64_t hi0 = mulhi64(M0, c0), lo0 = M0 * c0;
        const uint64_t hi1 = mulhi64(M1, c2), lo1 = M1 * c2;
        const uint64_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// Block `block` of the stream keyed by seed: counter (block + 1, 0, 0, 0), key (seed, 0).
__host__ __device__ __forceinline__ void philox4x64_10(uint64_t seed, uint64_t block, uint64_t out[4]) {
    philox4x64_10_counter(seed, block + 1, 0, 0, 0, out);
}

}  // namespace pic
#endif
