// Launch helper of the thin kernels (lwfa.cu, charge.cu): a kernel is a __host__ __device__ body taking
// the linear thread id and a POD argument block.  Product build: PIC_LAUNCH launches the __global__
// wrapper on the stream.  With -DPIC_HOST_HARNESS (tests/host_harness only) the same bodies run in a host
// loop over the same thread ids, so that the CPU test-suite can compare bodies and argument builders with
// the oracle where no GPU exists; the product library is never built that way.
#ifndef PIC_HARNESS_LAUNCH_CUH_
#define PIC_HARNESS_LAUNCH_CUH_
#include "pic_common.cuh"
#include <cstring>

namespace pic {

#ifndef PIC_HD
#define PIC_HD __host__ __device__ __forceinline__
#endif

#ifdef PIC_HOST_HARNESS
#define PIC_LAUNCH(kernel, body, args, total, stream) \
    do { for (long t_ = 0; t_ < (total); ++t_) body(t_, args); } while (0)
static inline void dev_copy(void* dst, const void* src, size_t bytes, void*) { memcpy(dst, src, bytes); }
static inline void dev_zero(void* dst, size_t bytes, void*) { memset(dst, 0, bytes); }
static inline bool launched_ok(const char*) { return true; }
static inline void* dev_alloc(size_t bytes) { return malloc(bytes ? bytes : 1); }
static inline void dev_free(void* p) { free(p); }
static inline bool copy_sync(void* dst, const void* src, size_t bytes, void*) { memcpy(dst, src, bytes); return true; }
#else
#define PIC_LAUNCH(kernel, body, args, total, stream) \
    do { if ((total) > 0) { kernel<<<(unsigned)(((total) + 255) / 256), 256, 0, (cudaStream_t)(stream)>>>(args); count_launch(); } } while (0)
static inline void dev_copy(void* dst, const void* src, size_t bytes, void* s) {
    cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)s);
}
static inline void dev_zero(void* dst, size_t bytes, void* s) { cudaMemsetAsync(dst, 0, bytes, (cudaStream_t)s); }
static inline bool launched_ok(const char* what) { return check_launch(what); }
// Scratch for the duration of one call (initial conditions only, never on the step path)
static inline void* dev_alloc(size_t bytes) {
    void* p = nullptr;
    return cudaMalloc(&p, bytes ? bytes : 1) == cudaSuccess ? p : nullptr;
}
static inline void dev_free(void* p) { cudaFree(p); }
// Host <-> device copy on the stream, then wait for it (the caller needs the data now)
static inline bool copy_sync(void* dst, const void* src, size_t bytes, void* s) {
    return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, (cudaStream_t)s) == cudaSuccess &&
           cudaStreamSynchronize((cudaStream_t)s) == cudaSuccess;
}
#endif

PIC_HD int slot_add(int* c) {
#ifdef __CUDA_ARCH__
    return atomicAdd(c, 1);
#else
    return (*c)++;
#endif
}
PIC_HD void real_add(double* p, double v) {
#ifdef __CUDA_ARCH__
    atomicAdd(p, v);
#else
    *p += v;
#endif
}

}  // namespace pic
#endif
