// Run-time binding of the few NCCL entry points the step driver uses (see comm.cu).
// The declarations restate NCCL's public C API (nccl.h: ncclUniqueId :37-38, ncclCommInitRank :160,
// ncclAllReduce :392, ncclSend :442, ncclRecv :461, ncclDataType_t / ncclRedOp_t :260-286 of 2.27).
#ifndef PIC_COMM_CUH_
#define PIC_COMM_CUH_
#include <cuda_runtime.h>
#include <cstddef>

namespace pic {

struct PicNcclUniqueId { char internal[128]; };
typedef struct ncclComm* PicNcclComm;
constexpr int PIC_NCCL_INT32 = 2, PIC_NCCL_FLOAT64 = 8;   // ncclDataType_t
constexpr int PIC_NCCL_SUM = 0, PIC_NCCL_MAX = 2;          // ncclRedOp_t

struct NcclApi {
    bool loaded = false;
    int (*GetUniqueId)(PicNcclUniqueId*) = nullptr;
    int (*CommInitRank)(PicNcclComm*, int, PicNcclUniqueId, int) = nullptr;
    int (*CommDestroy)(PicNcclComm) = nullptr;
    int (*Send)(const void*, size_t, int, int, PicNcclComm, cudaStream_t) = nullptr;
    int (*Recv)(void*, size_t, int, int, PicNcclComm, cudaStream_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, PicNcclComm, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};
extern NcclApi g_nccl;
bool nccl_load();
int nccl_fail(const char* what, int rc);

struct Comm {
    PicNcclComm comm;
    int nranks, rank;
};

}  // namespace pic
#endif
