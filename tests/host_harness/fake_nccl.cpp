// TEST INFRASTRUCTURE -- an in-process stand-in for the eight NCCL entry points the step driver binds at run time
// (warpx_b200/csrc/comm.cu), for the test-suite: the "ranks" are THREADS of one process, each driving its own engine
// instance, and exchange through mailboxes.
// Semantics kept: messages between a pair of ranks arrive in the order they were sent; sends are buffered, receives
// posted inside a group complete at ncclGroupEnd (outside a group, immediately); ncclAllReduce(max / sum) over all
// ranks of the communicator.  Select with PIC_NCCL_LIBRARY=<this library>.
//
// Two builds of this file (tests/host_harness/harness.py):
//   build_fake_nccl()    buffers are host memory: the ranks run the host library (SIMT emulator);
//   build_device_nccl()  -DPIC_STANDIN_DEVICE: buffers are device memory, the ranks run the real library on one GPU,
//                        each on its own stream.  A send waits for the work queued on its stream, then copies the
//                        buffer to a host message; a completed receive / all-reduce copies into the device buffer on
//                        the rank's stream and waits for it.  The driver API (cuMemcpyAsync: unified addressing infers
//                        the direction; cuStreamSynchronize) is bound at run time from libcuda.so.1, so that no second
//                        CUDA runtime is loaded next to the application's.  Nothing here makes the device wait for
//                        another rank: a message that never comes is an error code after PATIENCE, never a GPU hang.
// Both builds count their calls (standin_sends / standin_recvs / standin_allreduces), so that a test can prove the
// stand-in -- and not a real NCCL -- was bound.
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstring>
#include <deque>
#include <map>
#include <mutex>
#include <vector>
#ifdef PIC_STANDIN_DEVICE
#include <dlfcn.h>
#endif

namespace {
struct Message { std::vector<char> data; };
struct World {
    std::mutex mu;
    std::condition_variable cv;
    std::map<std::pair<int, int>, std::deque<Message>> box;     // (src, dst) -> FIFO
    // all-reduce rendezvous
    int arrived = 0, departed = 0;
    unsigned long generation = 0;
    std::vector<char> acc;
};
std::mutex g_mu;
std::map<std::vector<char>, World*> g_worlds;                   // by unique id
int g_next_id = 1;
std::atomic<long> g_sends{0}, g_recvs{0}, g_allreduces{0};

struct Comm { World* w; int nranks, rank; };
struct PendingRecv { void* p; size_t bytes; int peer; Comm* c; void* stream; };
thread_local int t_group = 0;
thread_local std::vector<PendingRecv> t_pending;

size_t dtype_bytes(int dt) { return dt == 2 ? 4 : dt == 8 ? 8 : dt == 7 ? 4 : 1; }   // int32, float64, float32

// a peer that died (a failed assertion in its thread) must not hang the test-suite: give up after two minutes
constexpr std::chrono::seconds PATIENCE(120);
// error codes (NCCL's numbering): a CUDA call failed / a peer did not answer
constexpr int ERR_CUDA = 1, ERR_PEER = 6;

#ifdef PIC_STANDIN_DEVICE
// the three driver entry points, bound once (CUresult = int, CUdeviceptr = unsigned long long, CUstream = void*)
struct Driver {
    int (*memcpy_async)(unsigned long long dst, unsigned long long src, size_t bytes, void* stream) = nullptr;
    int (*stream_sync)(void* stream) = nullptr;
    int (*ctx_current)(void** ctx) = nullptr;
};
const Driver* driver() {
    static const Driver* d = [] {
        void* h = dlopen("libcuda.so.1", RTLD_NOW | RTLD_NOLOAD);
        if (!h) h = dlopen("libcuda.so.1", RTLD_NOW);
        if (!h) return (const Driver*)nullptr;
        Driver* x = new Driver();
        *(void**)&x->memcpy_async = dlsym(h, "cuMemcpyAsync");
        *(void**)&x->stream_sync = dlsym(h, "cuStreamSynchronize");
        *(void**)&x->ctx_current = dlsym(h, "cuCtxGetCurrent");
        if (!x->memcpy_async || !x->stream_sync || !x->ctx_current) return (const Driver*)nullptr;
        return (const Driver*)x;
    }();
    return d;
}
// the driver, when this thread has a current context
const Driver* ready() {
    const Driver* d = driver();
    void* ctx = nullptr;
    if (!d || d->ctx_current(&ctx) != 0 || !ctx) return nullptr;
    return d;
}
// device buffer -> host, after everything queued on the stream (the buffer's producer) has run
int load(void* host, const void* buf, size_t bytes, void* stream) {
    const Driver* d = ready();
    if (!d || d->stream_sync(stream) != 0) return ERR_CUDA;
    if (bytes == 0) return 0;
    if (d->memcpy_async((unsigned long long)host, (unsigned long long)buf, bytes, stream) != 0) return ERR_CUDA;
    return d->stream_sync(stream) != 0 ? ERR_CUDA : 0;
}
// host -> device buffer, ordered on the stream and finished on return
int store(void* buf, const void* host, size_t bytes, void* stream) {
    const Driver* d = ready();
    if (!d) return ERR_CUDA;
    if (bytes == 0) return 0;
    if (d->memcpy_async((unsigned long long)buf, (unsigned long long)host, bytes, stream) != 0) return ERR_CUDA;
    return d->stream_sync(stream) != 0 ? ERR_CUDA : 0;
}
#else
int load(void* host, const void* buf, size_t bytes, void*) { std::memcpy(host, buf, bytes); return 0; }
int store(void* buf, const void* host, size_t bytes, void*) { std::memcpy(buf, host, bytes); return 0; }
#endif

int complete(const PendingRecv& r) {
    World* w = r.c->w;
    Message m;
    {
        std::unique_lock<std::mutex> lk(w->mu);
        auto& q = w->box[{r.peer, r.c->rank}];
        if (!w->cv.wait_for(lk, PATIENCE, [&] { return !q.empty(); })) return ERR_PEER;
        m = std::move(q.front());
        q.pop_front();
    }
    return store(r.p, m.data.data(), std::min(r.bytes, m.data.size()), r.stream);
}
}  // namespace

extern "C" {
struct FakeId { char internal[128]; };

int ncclGetUniqueId(FakeId* id) {
    std::lock_guard<std::mutex> lk(g_mu);
    std::memset(id->internal, 0, 128);
    std::memcpy(id->internal, &g_next_id, sizeof(int));
    ++g_next_id;
    return 0;
}
int ncclCommInitRank(void** comm, int nranks, FakeId id, int rank) {
    std::lock_guard<std::mutex> lk(g_mu);
    std::vector<char> key(id.internal, id.internal + 128);
    World*& w = g_worlds[key];
    if (!w) w = new World();
    *comm = new Comm{w, nranks, rank};
    return 0;
}
int ncclCommDestroy(void* comm) { delete static_cast<Comm*>(comm); return 0; }
int ncclGroupStart() { ++t_group; return 0; }
int ncclGroupEnd() {
    if (--t_group == 0) {
        std::vector<PendingRecv> todo;
        todo.swap(t_pending);
        int rc = 0;
        for (const auto& r : todo) if (int e = complete(r)) rc = e;
        return rc;
    }
    return 0;
}
int ncclSend(const void* p, size_t count, int dtype, int peer, void* comm, void* stream) {
    Comm* c = static_cast<Comm*>(comm);
    Message m;
    m.data.resize(count * dtype_bytes(dtype));
    if (int rc = load(m.data.data(), p, m.data.size(), stream)) return rc;
    {
        std::lock_guard<std::mutex> lk(c->w->mu);
        c->w->box[{c->rank, peer}].push_back(std::move(m));
    }
    c->w->cv.notify_all();
    ++g_sends;
    return 0;
}
int ncclRecv(void* p, size_t count, int dtype, int peer, void* comm, void* stream) {
    PendingRecv r{p, count * dtype_bytes(dtype), peer, static_cast<Comm*>(comm), stream};
    ++g_recvs;
    if (t_group > 0) { t_pending.push_back(r); return 0; }
    return complete(r);
}
int ncclAllReduce(const void* in, void* out, size_t count, int dtype, int op, void* comm, void* stream) {
    Comm* c = static_cast<Comm*>(comm);
    World* w = c->w;
    const size_t bytes = count * dtype_bytes(dtype);
    std::vector<char> mine(bytes), result(bytes);
    if (int rc = load(mine.data(), in, bytes, stream)) return rc;
    {
        std::unique_lock<std::mutex> lk(w->mu);
        if (!w->cv.wait_for(lk, PATIENCE, [&] { return w->departed == 0 || w->arrived > 0; })) return ERR_PEER;   // previous round fully drained
        const unsigned long gen = w->generation;
        if (w->arrived == 0) w->acc = mine;
        else
            for (size_t i = 0; i < count; ++i) {
                if (dtype == 2) { int* a = reinterpret_cast<int*>(w->acc.data()); const int v = reinterpret_cast<const int*>(mine.data())[i];
                                  a[i] = op == 2 ? (v > a[i] ? v : a[i]) : a[i] + v; }
                else { double* a = reinterpret_cast<double*>(w->acc.data()); const double v = reinterpret_cast<const double*>(mine.data())[i];
                       a[i] = op == 2 ? (v > a[i] ? v : a[i]) : a[i] + v; }
            }
        if (++w->arrived == c->nranks) { w->departed = c->nranks; w->arrived = 0; ++w->generation; w->cv.notify_all(); }
        else if (!w->cv.wait_for(lk, PATIENCE, [&] { return w->generation != gen; })) return ERR_PEER;
        std::memcpy(result.data(), w->acc.data(), bytes);
        if (--w->departed == 0) w->cv.notify_all();
    }
    ++g_allreduces;
    return store(out, result.data(), bytes, stream);
}
const char* ncclGetErrorString(int rc) {
    return rc == ERR_CUDA ? "stand-in NCCL: a CUDA driver call failed (or the thread has no current context)"
                          : "stand-in NCCL: a peer did not answer";
}

long standin_sends() { return g_sends.load(); }
long standin_recvs() { return g_recvs.load(); }
long standin_allreduces() { return g_allreduces.load(); }
}
