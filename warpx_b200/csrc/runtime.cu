// Error handling, launch accounting and version string of the C ABI.
#include "pic_common.cuh"
#include <stdarg.h>
#include <string.h>
#include <atomic>

namespace pic {

static int g_error_mode = PIC_ERR_ABORT;
static char g_last_error[1024] = "";
static std::atomic<long> g_launches{0};

// Precondition failure: WarpX aborts (WARPX_ABORT_WITH_MESSAGE -> amrex::Abort, e.g.
// Source/Particles/PhysicalParticleContainer.cpp:2564-2566); tests may ask for a return code.
int fail(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
    va_end(ap);
    if (g_error_mode == PIC_ERR_ABORT) {
        fprintf(stderr, "pic_b200::Abort: %s\n", g_last_error);
        abort();
    }
    return 1;
}

void count_launch(long n) { g_launches += n; }

bool check_launch(const char* what) {
    const cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) return true;
    fail("%s: CUDA launch failed: %s", what, cudaGetErrorString(e));
    return false;
}

}  // namespace pic

extern "C" void pic_set_error_mode(int mode) { pic::g_error_mode = mode; }
extern "C" const char* pic_last_error(void) { return pic::g_last_error; }
extern "C" const char* pic_version(void) { return "pic_b200 0.1 (sm_90a, fp64)"; }
extern "C" long pic_launch_count(void) { return pic::g_launches.load(); }
