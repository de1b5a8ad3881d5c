// api.cu -- error plumbing shared by every entry point of libgraphgan_b200.
#include <stdarg.h>
#include <string.h>

#include "gg_common.cuh"

namespace gg {
namespace {
thread_local char g_err[512] = "";
}

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int check_cuda(cudaError_t e, const char *what) {
    if (e == cudaSuccess) return 0;
    set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
    return 1;
}

int sm_count() {
    static int cached = 0;
    if (cached == 0) {
        int dev = 0, n = 0;
        if (cudaGetDevice(&dev) != cudaSuccess ||
            cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
            n = 132;  // H100 SXM
        cached = n;
    }
    return cached;
}
}  // namespace gg

extern "C" const char *gg_last_error(void) { return gg::g_err; }
extern "C" int gg_abi_version(void) { return GG_ABI_VERSION; }
