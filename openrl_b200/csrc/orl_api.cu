// Library-level C-ABI entry points: version, error string, device query.
#include <stdarg.h>
#include <string.h>

#include "orl_common.cuh"

namespace orl {
static thread_local char g_err[512] = "";

void set_last_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int check_cuda(cudaError_t e, const char* what) {
    if (e == cudaSuccess) return 0;
    set_last_error("%s: %s (%s)", what, cudaGetErrorString(e), cudaGetErrorName(e));
    return (int)e;
}

int sm_count() {
    static int cached[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (cached[dev] == 0) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        cached[dev] = n;
    }
    return cached[dev];
}
}  // namespace orl

extern "C" {

int orl_abi_version(void) { return ORL_ABI_VERSION; }

const char* orl_last_error(void) { return orl::g_err; }

int orl_device_sm_count(int* sm_count_out) {
    if (!sm_count_out) return ORL_ERR_BAD_ARG;
    int dev = 0;
    int e = orl::check_cuda(cudaGetDevice(&dev), "cudaGetDevice");
    if (e) return e;
    int n = 0;
    e = orl::check_cuda(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev), "cudaDeviceGetAttribute");
    if (e) return e;
    *sm_count_out = n;
    return 0;
}

}  // extern "C"
