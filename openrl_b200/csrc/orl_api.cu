// Library-level C-ABI entry points: version, error string, device query; the rollouts' noise-counter bump; the kernels'
// dynamic shared-memory opt-in.
#include <stdarg.h>
#include <string.h>

#include <map>
#include <mutex>

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

__global__ void bump_rng_counter_kernel(uint64_t* c, uint64_t by) { *c += by; }

int bump_rng_counter(uint64_t* counter, int steps, cudaStream_t st) {
    if (!counter) return 0;
    bump_rng_counter_kernel<<<1, 1, 0, st>>>(counter, (uint64_t)steps);
    return check_cuda(cudaGetLastError(), "bump_rng_counter_kernel");
}

// the attribute belongs to the (kernel, device) pair: a process that launches on several devices opts in on each
int allow_dynamic_smem(const void* kernel, size_t smem_bytes, bool max_carveout) {
    static std::mutex mu;
    static std::map<std::pair<const void*, int>, size_t> allowed;
    int dev = 0;
    if (int e = check_cuda(cudaGetDevice(&dev), "cudaGetDevice")) return e;
    std::lock_guard<std::mutex> lock(mu);
    size_t& have = allowed[{kernel, dev}];
    if (have >= smem_bytes) return 0;
    if (int e = check_cuda(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes),
                           "cudaFuncSetAttribute(MaxDynamicSharedMemorySize)"))
        return e;
    if (max_carveout) cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    have = smem_bytes;
    return 0;
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
