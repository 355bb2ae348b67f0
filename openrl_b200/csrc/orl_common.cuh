// Shared device/host helpers for libopenrl_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "openrl_b200.h"

namespace orl {

void set_last_error(const char* fmt, ...);
int check_cuda(cudaError_t e, const char* what);
int sm_count();

#define ORL_CHECK_ARG(cond, msg)                                   \
    do {                                                           \
        if (!(cond)) {                                             \
            orl::set_last_error("%s: bad argument: %s", __func__, msg); \
            return ORL_ERR_BAD_ARG;                                \
        }                                                          \
    } while (0)

#define ORL_LAUNCH_CHECK(what) \
    do { int _e = orl::check_cuda(cudaGetLastError(), what); if (_e) return _e; } while (0)

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ValueNorm.running_mean_var (openrl/modules/utils/valuenorm.py:51-57), float32, IEEE ops
// so that the scalars equal the reference's torch-CPU values bit for bit.
struct VnScalars { float mean, std, var; };
__device__ __forceinline__ VnScalars vn_mean_std(const float* __restrict__ vn_state) {
    const float rm = vn_state[0], rms = vn_state[1], db = vn_state[2];
    const float d = fmaxf(db, 1e-5f);
    const float m = __fdiv_rn(rm, d);
    const float msq = __fdiv_rn(rms, d);
    float var = __fsub_rn(msq, __fmul_rn(m, m));
    var = fmaxf(var, 1e-2f);
    VnScalars s; s.mean = m; s.var = var; s.std = __fsqrt_rn(var);
    return s;
}

}  // namespace orl
