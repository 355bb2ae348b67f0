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
// advances the device Philox step counter of the action noise by the `steps` steps a rollout launch consumed; no-op
// when `counter` is null
int bump_rng_counter(uint64_t* counter, int steps, cudaStream_t st);
// lets `kernel` take up to `smem_bytes` of dynamic shared memory on the current device, once per (kernel, device);
// `max_carveout` also asks for the largest shared-memory carveout (best effort).  Thread-safe.
int allow_dynamic_smem(const void* kernel, size_t smem_bytes, bool max_carveout = false);
template <typename K>
int allow_dynamic_smem(K* kernel, size_t smem_bytes, bool max_carveout = false) {
    return allow_dynamic_smem(reinterpret_cast<const void*>(kernel), smem_bytes, max_carveout);
}

// ---- tape-gradient reductions of the recurrent and shared-model updates (orl_tape.cu) ----
// A job reads columns of the `tape_width`-float tape rows: a gemm job writes sum_rows tape[p_off + m] * tape[q_off + k]
// (m < M, k < N) to grads[out_off + m*N + k], a column job sum_rows tape[p_off + m] (m < M) to grads[out_off + m].
struct TapeJob { int p_off, M, q_off, N, out_off; };
constexpr int TAPE_MAX_GEMM_JOBS = 6, TAPE_MAX_COL_JOBS = 15;   // the shared model's tables with a Gaussian head (the GRU's: 5 and 11)
struct TapeJobs { TapeJob gemm[TAPE_MAX_GEMM_JOBS]; TapeJob col[TAPE_MAX_COL_JOBS]; int n_gemm, n_col; };
constexpr int TAPE_ROW_BLOCK = 1024;   // tape rows per partial result: partials hold ceil(rows / TAPE_ROW_BLOCK) x stride floats
// grads[0, total) = the jobs over tape rows [0, rows), summed per row block into partials and then over the row blocks
// in a fixed order (deterministic).  ORL_ERR_BAD_ARG when a gemm job's tiles are not 16-byte aligned (tape_width, p_off,
// q_off multiples of 4) or leave the tape row (q_off + 64, p_off + 16*ceil(M/16)), or M > 192, N > 64, or tape_width
// is neither the GRU's nor the shared model's.
int reduce_tape(const float* tape, int tape_width, long long rows, const TapeJobs& jobs, float* partials, int stride, int total,
                float* grads, cudaStream_t st);

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
