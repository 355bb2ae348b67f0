// Parameter gradients of the recurrent (orl_rnn.cu) and shared-model (orl_share.cu) updates as reductions of their
// per-row tapes, deterministic, in two stages:
// Stage 1: every CTA owns TAPE_ROW_BLOCK tape rows and one job and writes its partial result to partials[row_block][...]:
//   gemm job   part[out_off + m*N + k] = sum_rows tape[r][p_off+m] * tape[r][q_off+k]     (register-tiled, 12x4 per thread)
//   column job part[out_off + m]       = sum_rows tape[r][p_off+m]
// Stage 2: grads[i] = sum over row blocks of partials[rb][i], pairwise in a fixed order.
// The kernels are built per tape width (the GRU's, the wide-head GRU policy's and the DiagGaussian GRU policy's, each with
// or without the X field of a wide observation, and the shared model's): with the width a runtime value the gemm
// kernel's row addressing takes 92 registers instead of 80 on sm_90a, one CTA less per SM.
#include "orl_common.cuh"
#include "orl_deep_core.h"
#include "orl_rnn_warp.cuh"
#include "orl_tc16.cuh"

namespace {
using namespace orl;

// 16 x 16 threads; thread tile (M/16) x 4.  P tiles are TR_MAX_M columns wide, Q tiles TR_N.
constexpr int TR_NT = 256, TR_ROWS = TAPE_ROW_BLOCK, TR_SUB = 32, TR_MAX_M = 192, TR_N = 64, TR_MI = TR_MAX_M / 16;
constexpr size_t TR_SMEM = 2 * (size_t)TR_SUB * (TR_MAX_M + TR_N) * sizeof(float);   // two stages of P and Q tiles

template <int TAPE_W>
__global__ void __launch_bounds__(TR_NT) tape_gemm_kernel(const float* __restrict__ tape, long long rows, TapeJobs jobs,
                                                          float* __restrict__ partials, int stride) {
    extern __shared__ __align__(16) float tsm[];
    const TapeJob jb = jobs.gemm[blockIdx.y];
    const long long r_begin = (long long)blockIdx.x * TR_ROWS;
    const int rows_here = (int)min((long long)TR_ROWS, rows - r_begin);
    auto Ps = [&](int buf) { return tsm + buf * (TR_SUB * TR_MAX_M); };
    auto Qs = [&](int buf) { return tsm + 2 * TR_SUB * TR_MAX_M + buf * (TR_SUB * TR_N); };
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int MI = (jb.M + 15) >> 4, Mq = MI * 4;   // P columns are read in whole float4 up to 16*MI (fields are zero / foreign beyond M: discarded)
    // stage loader: rows beyond the block's tail are zero-filled
    auto load_stage = [&](int buf, int s0) {
        const int sub = min(TR_SUB, rows_here - s0);
        const float* base = tape + (size_t)(r_begin + s0) * TAPE_W;
        for (int i = tid; i < TR_SUB * Mq; i += TR_NT) {
            const int r = i / Mq, c = i % Mq;
            tc::cp_async16(Ps(buf) + r * TR_MAX_M + 4 * c, base + (size_t)(r < sub ? r : 0) * TAPE_W + jb.p_off + 4 * c, r < sub);
        }
        for (int i = tid; i < TR_SUB * (TR_N / 4); i += TR_NT) {
            const int r = i >> 4, c = i & 15;
            tc::cp_async16(Qs(buf) + r * TR_N + 4 * c, base + (size_t)(r < sub ? r : 0) * TAPE_W + jb.q_off + 4 * c, r < sub);
        }
        asm volatile("cp.async.commit_group;\n" ::);
    };
    float acc[TR_MI][4];
#pragma unroll
    for (int i = 0; i < TR_MI; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }
    const int n_sub = (rows_here + TR_SUB - 1) / TR_SUB;
    load_stage(0, 0);
    for (int s = 0; s < n_sub; ++s) {
        const int buf = s & 1;
        if (s + 1 < n_sub) { load_stage(buf ^ 1, (s + 1) * TR_SUB); asm volatile("cp.async.wait_group 1;\n" ::); }
        else asm volatile("cp.async.wait_group 0;\n" ::);
        __syncthreads();
        const float* P = Ps(buf);
        const float* Q = Qs(buf);
#pragma unroll 4
        for (int r = 0; r < TR_SUB; ++r) {
            const float4 q = *reinterpret_cast<const float4*>(Q + r * TR_N + 4 * tx);
#pragma unroll
            for (int i = 0; i < TR_MI; ++i) {
                if (i < MI) {
                    const float p = P[r * TR_MAX_M + ty + 16 * i];
                    acc[i][0] = fmaf(p, q.x, acc[i][0]); acc[i][1] = fmaf(p, q.y, acc[i][1]);
                    acc[i][2] = fmaf(p, q.z, acc[i][2]); acc[i][3] = fmaf(p, q.w, acc[i][3]);
                }
            }
        }
        __syncthreads();   // the stage just read is refilled by the next iteration's load
    }
    float* part = partials + (size_t)blockIdx.x * stride + jb.out_off;
#pragma unroll
    for (int i = 0; i < TR_MI; ++i) {
        const int m = ty + 16 * i;
        if (i < MI && m < jb.M) {
#pragma unroll
            for (int c = 0; c < 4; ++c) { const int k = 4 * tx + c; if (k < jb.N) part[m * jb.N + k] = acc[i][c]; }
        }
    }
}

template <int TAPE_W>
__global__ void __launch_bounds__(TR_MAX_M) tape_colsum_kernel(const float* __restrict__ tape, long long rows, TapeJobs jobs,
                                                               float* __restrict__ partials, int stride) {
    const TapeJob jb = jobs.col[blockIdx.y];
    const long long r_begin = (long long)blockIdx.x * TR_ROWS;
    const int rows_here = (int)min((long long)TR_ROWS, rows - r_begin);
    const int m = threadIdx.x;
    if (m >= jb.M) return;
    const float* p = tape + (size_t)r_begin * TAPE_W + jb.p_off + m;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    int r = 0;
    for (; r + 4 <= rows_here; r += 4) {
        s0 += p[(size_t)r * TAPE_W]; s1 += p[(size_t)(r + 1) * TAPE_W];
        s2 += p[(size_t)(r + 2) * TAPE_W]; s3 += p[(size_t)(r + 3) * TAPE_W];
    }
    for (; r < rows_here; ++r) s0 += p[(size_t)r * TAPE_W];
    partials[(size_t)blockIdx.x * stride + jb.out_off + m] = (s0 + s1) + (s2 + s3);
}

// Pairwise in a fixed order (deterministic): partial rb joins the pending sums as a binary counter carries, so the
// rounding error grows with log2(row_blocks), not with row_blocks as in one running sum (whose nearly equal addends
// round alike against the growing total: 1.4e-6 relative on a C2 bias gradient over 512 blocks).  Up to three row
// blocks the order is the running sum's.
__global__ void row_block_sum_kernel(const float* __restrict__ partials, int row_blocks, int stride, int total,
                                     float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    float pend[32];   // pend[d]: the sum of the last complete run of 2^k partials, k decreasing with d
    int depth = 0;
    for (int rb = 0; rb < row_blocks; ++rb) {
        float v = partials[(size_t)rb * stride + i];
        for (int c = rb; c & 1; c >>= 1) v = pend[--depth] + v;
        pend[depth++] = v;
    }
    float s = pend[--depth];
    while (depth > 0) s = pend[--depth] + s;
    out[i] = 0.f + s;   // as the running sum from 0 does: -0 becomes +0
}

// the tile loads of tape_gemm_kernel: 16-byte cp.async of whole float4 (aligned offsets), a Q tile of TR_N columns
// and a P tile of 16*ceil(M/16) columns, all inside the tape row
bool jobs_fit(const TapeJobs& jobs, int tape_width) {
    if (tape_width % 4 != 0 || jobs.n_gemm < 0 || jobs.n_gemm > TAPE_MAX_GEMM_JOBS || jobs.n_col < 0 || jobs.n_col > TAPE_MAX_COL_JOBS ||
        jobs.n_gemm + jobs.n_col < 1)
        return false;
    for (int j = 0; j < jobs.n_gemm; ++j) {
        const TapeJob& g = jobs.gemm[j];
        if (g.p_off < 0 || g.p_off % 4 != 0 || g.q_off < 0 || g.q_off % 4 != 0 || g.M < 1 || g.M > TR_MAX_M || g.N < 1 || g.N > TR_N ||
            g.q_off + TR_N > tape_width || g.p_off + 16 * ((g.M + 15) / 16) > tape_width)
            return false;
    }
    for (int j = 0; j < jobs.n_col; ++j) {
        const TapeJob& c = jobs.col[j];
        if (c.p_off < 0 || c.M < 1 || c.M > TR_MAX_M || c.p_off + c.M > tape_width) return false;
    }
    return true;
}

template <int TAPE_W>
int launch_jobs(const float* tape, long long rows, const TapeJobs& jobs, float* partials, int stride, int rb, cudaStream_t st) {
    if (jobs.n_gemm > 0) {
        if (int e = allow_dynamic_smem(tape_gemm_kernel<TAPE_W>, TR_SMEM)) return e;
        tape_gemm_kernel<TAPE_W><<<dim3(rb, jobs.n_gemm), TR_NT, TR_SMEM, st>>>(tape, rows, jobs, partials, stride);
    }
    if (jobs.n_col > 0) tape_colsum_kernel<TAPE_W><<<dim3(rb, jobs.n_col), TR_MAX_M, 0, st>>>(tape, rows, jobs, partials, stride);
    return 0;
}

}  // namespace

namespace orl {

int reduce_tape(const float* tape, int tape_width, long long rows, const TapeJobs& jobs, float* partials, int stride, int total,
                float* grads, cudaStream_t st) {
    ORL_CHECK_ARG(tape && partials && grads && rows > 0 && total > 0 && stride >= total, "tape / partials / grads");
    ORL_CHECK_ARG(jobs_fit(jobs, tape_width), "tape job layout (16-byte aligned tiles inside the tape row, M <= 192, N <= 64)");
    const int rb = (int)((rows + TR_ROWS - 1) / TR_ROWS);
    int e = 0;
    switch (tape_width) {
        case orl_rnnw::TAPE_W: e = launch_jobs<orl_rnnw::TAPE_W>(tape, rows, jobs, partials, stride, rb, st); break;
        case orl_rnnw::TAPE_WIDE: e = launch_jobs<orl_rnnw::TAPE_WIDE>(tape, rows, jobs, partials, stride, rb, st); break;
        case orl_rnnw::TAPE_W + orl_rnnw::MAXD_WIDE:   // the GRU's rows with the X field of a wide observation
            e = launch_jobs<orl_rnnw::TAPE_W + orl_rnnw::MAXD_WIDE>(tape, rows, jobs, partials, stride, rb, st); break;
        case orl_rnnw::TAPE_WIDE + orl_rnnw::MAXD_WIDE:
            e = launch_jobs<orl_rnnw::TAPE_WIDE + orl_rnnw::MAXD_WIDE>(tape, rows, jobs, partials, stride, rb, st); break;
        case orl_rnnw::TAPE_GAUSS: e = launch_jobs<orl_rnnw::TAPE_GAUSS>(tape, rows, jobs, partials, stride, rb, st); break;
        case orl_rnnw::TAPE_GAUSS + orl_rnnw::MAXD_WIDE:   // a DiagGaussian GRU policy's rows with the X field
            e = launch_jobs<orl_rnnw::TAPE_GAUSS + orl_rnnw::MAXD_WIDE>(tape, rows, jobs, partials, stride, rb, st); break;
        case orl_deep::TAPE: e = launch_jobs<orl_deep::TAPE>(tape, rows, jobs, partials, stride, rb, st); break;
        case orl_deep::TAPE_GAUSSIAN: e = launch_jobs<orl_deep::TAPE_GAUSSIAN>(tape, rows, jobs, partials, stride, rb, st); break;
        default: ORL_CHECK_ARG(false, "tape_width (one of the GRU's or the shared model's tapes)");
    }
    if (e) return e;
    row_block_sum_kernel<<<(total + 255) / 256, 256, 0, st>>>(partials, rb, stride, total, grads);
    return check_cuda(cudaGetLastError(), "tape reduction launches");
}

}  // namespace orl
