// Forward-only passes of the 64-wide MLPs on the tensor cores (wgmma, split-fp16 operands, fp32 accumulate —
// the same building blocks and accuracy class as the update kernel, orl_ppo_tc.cu / orl_tc16.cuh):
//
//   critic_values_tc_kernel : ValueNetwork.forward over a flat batch of rows (value_network.py:113-136), the
//                             (T+1)*B-row pass of OnPolicyDriver.compute_returns (onpolicy_driver.py:206-215).
//   rollout_tc_kernel       : the fused rollout (policy forward + Categorical sampling + device env.step + in-place
//                             buffer insert, onpolicy_driver.py:154-203,236-279) for single-agent device envs
//                             (CartPole-v1, GridWorldEnv): a CTA owns 128 envs for all T steps, ONE launch.
//
// CTA = 256 threads = 128 rows x 2 column halves (warps w, w+4 share rows [32(w%4), +32)).
// Per 128-row tile: fc1 (K = d <= 8, FFMA) + activation + LayerNorm-1 in registers -> n1 as fp16 hi/lo panels ->
// Z3 = n1 . W3f^T as 12 wgmma (3 split passes x K/16; warpgroup g computes rows [64g, +64)) -> fp32 staging tile in
// shared memory -> every thread reads its row's columns -> LayerNorm-3 + head in registers.  The rollout's
// per-step critical path is one row's work (no shared-memory GEMM, no cross-row shuffles): ~1/3 of the FFMA kernel's.
#include <algorithm>
#include <cstdlib>
#include <map>
#include <mutex>

#include "orl_envstep.cuh"
#include "orl_tc16.cuh"

namespace {
using namespace orl;
using namespace orl::tc;

constexpr int F_M = 128, F_NT = 256, FCW = 32;
constexpr uint32_t FPANEL = F_M * 16, FPANEL_W = H * 16;
// Z3 staging tile: 128 rows x 64 fp32, row pitch 68 floats (row-per-thread float4 reads are conflict-free)
constexpr int S_LD = 68;
constexpr uint32_t FOFF_R1H = 0, FOFF_R1L = 8 * FPANEL, FOFF_WH = 16 * FPANEL, FOFF_WL = FOFF_WH + 8 * FPANEL_W, FOFF_S = FOFF_WL + 8 * FPANEL_W,
                   FOFF_SMALL = FOFF_S + F_M * S_LD * 4;
// fp32: w1t[8][64] b1[64] b3f[64] whf[8][64] bhf[8] | xs[2][128][2] xh[8][2][128] xst[128][8]
constexpr uint32_t F_SMALL_FLOATS = 8 * H + H + H + MAX_OUT * H + MAX_OUT;
constexpr uint32_t F_XCH_FLOATS = 2 * F_M * 2 + 2 * F_M * 8 + F_M * 8;
constexpr uint32_t F_SMEM = FOFF_SMALL + 4 * (F_SMALL_FLOATS + F_XCH_FLOATS);

#define F_FOR_OUT(j) _Pragma("unroll") for (int j = 0; j < NOUT; ++j) if (NOUT != 8 || j < n)
#define F_ROWGROUP_SYNC()                                                      \
    do {                                                                       \
        switch (warp & 3) {                                                    \
            case 0: asm volatile("bar.sync 1, 64;" ::: "memory"); break;       \
            case 1: asm volatile("bar.sync 2, 64;" ::: "memory"); break;       \
            case 2: asm volatile("bar.sync 3, 64;" ::: "memory"); break;       \
            default: asm volatile("bar.sync 4, 64;" ::: "memory"); break;      \
        }                                                                      \
    } while (0)

template <int ACT>
__device__ __forceinline__ float f_act(float z, int activation_id) { return ACT == 1 ? fmaxf(z, 0.f) : act_fwd(z, activation_id); }

struct FwdCtx {
    uint8_t *R1h, *R1l;
    float *S, *w1t, *b1s, *b3f, *whf, *bhf, *xs, *xh, *xst;
    uint32_t aR1h, aR1l, aWh, aWl;
};

// carve shared memory, stage + fold the weights (fc3 matrix as split fp16); ends with a CTA barrier.
__device__ __forceinline__ FwdCtx fwd_setup(uint8_t* smem, const float* __restrict__ params, int d, int n) {
    const int tid = threadIdx.x, nt = blockDim.x;
    FwdCtx c;
    c.R1h = smem + FOFF_R1H; c.R1l = smem + FOFF_R1L;
    uint8_t* Wh = smem + FOFF_WH; uint8_t* Wl = smem + FOFF_WL;
    c.S = reinterpret_cast<float*>(smem + FOFF_S);
    c.w1t = reinterpret_cast<float*>(smem + FOFF_SMALL);
    c.b1s = c.w1t + 8 * H; c.b3f = c.b1s + H; c.whf = c.b3f + H; c.bhf = c.whf + MAX_OUT * H;
    c.xs = c.bhf + MAX_OUT; c.xh = c.xs + 2 * F_M * 2; c.xst = c.xh + 2 * F_M * 8;   // the 2-half layout of the exchange area
    const NetOffsets po = net_offsets(d, n);
    for (int i = tid; i < 8 * H; i += nt) { const int k = i / H, j = i % H; c.w1t[i] = (k < d) ? params[po.w1 + j * d + k] : 0.f; }
    for (int i = tid; i < H; i += nt) c.b1s[i] = params[po.b1 + i];
    for (int i = tid; i < H * 8; i += nt) {   // item = (panel p, row j): lanes own consecutive rows -> conflict-free 16-byte stores
        const int pnl = i / H, j = i % H;
        float w8[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) w8[c] = params[po.w3 + j * H + 8 * pnl + c] * params[po.g1 + 8 * pnl + c];
        const uint32_t off = (uint32_t)pnl * FPANEL_W + j * 16;
        split_store8(Wh + off, Wl + off, w8, 1.0f);
    }
    for (int i = tid; i < MAX_OUT * H; i += nt) { const int j = i / H, k = i % H; c.whf[i] = (j < n) ? params[po.wh + j * H + k] * params[po.g3 + k] : 0.f; }
    for (int j = tid; j < H; j += nt) {
        float s = params[po.b3 + j];
        for (int k = 0; k < H; ++k) s = fmaf(params[po.w3 + j * H + k], params[po.be1 + k], s);
        c.b3f[j] = s;
    }
    for (int j = tid; j < MAX_OUT; j += nt) {
        float s = 0.f;
        if (j < n) { s = params[po.bh + j]; for (int k = 0; k < H; ++k) s = fmaf(params[po.wh + j * H + k], params[po.be3 + k], s); }
        c.bhf[j] = s;
    }
    fence_proxy_async();
    __syncthreads();
    c.aR1h = smem_u32(c.R1h); c.aR1l = smem_u32(c.R1l); c.aWh = smem_u32(Wh); c.aWl = smem_u32(Wl);
    return c;
}

// One 128-row tile forward: x (this thread's row, zero padded) -> out[j] = head(j) incl. the folded bias, valid in
// BOTH column halves of the row.
// `overlap()` runs between the MMA issue and the wait for its completion: work that does not depend on this tile's
// result (the rollout's sampling noise) hides in the tensor-core latency.
template <int NOUT, int ACT, typename Overlap>
__device__ __forceinline__ void fwd_tile(const FwdCtx& c, const float (&x)[8], int d, int n, int activation_id,
                                         float (&out)[MAX_OUT], Overlap&& overlap) {
    const int tid = threadIdx.x, warp = tid >> 5, row = tid & 127, half = tid >> 7, cb = FCW * half;
    float n1[FCW];
#pragma unroll
    for (int q4 = 0; q4 < FCW; q4 += 4) {
        const float4 b = *reinterpret_cast<const float4*>(c.b1s + cb + q4);
        n1[q4] = b.x; n1[q4 + 1] = b.y; n1[q4 + 2] = b.z; n1[q4 + 3] = b.w;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        if (k < d) {
#pragma unroll
            for (int q4 = 0; q4 < FCW; q4 += 4) {
                const float4 wv = *reinterpret_cast<const float4*>(c.w1t + k * H + cb + q4);
                n1[q4] = fmaf(x[k], wv.x, n1[q4]); n1[q4 + 1] = fmaf(x[k], wv.y, n1[q4 + 1]);
                n1[q4 + 2] = fmaf(x[k], wv.z, n1[q4 + 2]); n1[q4 + 3] = fmaf(x[k], wv.w, n1[q4 + 3]);
            }
        }
    }
    float s = 0.f, sq = 0.f;
#pragma unroll
    for (int i = 0; i < FCW; ++i) { n1[i] = f_act<ACT>(n1[i], activation_id); s += n1[i]; sq = fmaf(n1[i], n1[i], sq); }
    {
        *reinterpret_cast<float2*>(c.xs + (half * F_M + row) * 2) = make_float2(s, sq);
        F_ROWGROUP_SYNC();
        const float2 o = *reinterpret_cast<const float2*>(c.xs + ((half ^ 1) * F_M + row) * 2);
        s += o.x; sq += o.y;
    }
    const float mu1 = s * (1.f / H);
    const float rstd1 = 1.0f / sqrtf(fmaxf(sq * (1.f / H) - mu1 * mu1, 0.f) + LN_EPS);
#pragma unroll
    for (int i = 0; i < FCW; ++i) n1[i] = (n1[i] - mu1) * rstd1;
#pragma unroll
    for (int q8 = 0; q8 < FCW; q8 += 8) {
        const uint32_t off = (uint32_t)((cb + q8) >> 3) * FPANEL + row * 16;
        split_store8(c.R1h + off, c.R1l + off, n1 + q8, 1.0f);
    }
    fence_proxy_async();
    __syncthreads();
    {   // Z3 = n1 . W3f^T: warpgroup `half` computes rows [64 half, +64)
        const uint64_t dK_A = desc_const(FPANEL, 128), dK_W = desc_const(FPANEL_W, 128);
        float z[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) z[i] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int pass = 0; pass < 3; ++pass) {
            const uint32_t aa = (pass == 0 ? c.aR1l : c.aR1h) + half * 64 * 16, bb = pass == 1 ? c.aWl : c.aWh;
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
                wgmma_f16_n64<0, 0>(z, desc_at(dK_A, aa + 2 * kk * FPANEL), desc_at(dK_W, bb + 2 * kk * FPANEL_W), (pass | kk) > 0);
        }
        wgmma_commit();
        overlap();
        wgmma_wait0();
        frag_store<64>(z, c.S + half * 64 * S_LD, S_LD);
    }
    __syncthreads();   // the staging tile is complete; the next tile's stores follow its CTA barrier in front of the MMAs
    float n3[FCW];
#pragma unroll
    for (int q4 = 0; q4 < FCW; q4 += 4) {
        const float4 v = *reinterpret_cast<const float4*>(c.S + row * S_LD + cb + q4);
        n3[q4] = v.x; n3[q4 + 1] = v.y; n3[q4 + 2] = v.z; n3[q4 + 3] = v.w;
    }
    float s3 = 0.f, q3 = 0.f;
#pragma unroll
    for (int i = 0; i < FCW; ++i) { n3[i] += c.b3f[cb + i]; s3 += n3[i]; q3 = fmaf(n3[i], n3[i], q3); }
    {
        __syncwarp();
        // slot xs is free again: every partner read of exchange 1 happened before the CTA barrier above
        *reinterpret_cast<float2*>(c.xs + (half * F_M + row) * 2) = make_float2(s3, q3);
        F_ROWGROUP_SYNC();
        const float2 o = *reinterpret_cast<const float2*>(c.xs + ((half ^ 1) * F_M + row) * 2);
        s3 += o.x; q3 += o.y;
    }
    const float mu3 = s3 * (1.f / H);
    const float rstd3 = 1.0f / sqrtf(fmaxf(q3 * (1.f / H) - mu3 * mu3, 0.f) + LN_EPS);
#pragma unroll
    for (int j = 0; j < MAX_OUT; ++j) out[j] = 0.f;
#pragma unroll
    for (int q4 = 0; q4 < FCW; q4 += 4) {
#pragma unroll
        for (int i = 0; i < 4; ++i) n3[q4 + i] = (n3[q4 + i] - mu3) * rstd3;
        F_FOR_OUT(j) {
            const float4 wv = *reinterpret_cast<const float4*>(c.whf + j * H + cb + q4);
            out[j] = fmaf(n3[q4], wv.x, fmaf(n3[q4 + 1], wv.y, fmaf(n3[q4 + 2], wv.z, fmaf(n3[q4 + 3], wv.w, out[j]))));
        }
    }
    {
        F_FOR_OUT(j) c.xh[(j * 2 + half) * F_M + row] = out[j];   // [j][half][row]: conflict-free
        F_ROWGROUP_SYNC();
        // both halves add the two partial dots in the SAME order (half 0 first), so they hold identical logits
        F_FOR_OUT(j) {
            const float p0 = c.xh[(j * 2 + 0) * F_M + row], p1 = c.xh[(j * 2 + 1) * F_M + row];
            out[j] = (p0 + p1) + c.bhf[j];
        }
    }
}

template <int ACT>
__global__ void __launch_bounds__(F_NT, 2) critic_values_tc_kernel(const float* __restrict__ params, int d, int activation_id,
                                                                   const float* __restrict__ obs, float* __restrict__ values,
                                                                   long long rows) {
    extern __shared__ __align__(1024) uint8_t smem_f[];
    const FwdCtx c = fwd_setup(smem_f, params, d, 1);
    const int tid = threadIdx.x, warp = tid >> 5, row = tid & 127, half = tid >> 7;
    const long long n_tiles = (rows + F_M - 1) / F_M;
    for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const long long r = tile * F_M + row;
        float x[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) x[k] = (r < rows && k < d) ? obs[r * d + k] : 0.f;
        float out[MAX_OUT];
        fwd_tile<1, ACT>(c, x, d, 1, activation_id, out, [] {});
        if (half == 0 && r < rows) values[r] = out[0];
        // the exchange slots are reused by the next tile: its first write follows this row group's last read only
        // through the barriers inside fwd_tile of the NEXT tile -> order them here
        F_ROWGROUP_SYNC();
    }
}

// Categorical sampling of one row from its logits (rollout tail, half 0): masks, log-softmax, argmax / multinomial rule
template <int NOUT>
__device__ __forceinline__ int sample_row(float (&logit)[MAX_OUT], int n, const float (&q)[MAX_OUT], const float* __restrict__ mask_row,
                                          bool deterministic, float& lp) {
    if (mask_row) {
#pragma unroll
        for (int j = 0; j < MAX_OUT; ++j)
            if (j < n && mask_row[j] == 0.f) logit[j] = -6e4f;
    }
#pragma unroll
    for (int j = 0; j < MAX_OUT; ++j) if (j >= n) logit[j] = 0.f;
    float nl[MAX_OUT], pr[MAX_OUT];
    log_softmax_n(logit, n, nl, pr);
    int act;
    if (deterministic) {
        act = 0;
#pragma unroll
        for (int j = 1; j < MAX_OUT; ++j) if (j < n && pr[j] > pr[act]) act = j;
    } else {
        act = sample_categorical(pr, n, q);   // argmax(probs / q): torch.multinomial's rule, as in the FFMA kernel
    }
    lp = nl[0];
#pragma unroll
    for (int j = 1; j < MAX_OUT; ++j) if (j == act) lp = nl[j];
    return act;
}

// Exp(1) noise of (step t, row): the supplied reference-order table, else Philox4x32-10 keyed by the seed
template <int NOUT>
__device__ __forceinline__ void row_noise(const OrlRolloutArgs& a, int n, size_t grow, uint64_t step, int e, float (&q)[MAX_OUT]) {
    if (a.exp_noise) {
#pragma unroll
        for (int j = 0; j < MAX_OUT; ++j) q[j] = (j < n) ? a.exp_noise[grow * n + j] : 1.f;
    } else {
        const uint2 key = make_uint2((uint32_t)a.rng_seed, (uint32_t)(a.rng_seed >> 32));
        const uint4 r0 = philox4x32_10(make_uint4((uint32_t)step, (uint32_t)(step >> 32), (uint32_t)(e + a.rng_row_offset), 0u), key);
        const uint4 r1 = philox4x32_10(make_uint4((uint32_t)step, (uint32_t)(step >> 32), (uint32_t)(e + a.rng_row_offset), 1u), key);
        const uint32_t rr[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
        for (int j = 0; j < MAX_OUT; ++j) q[j] = -logf(u32_to_unit_open(rr[j]));
    }
}

template <int ENV, int NOUT, int ACT>
__global__ void __launch_bounds__(F_NT, 1) rollout_tc_kernel(const OrlRolloutArgs a) {
    extern __shared__ __align__(1024) uint8_t smem_f[];
    const int N = a.n_envs, B = N, d = a.obs_dim;
    const int n = NOUT == 8 ? a.n_actions : NOUT;
    const FwdCtx c = fwd_setup(smem_f, a.policy_params, d, n);
    const int tid = threadIdx.x, warp = tid >> 5, row = tid & 127, half = tid >> 7;
    const int e = blockIdx.x * F_M + row;          // env == buffer row (single-agent envs)
    const bool valid = e < N;
    const uint64_t rng_base = a.rng_step_base + (a.rng_counter ? *a.rng_counter : 0ull);
    float x[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) x[k] = (valid && k < d) ? a.policy_obs[((size_t)a.t_begin * B + e) * d + k] : 0.f;
    {
        for (int t = a.t_begin; t < a.t_end; ++t) {
            float logit[MAX_OUT];
            float q[MAX_OUT];
            const size_t grow = (size_t)t * B + (valid ? e : 0);
            fwd_tile<NOUT, ACT>(c, x, d, n, a.activation_id, logit, [&] {
                if (half == 0 && valid && !a.deterministic) row_noise<NOUT>(a, n, grow, rng_base + (uint64_t)t, e, q);
            });
            if (half == 0 && valid) {
                float lp;
                const int act = sample_row<NOUT>(logit, n, q, a.action_masks ? a.action_masks + grow * n : nullptr, a.deterministic != 0, lp);
                a.actions[grow] = (float)act;
                a.action_log_probs[grow] = lp;
                // ---- env.step of this thread's env, in-place insert into slot t / t+1 ----
                EnvPtrs E{a.env_f64, a.env_u64, a.env_i32, a.env_table, a.env_table_len, a.rng_seed,
                          a.ep_return, a.ep_length, a.episode_stats, a.rng_row_offset};
                float ob[4], fin[4], reward; bool done;
                env_step_single(E, ENV, e, N, act, ob, reward, done, fin);
                const size_t o1 = (size_t)(t + 1) * B + e;
                *reinterpret_cast<float4*>(a.policy_obs + o1 * 4) = make_float4(ob[0], ob[1], ob[2], ob[3]);
                a.rewards[grow] = reward;
                a.masks[o1] = done ? 0.f : 1.f;
                a.active_masks[o1] = 1.f;   // onpolicy_driver.py:118-124 with one agent
                *reinterpret_cast<float4*>(c.xst + row * 8) = make_float4(ob[0], ob[1], ob[2], ob[3]);
            }
            F_ROWGROUP_SYNC();   // publishes the next observation to the row's other half; orders the exchange slots
            if (valid) {
                const float4 o = *reinterpret_cast<const float4*>(c.xst + row * 8);
                x[0] = o.x; x[1] = o.y; x[2] = o.z; x[3] = o.w;
            }
        }
    }
}


// ---- CartPole rollout: 4 forward threads + 2 env threads per row -----------------------------------------------------
// The rollout is a chain of T dependent steps whose length is one row's work.  The f64 CartPole physics (sin / cos and
// three dependent divides: ~250 dependent instructions) is a large share of a step when it runs after sampling, the
// policy forward most of the rest.  So:
//   * CTA = 768 threads = 128 rows x 6 groups.  Groups 0-3 (warps w, w+4, w+8, w+12 share rows [32(w%4), +32)) are the
//     column quarters of the policy forward: quarter qd owns hidden columns [16 qd, +16).  They are also the four
//     warpgroups of the fc3 GEMM: warpgroup g computes rows [64 (g % 2), +64) x columns [32 (g / 2), +32) of Z3.
//   * Groups 4 and 5 are the env.  As soon as the state of step t is known, group 4 advances the physics for action 0 and
//     draws the reset state (PCG64), group 5 advances the physics for action 1 and draws the sampling noise of step t+1 -
//     concurrently with the whole forward pass of step t - and publish the candidates through (parity double-buffered)
//     shared memory.  Quarter 0 samples.
// After sampling a step is: publish the action, one row-group barrier (192 threads), every thread picks the candidate.
// Same functions and explicitly rounded f64 operations as env_step_single -> bit-identical trajectories.
constexpr int Q_NT = 768, Q_FWD = 512, QCW = 16;
// exchange area: xs[4][128][2] | xh[8][4][128] | qn[2 parity][8][128] | act[2][128] (int) | termf[2][2][128] (int) |
//                f64: cand[2 parity][2 action][4][128]  sr[2 parity][4][128]
constexpr uint32_t Q_XCH_FLOATS = 4 * F_M * 2 + MAX_OUT * 4 * F_M + 2 * MAX_OUT * F_M + 2 * F_M + 4 * F_M;
constexpr uint32_t Q_F64 = 2 * (2 * 4 + 4) * F_M;
constexpr uint32_t Q_XCH_BYTES = 4 * Q_XCH_FLOATS + 8 * Q_F64;
constexpr uint32_t Q_SMEM = FOFF_SMALL + 4 * F_SMALL_FLOATS + Q_XCH_BYTES;
static_assert((FOFF_SMALL + 4 * F_SMALL_FLOATS + 4 * Q_XCH_FLOATS) % 8 == 0, "f64 exchange area must be 8-byte aligned");

// named barriers: 1-4 = the 4 forward warps of a row group (128 threads), 5-8 = those + the row group's two env warps
// (192), 9 = all forward threads (the CTA barrier in front of the MMA issue)
#define Q_BAR(id, count) asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory")
#define Q_ROWGROUP_SYNC() Q_BAR(1 + (warp & 3), 128)
#define Q_PUBLISH_SYNC() Q_BAR(5 + (warp & 3), 192)
#define Q_FWD_SYNC() Q_BAR(9, Q_FWD)

template <int NOUT, int ACT>
__global__ void __launch_bounds__(Q_NT, 1) rollout_cartpole_q5_kernel(const OrlRolloutArgs a) {
    extern __shared__ __align__(1024) uint8_t smem_f[];
    const int N = a.n_envs, B = N, d = 4;
    const int n = NOUT == 8 ? a.n_actions : NOUT;
    const FwdCtx c = fwd_setup(smem_f, a.policy_params, d, n);
    const int tid = threadIdx.x, warp = tid >> 5, row = tid & 127, qd = tid >> 7, cb = QCW * (qd & 3);
    float* xs = c.xs;                                   // [4][128][2]
    float* xh = xs + 4 * F_M * 2;                       // [8][4][128]
    float* qn = xh + MAX_OUT * 4 * F_M;                 // [2][8][128]
    int* act_slot = reinterpret_cast<int*>(qn + 2 * MAX_OUT * F_M);   // [2][128]
    int* termf = act_slot + 2 * F_M;                    // [2][2][128]
    double* cand = reinterpret_cast<double*>(termf + 4 * F_M);    // [2][2][4][128]
    double* srs = cand + 2 * 2 * 4 * F_M;               // [2][4][128]
    const int e = blockIdx.x * F_M + row;               // env == buffer row (single-agent env)
    const bool valid = e < N;
    const uint64_t rng_base = a.rng_step_base + (a.rng_counter ? *a.rng_counter : 0ull);
    int elapsed = valid ? a.env_i32[e] : 0;
    uint32_t it = 0;
    if (qd >= 4) {
        // ================= env groups: one action each, one step ahead of the sampling ==================================
        const int my_act = qd - 4;
        double s[4] = {0, 0, 0, 0};
        Pcg64 g; g.state = 0; g.inc = 0;
        if (valid) {
#pragma unroll
            for (int k = 0; k < 4; ++k) s[k] = a.env_f64[(size_t)k * N + e];
            if (my_act == 0) g = pcg_load(a.env_u64, e, N);
        }
        const bool draw = my_act == 1 && valid && !a.deterministic;
        if (draw) {   // noise of the first step
            float q[MAX_OUT];
            row_noise<NOUT>(a, n, (size_t)a.t_begin * B + e, rng_base + (uint64_t)a.t_begin, e, q);
#pragma unroll
            for (int j = 0; j < MAX_OUT; ++j) if (j < n) qn[j * F_M + row] = q[j];
        }
        Q_PUBLISH_SYNC();
        for (int t = a.t_begin; t < a.t_end; ++t, ++it) {
            const uint32_t pb = it & 1u;
            double cs[4] = {s[0], s[1], s[2], s[3]};
            const bool term = cartpole_dynamics(cs, my_act);
#pragma unroll
            for (int k = 0; k < 4; ++k) cand[((pb * 2 + my_act) * 4 + k) * F_M + row] = cs[k];
            termf[(pb * 2 + my_act) * F_M + row] = term ? 1 : 0;
            Pcg64 g2 = g;
            if (my_act == 0) {
                double sr[4];
                cartpole_reset(sr, g2);
#pragma unroll
                for (int k = 0; k < 4; ++k) srs[(pb * 4 + k) * F_M + row] = sr[k];
            } else if (draw && t + 1 < a.t_end) {   // noise of the next step, into the other parity
                float q[MAX_OUT];
                row_noise<NOUT>(a, n, (size_t)(t + 1) * B + e, rng_base + (uint64_t)(t + 1), e, q);
#pragma unroll
                for (int j = 0; j < MAX_OUT; ++j) if (j < n) qn[((pb ^ 1u) * MAX_OUT + j) * F_M + row] = q[j];
            }
            Q_PUBLISH_SYNC();   // candidates out, action in
            const int act = act_slot[pb * F_M + row] & 1;
            const bool terminated = termf[(pb * 2 + act) * F_M + row] != 0;
            elapsed += 1;
            const bool done = terminated || (elapsed >= 500);
            const double* src = done ? srs + (size_t)pb * 4 * F_M : cand + (size_t)(pb * 2 + act) * 4 * F_M;
#pragma unroll
            for (int k = 0; k < 4; ++k) s[k] = src[k * F_M + row];
            if (done) { elapsed = 0; g = g2; }
        }
        if (valid && my_act == 0) {
#pragma unroll
            for (int k = 0; k < 4; ++k) a.env_f64[(size_t)k * N + e] = s[k];
            a.env_i32[e] = elapsed;
            pcg_store(a.env_u64, e, N, g);
        }
    } else {
        // ================= forward quarters =================================================================================
        int len = 0;
        float ret = 0.f;
        if (valid && qd == 0) { ret = a.ep_return[e]; len = a.ep_length[e]; }
        float x[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) x[k] = valid ? a.policy_obs[((size_t)a.t_begin * B + e) * 4 + k] : 0.f;
        Q_PUBLISH_SYNC();   // the first step's noise is in place
        for (int t = a.t_begin; t < a.t_end; ++t, ++it) {
            const uint32_t pb = it & 1u;
            const size_t grow = (size_t)t * B + (valid ? e : 0);
            // ---- fc1 + activation + LayerNorm-1 over this quarter's 16 columns ----
            float n1[QCW];
#pragma unroll
            for (int q4 = 0; q4 < QCW; q4 += 4) {
                const float4 b = *reinterpret_cast<const float4*>(c.b1s + cb + q4);
                n1[q4] = b.x; n1[q4 + 1] = b.y; n1[q4 + 2] = b.z; n1[q4 + 3] = b.w;
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) {
#pragma unroll
                for (int q4 = 0; q4 < QCW; q4 += 4) {
                    const float4 wv = *reinterpret_cast<const float4*>(c.w1t + k * H + cb + q4);
                    n1[q4] = fmaf(x[k], wv.x, n1[q4]); n1[q4 + 1] = fmaf(x[k], wv.y, n1[q4 + 1]);
                    n1[q4 + 2] = fmaf(x[k], wv.z, n1[q4 + 2]); n1[q4 + 3] = fmaf(x[k], wv.w, n1[q4 + 3]);
                }
            }
            float sm = 0.f, sq = 0.f;
#pragma unroll
            for (int i = 0; i < QCW; ++i) { n1[i] = f_act<ACT>(n1[i], a.activation_id); sm += n1[i]; sq = fmaf(n1[i], n1[i], sq); }
            *reinterpret_cast<float2*>(xs + (qd * F_M + row) * 2) = make_float2(sm, sq);
            Q_ROWGROUP_SYNC();
            {   // all quarters add the four partials in the same order -> identical statistics
                sm = 0.f; sq = 0.f;
#pragma unroll
                for (int p = 0; p < 4; ++p) { const float2 o = *reinterpret_cast<const float2*>(xs + (p * F_M + row) * 2); sm += o.x; sq += o.y; }
            }
            const float mu1 = sm * (1.f / H);
            const float rstd1 = 1.0f / sqrtf(fmaxf(sq * (1.f / H) - mu1 * mu1, 0.f) + LN_EPS);
#pragma unroll
            for (int i = 0; i < QCW; ++i) n1[i] = (n1[i] - mu1) * rstd1;
#pragma unroll
            for (int q8 = 0; q8 < QCW; q8 += 8) {
                const uint32_t off = (uint32_t)((cb + q8) >> 3) * FPANEL + row * 16;
                split_store8(c.R1h + off, c.R1l + off, n1 + q8, 1.0f);
            }
            fence_proxy_async();
            Q_FWD_SYNC();
            {   // Z3 = n1 . W3f^T: warpgroup qd computes rows [64 (qd & 1), +64) x columns [32 (qd >> 1), +32)
                const uint64_t dK_A = desc_const(FPANEL, 128), dK_W = desc_const(FPANEL_W, 128);
                const int mb = qd & 1, nb = qd >> 1;
                float z[16];
#pragma unroll
                for (int i = 0; i < 16; ++i) z[i] = 0.f;
                wgmma_fence();
#pragma unroll
                for (int pass = 0; pass < 3; ++pass) {
                    const uint32_t aa = (pass == 0 ? c.aR1l : c.aR1h) + mb * 64 * 16, bb = (pass == 1 ? c.aWl : c.aWh) + nb * 32 * 16;
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk)
                        wgmma_f16_n32<0, 0>(z, desc_at(dK_A, aa + 2 * kk * FPANEL), desc_at(dK_W, bb + 2 * kk * FPANEL_W), (pass | kk) > 0);
                }
                wgmma_commit();
                wgmma_wait0();
                frag_store<32>(z, c.S + mb * 64 * S_LD + 32 * nb, S_LD);
            }
            Q_FWD_SYNC();   // the staging tile is complete; the next step's stores follow its forward barrier in front of the MMAs
            float n3[QCW];
#pragma unroll
            for (int q4 = 0; q4 < QCW; q4 += 4) {
                const float4 v = *reinterpret_cast<const float4*>(c.S + row * S_LD + cb + q4);
                n3[q4] = v.x; n3[q4 + 1] = v.y; n3[q4 + 2] = v.z; n3[q4 + 3] = v.w;
            }
            float s3 = 0.f, q3 = 0.f;
#pragma unroll
            for (int i = 0; i < QCW; ++i) { n3[i] += c.b3f[cb + i]; s3 += n3[i]; q3 = fmaf(n3[i], n3[i], q3); }
            __syncwarp();
            // slot xs is free again: every partner read of exchange 1 happened before the forward barrier above
            *reinterpret_cast<float2*>(xs + (qd * F_M + row) * 2) = make_float2(s3, q3);
            Q_ROWGROUP_SYNC();
            {
                s3 = 0.f; q3 = 0.f;
#pragma unroll
                for (int p = 0; p < 4; ++p) { const float2 o = *reinterpret_cast<const float2*>(xs + (p * F_M + row) * 2); s3 += o.x; q3 += o.y; }
            }
            const float mu3 = s3 * (1.f / H);
            const float rstd3 = 1.0f / sqrtf(fmaxf(q3 * (1.f / H) - mu3 * mu3, 0.f) + LN_EPS);
            float out[MAX_OUT];
#pragma unroll
            for (int j = 0; j < MAX_OUT; ++j) out[j] = 0.f;
#pragma unroll
            for (int q4 = 0; q4 < QCW; q4 += 4) {
#pragma unroll
                for (int i = 0; i < 4; ++i) n3[q4 + i] = (n3[q4 + i] - mu3) * rstd3;
                F_FOR_OUT(j) {
                    const float4 wv = *reinterpret_cast<const float4*>(c.whf + j * H + cb + q4);
                    out[j] = fmaf(n3[q4], wv.x, fmaf(n3[q4 + 1], wv.y, fmaf(n3[q4 + 2], wv.z, fmaf(n3[q4 + 3], wv.w, out[j]))));
                }
            }
            F_FOR_OUT(j) xh[(j * 4 + qd) * F_M + row] = out[j];   // [j][quarter][row]: conflict-free
            Q_ROWGROUP_SYNC();
            // ---- quarter 0: logits, sampling, action outputs ----
            if (qd == 0) {
                int act = 0;
                if (valid) {
                    float logit[MAX_OUT], q[MAX_OUT];
#pragma unroll
                    for (int j = 0; j < MAX_OUT; ++j) { logit[j] = 0.f; q[j] = 1.f; }
                    F_FOR_OUT(j) {
                        logit[j] = ((xh[(j * 4 + 0) * F_M + row] + xh[(j * 4 + 1) * F_M + row]) + (xh[(j * 4 + 2) * F_M + row] + xh[(j * 4 + 3) * F_M + row])) + c.bhf[j];
                        if (!a.deterministic) q[j] = qn[(pb * MAX_OUT + j) * F_M + row];
                    }
                    float lp;
                    act = sample_row<NOUT>(logit, n, q, a.action_masks ? a.action_masks + grow * n : nullptr, a.deterministic != 0, lp);
                    a.actions[grow] = (float)act;
                    a.action_log_probs[grow] = lp;
                }
                act_slot[pb * F_M + row] = act;
            }
            Q_PUBLISH_SYNC();   // action out, candidates in; orders every exchange slot against the next step's writes
            // ---- commit env.step (sync_venv.py:213-218 auto-reset): every thread of the row picks the same candidate ----
            const int act = act_slot[pb * F_M + row] & 1;
            const bool terminated = termf[(pb * 2 + act) * F_M + row] != 0;
            elapsed += 1;
            const bool done = terminated || (elapsed >= 500);
            const double* src = done ? srs + (size_t)pb * 4 * F_M : cand + (size_t)(pb * 2 + act) * 4 * F_M;
#pragma unroll
            for (int k = 0; k < 4; ++k) x[k] = (float)src[k * F_M + row];
            if (done) elapsed = 0;
            if (qd == 0 && valid) {
                ret += 1.0f; len += 1;
                if (done) {
                    atomicAdd(a.episode_stats + 0, (double)ret);
                    atomicAdd(a.episode_stats + 1, (double)len);
                    atomicAdd(a.episode_stats + 2, 1.0);
                    ret = 0.f; len = 0;
                }
                const size_t o1 = (size_t)(t + 1) * B + e;
                *reinterpret_cast<float4*>(a.policy_obs + o1 * 4) = make_float4(x[0], x[1], x[2], x[3]);
                a.rewards[grow] = 1.0f;
                a.masks[o1] = done ? 0.f : 1.f;
                a.active_masks[o1] = 1.f;   // onpolicy_driver.py:118-124 with one agent
            }
        }
        if (valid && qd == 0) { a.ep_return[e] = ret; a.ep_length[e] = len; }
    }
}

template <typename K>
int prepare_kernel(K kern, uint32_t smem_bytes = F_SMEM) {
    static std::mutex mu;
    static std::map<const void*, bool> done;
    std::lock_guard<std::mutex> lock(mu);
    const void* key = reinterpret_cast<const void*>(kern);
    if (!done.count(key)) {
        int e = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes), "cudaFuncSetAttribute(fwd_tc)");
        if (e) return e;
        done[key] = true;
    }
    return 0;
}

}  // namespace

namespace orl {

bool fwd_tc_enabled() {
    static const bool on = [] { const char* v = getenv("ORL_FWD_FFMA"); return !(v && atoi(v) != 0); }();
    return on;
}

// ValueNetwork.forward over `rows` rows on the tensor cores; obs widths <= 8
int launch_critic_values_tc(const float* params, int d, int activation_id, const float* obs, float* values, long long rows, cudaStream_t st) {
    const long long n_tiles = (rows + F_M - 1) / F_M;
    const int grid = (int)std::min<long long>(n_tiles, 2LL * sm_count());
    if (activation_id == 1) {
        if (int e = prepare_kernel(critic_values_tc_kernel<1>)) return e;
        critic_values_tc_kernel<1><<<grid, F_NT, F_SMEM, st>>>(params, d, activation_id, obs, values, rows);
    } else {
        if (int e = prepare_kernel(critic_values_tc_kernel<-1>)) return e;
        critic_values_tc_kernel<-1><<<grid, F_NT, F_SMEM, st>>>(params, d, activation_id, obs, values, rows);
    }
    return check_cuda(cudaGetLastError(), "critic_values_tc_kernel");
}

bool rollout_tc_eligible(const OrlRolloutArgs& a) {
    return fwd_tc_enabled() && (a.env_kind == ORL_ENV_CARTPOLE || a.env_kind == ORL_ENV_GRIDWORLD) && a.n_agents == 1 && a.obs_dim == 4 &&
           a.head_kind == ORL_HEAD_CATEGORICAL && (reinterpret_cast<uintptr_t>(a.policy_obs) & 15) == 0;
}

int launch_rollout_tc(const OrlRolloutArgs& a, cudaStream_t st) {
    const int grid = (a.n_envs + F_M - 1) / F_M;
#define ORL_RTC(ENVK, NO)                                                                               \
    do {                                                                                                \
        if (a.activation_id == 1) {                                                                     \
            if (int e_ = prepare_kernel(rollout_tc_kernel<ENVK, NO, 1>)) return e_;                     \
            rollout_tc_kernel<ENVK, NO, 1><<<grid, F_NT, F_SMEM, st>>>(a);                              \
        } else {                                                                                        \
            if (int e_ = prepare_kernel(rollout_tc_kernel<ENVK, NO, -1>)) return e_;                    \
            rollout_tc_kernel<ENVK, NO, -1><<<grid, F_NT, F_SMEM, st>>>(a);                             \
        }                                                                                               \
    } while (0)
    static const bool q5 = [] { const char* v = getenv("ORL_ROLLOUT_Q5"); return !(v && atoi(v) == 0); }();
    if (a.env_kind == ORL_ENV_CARTPOLE && q5) {
        if (a.activation_id == 1) {
            if (int e_ = prepare_kernel(rollout_cartpole_q5_kernel<2, 1>, Q_SMEM)) return e_;
            rollout_cartpole_q5_kernel<2, 1><<<grid, Q_NT, Q_SMEM, st>>>(a);
        } else {
            if (int e_ = prepare_kernel(rollout_cartpole_q5_kernel<2, -1>, Q_SMEM)) return e_;
            rollout_cartpole_q5_kernel<2, -1><<<grid, Q_NT, Q_SMEM, st>>>(a);
        }
    } else if (a.env_kind == ORL_ENV_CARTPOLE) ORL_RTC(ORL_ENV_CARTPOLE, 2);
    else ORL_RTC(ORL_ENV_GRIDWORLD, 5);
#undef ORL_RTC
    return check_cuda(cudaGetLastError(), "rollout_tc_kernel");
}

}  // namespace orl
