// Forward-only passes of the 64-wide MLPs on the tensor cores (wgmma, split-fp16 operands, fp32 accumulate —
// the same building blocks and accuracy class as the update kernel, orl_ppo_tc.cu / orl_tc16.cuh):
//
//   critic_values_tc_kernel : ValueNetwork.forward over a flat batch of rows (value_network.py:113-136), the
//                             (T+1)*B-row pass of OnPolicyDriver.compute_returns (onpolicy_driver.py:206-215).
//   rollout_tc_kernel       : the fused rollout (policy forward + Categorical sampling + device env.step + in-place
//                             buffer insert, onpolicy_driver.py:154-203,236-279) for GridWorldEnv: a CTA owns 128 envs
//                             for all T steps, ONE launch.
//   rollout_cartpole_rows_kernel : the same for CartPole-v1 with 32 envs per CTA and the physics one step ahead
//                             (layout below, before the kernel).
//
// critic_values_tc_kernel and rollout_tc_kernel: CTA = 256 threads = 128 rows x 2 column halves, in the update kernel's
// layout (orl_tc16.cuh): warp w owns rows [16w, +16), the two halves of a row are lanes l and l ^ 16.
// Per 128-row tile: fc1 (K = d <= 8, FFMA) + activation + LayerNorm-1 in registers -> n1 as fp16 hi/lo panels ->
// Z3 = n1 . W3f^T as 12 wgmma (3 split passes x K/16; warpgroup g computes rows [64g, +64)) -> fp32 staging tile in
// shared memory, read back by the warp that owns the rows -> LayerNorm-3 + head in registers.  Both pass through the
// row functions of orl_tc16.cuh, which the update and the CartPole rollout use as well.  The rollout's per-step critical
// path is one row's work (no shared-memory GEMM, no cross-row shuffles): ~1/3 of the FFMA kernel's.
#include <algorithm>

#include "orl_envstep.cuh"
#include "orl_tc16.cuh"

namespace {
using namespace orl;
using namespace orl::tc;

constexpr int F_M = 128, F_NT = 256, FCW = 32;
// shared-memory carve of a forward kernel: n1 hi/lo panels of M1 rows | W3f hi/lo panels | staging tile of MS rows | small
template <int M1, int MS>
struct FwdLayout {
    static constexpr uint32_t PANEL = M1 * 16, R1H = 0, R1L = 8 * PANEL, WH = 16 * PANEL, WL = WH + 8 * W_PANEL, S = WL + 8 * W_PANEL,
                              SMALL = S + MS * S_LD * 4;
};
using FLay = FwdLayout<F_M, F_M>;
constexpr uint32_t FPANEL = FLay::PANEL;
// fp32: w1t[8][64] b1[64] b3f[64] whf[8][64] bhf[8]
constexpr uint32_t F_SMALL_FLOATS = 8 * H + H + H + MAX_OUT * H + MAX_OUT;
constexpr uint32_t F_SMEM = FLay::SMALL + 4 * F_SMALL_FLOATS;

struct FwdCtx {
    uint8_t *R1h, *R1l;
    float *S, *w1t, *b1s, *b3f, *whf, *bhf;
    uint32_t aR1h, aR1l, aWh, aWl;
};

// carve shared memory, stage + fold the weights (fc3 matrix as split fp16); ends with a CTA barrier.
template <typename L = FLay>
__device__ __forceinline__ FwdCtx fwd_setup(uint8_t* smem, const float* __restrict__ params, int d, int n) {
    FwdCtx c;
    c.R1h = smem + L::R1H; c.R1l = smem + L::R1L;
    uint8_t* Wh = smem + L::WH; uint8_t* Wl = smem + L::WL;
    c.S = reinterpret_cast<float*>(smem + L::S);
    c.w1t = reinterpret_cast<float*>(smem + L::SMALL);
    c.b1s = c.w1t + 8 * H; c.b3f = c.b1s + H; c.whf = c.b3f + H; c.bhf = c.whf + MAX_OUT * H;
    stage_weights_tc(c.w1t, Wh, Wl, params, d, n, blockDim.x);
    fence_proxy_async();
    __syncthreads();
    c.aR1h = smem_u32(c.R1h); c.aR1l = smem_u32(c.R1l); c.aWh = smem_u32(Wh); c.aWl = smem_u32(Wl);
    return c;
}

// One 128-row tile forward: x (this thread's row, zero padded) -> out[j] = head(j) incl. the folded bias, valid in
// BOTH column halves of the row.  Every hand-off is inside the warp or the warpgroup: the n1 rows a warpgroup's MMA
// reads are its own, and the staging-tile rows a warp reads are those of its own accumulator fragment.  A warp
// rewrites its n1 rows (next tile) only after its wgmma_wait has seen the MMA that read them complete.
// `overlap()` runs between the MMA issue and the wait for its completion: work that does not depend on this tile's
// result (the rollout's sampling noise) hides in the tensor-core latency.
template <int NOUT, int ACT, typename Overlap>
__device__ __forceinline__ void fwd_tile(const FwdCtx& c, const float (&x)[8], int d, int n, int activation_id,
                                         float (&out)[MAX_OUT], Overlap&& overlap) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, row = 16 * warp + (lane & 15), wg = warp >> 2, cb = FCW * (lane >> 4);
    float n1[FCW], s, sq;
    row_fc1<FCW, ACT>(x, d, c.w1t, c.b1s, cb, activation_id, n1, s, sq);
    row_sum_stats<FCW>(s, sq);
    row_ln1_store<FCW>(n1, ln_stats(s, sq), c.R1h, c.R1l, FPANEL, row, cb);
    fence_proxy_async();
    warpgroup_sync(wg);   // the MMA reads this warpgroup's rows of n1
    {   // Z3 = n1 . W3f^T: warpgroup wg computes rows [64 wg, +64)
        const uint64_t dK_A = desc_const(FPANEL, 128), dK_W = desc_const(W_PANEL, 128);
        float z[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) z[i] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int pass = 0; pass < 3; ++pass) {
            const uint32_t aa = (pass == 0 ? c.aR1l : c.aR1h) + wg * 64 * 16, bb = pass == 1 ? c.aWl : c.aWh;
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
                wgmma_f16_n64<0, 0>(z, desc_at(dK_A, aa + 2 * kk * FPANEL), desc_at(dK_W, bb + 2 * kk * W_PANEL), (pass | kk) > 0);
        }
        wgmma_commit();
        overlap();
        wgmma_wait<0>();
        frag_store<64>(z, c.S + wg * 64 * S_LD, S_LD);
    }
    __syncwarp();   // rows [16 warp, +16) of the staging tile: written and read by this warp
    float n3[FCW], s3, q3;
    row_z3<FCW>(c.S, row, cb, c.b3f, n3, s3, q3);
    row_sum_stats<FCW>(s3, q3);
    row_head<FCW, NOUT>(n3, ln_stats(s3, q3), c.whf, cb, n, out);
    row_sum_head<FCW, NOUT>(out, n);
    FOR_OUT(j) out[j] += c.bhf[j];
}

template <int ACT>
__global__ void __launch_bounds__(F_NT, 2) critic_values_tc_kernel(const float* __restrict__ params, int d, int activation_id,
                                                                   const float* __restrict__ obs, float* __restrict__ values,
                                                                   long long rows) {
    extern __shared__ __align__(1024) uint8_t smem_f[];
    const FwdCtx c = fwd_setup(smem_f, params, d, 1);
    const int lane = threadIdx.x & 31, row = 16 * (threadIdx.x >> 5) + (lane & 15), half = lane >> 4;
    const long long n_tiles = (rows + F_M - 1) / F_M;
    for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const long long r = tile * F_M + row;
        float x[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) x[k] = (r < rows && k < d) ? obs[r * d + k] : 0.f;
        float out[MAX_OUT];
        fwd_tile<1, ACT>(c, x, d, 1, activation_id, out, [] {});
        if (half == 0 && r < rows) values[r] = out[0];
    }
}

template <int ACT>
__global__ void __launch_bounds__(F_NT, 1) rollout_tc_kernel(const OrlRolloutArgs a) {
    extern __shared__ __align__(1024) uint8_t smem_f[];
    constexpr int NOUT = 5;   // GridWorldEnv's actions
    const int N = a.n_envs, B = N, d = a.obs_dim, n = NOUT;
    const FwdCtx c = fwd_setup(smem_f, a.policy_params, d, n);
    const int lane = threadIdx.x & 31, row = 16 * (threadIdx.x >> 5) + (lane & 15), half = lane >> 4;
    const int e = blockIdx.x * F_M + row;          // env == buffer row (single-agent envs)
    const bool valid = e < N;
    const uint64_t rng_base = a.rng_step_base + (a.rng_counter ? *a.rng_counter : 0ull);
    float x[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) x[k] = (valid && k < d) ? a.policy_obs[((size_t)a.t_begin * B + e) * d + k] : 0.f;
    for (int t = a.t_begin; t < a.t_end; ++t) {
        float logit[MAX_OUT];
        float q[MAX_OUT];
        const size_t grow = (size_t)t * B + (valid ? e : 0);
        fwd_tile<NOUT, ACT>(c, x, d, n, a.activation_id, logit, [&] {
            if (half == 0 && valid && !a.deterministic)
                action_noise(a.exp_noise, grow, n, a.rng_seed, rng_base + (uint64_t)t, (uint32_t)(e + a.rng_row_offset), q);
        });
        float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
        if (half == 0 && valid) {
            float lp;
            const int act = sample_action(logit, n, a.action_masks ? a.action_masks + grow * n : nullptr, a.deterministic != 0,
                                          [&](float (&qs)[MAX_OUT]) { for (int j = 0; j < MAX_OUT; ++j) qs[j] = q[j]; }, lp);
            a.actions[grow] = (float)act;
            a.action_log_probs[grow] = lp;
            // ---- env.step of this thread's env, in-place insert into slot t / t+1 ----
            bool done;
            o = step_insert_single(a, env_ptrs(a, a.rng_row_offset / a.n_agents), ORL_ENV_GRIDWORLD, e, t, act, done);
        }
        // the next observation, from half 0 (lane l % 16) to both halves of the row
        o.x = __shfl_sync(0xffffffffu, o.x, lane & 15); o.y = __shfl_sync(0xffffffffu, o.y, lane & 15);
        o.z = __shfl_sync(0xffffffffu, o.z, lane & 15); o.w = __shfl_sync(0xffffffffu, o.w, lane & 15);
        if (valid) { x[0] = o.x; x[1] = o.y; x[2] = o.z; x[3] = o.w; }
    }
}

// ---- CartPole rollout: R envs per CTA, 4 forward lanes + 2 env threads per env -------------------------------------
// The rollout is a chain of T dependent steps whose length is one row's work.  The f64 CartPole physics (sin / cos and
// three dependent divides: ~250 dependent instructions) is a large share of a step when it runs after sampling, the
// policy forward most of the rest.  A CTA owns R = 32 envs, so 4096 envs spread over 128 CTAs, one per SM, and each SM
// issues the forward of 32 rows instead of 128 (DESIGN.md §6 has R = 32 against the removed R = 64):
//   * Forward: 4R threads = R rows x 4 column quarters, the 4 quarters of a row in one warp (lane = 4 row + quarter,
//     quarter qd owns hidden columns [16 qd, +16)); the row functions of orl_tc16.cuh with CW = 16, whose LayerNorm
//     and head partials meet through shuffles, added in a fixed order.  The fc3 GEMM is one M = 64 tile over R1 rows [0, 64) (rows [R, 64) zero padding): the one forward
//     warpgroup computes both 32-column halves.  Each Z3 element is the same wgmma_f16_n32 chain (Al.Bh, Ah.Bl, Ah.Bh;
//     kk = 0..3) as in the row-parallel kernels.
//   * Env: 2R threads, lane = row.  As soon as the state of step t is known, the action-0 threads advance the physics
//     for action 0 and draw the reset state (PCG64), the action-1 threads advance the physics for action 1 and draw the
//     sampling noise of step t+1 - concurrently with the whole forward pass of step t - and publish the candidates
//     through (parity double-buffered) shared memory.  Quarter 0 samples.
// Per step: one forward barrier in front of the MMA issue, one after the staging tile is written, one CTA barrier
// (publish the action, every thread picks the candidate).  Same functions and explicitly rounded f64 operations as
// env_step_single -> bit-identical trajectories.
constexpr int QCW = 16, RW_M = 64;
struct RowsCfg {
    static constexpr int R = 32, FWD = 4 * R, NT = 6 * R;
    // resident CTAs per SM the register budget is sized for: three (96 registers, no spills; four would spill), so up
    // to 3 x 32 x #SMs envs run in one wave
    static constexpr int MIN_CTAS = 3;
    using L = FwdLayout<RW_M, R>;
    // exchange area: qn[2 parity][8][R] | act[2][R] (int) | termf[2][2][R] (int) | f64: cand[2 parity][2 action][4][R]
    // srs[2 parity][4][R]
    static constexpr uint32_t XCH = L::SMALL + 4 * F_SMALL_FLOATS;
    static constexpr uint32_t XCH_F64 = XCH + 4 * (2 * MAX_OUT * R + 2 * R + 4 * R);
    static constexpr uint32_t SMEM = XCH_F64 + 8 * (2 * 2 * 4 * R + 2 * 4 * R);
    static_assert(XCH_F64 % 8 == 0, "f64 exchange area must be 8-byte aligned");
};

// named barriers: 1 = the forward threads (in front of the MMA issue, after the staging tile), 2 = the whole CTA
#define RW_FWD_SYNC() asm volatile("bar.sync 1, %0;" ::"n"(C::FWD) : "memory")
#define RW_PUBLISH_SYNC() asm volatile("bar.sync 2, %0;" ::"n"(C::NT) : "memory")

template <int ACT>
__global__ void __launch_bounds__(RowsCfg::NT, RowsCfg::MIN_CTAS) rollout_cartpole_rows_kernel(const OrlRolloutArgs a) {
    using C = RowsCfg;
    constexpr int R = C::R, NOUT = 2;   // CartPole's actions
    extern __shared__ __align__(1024) uint8_t smem_f[];
    const int N = a.n_envs, B = N, n = NOUT;
    const int tid = threadIdx.x;
    // the MMA tile's padding rows [R, 64) of the 16 n1 panels: zeroed once, never written again
    for (int i = tid; i < 16 * (RW_M - R); i += C::NT) {
        const int p = i / (RW_M - R), r = R + i % (RW_M - R);
        *reinterpret_cast<uint4*>(smem_f + C::L::R1H + p * C::L::PANEL + r * 16) = make_uint4(0u, 0u, 0u, 0u);
    }
    const FwdCtx c = fwd_setup<typename C::L>(smem_f, a.policy_params, 4, n);
    float* qn = reinterpret_cast<float*>(smem_f + C::XCH);            // [2][8][R]
    int* act_slot = reinterpret_cast<int*>(qn + 2 * MAX_OUT * R);     // [2][R]
    int* termf = act_slot + 2 * R;                                    // [2][2][R]
    double* cand = reinterpret_cast<double*>(smem_f + C::XCH_F64);    // [2][2][4][R]
    double* srs = cand + 2 * 2 * 4 * R;                               // [2][4][R]
    const uint64_t rng_base = a.rng_step_base + (a.rng_counter ? *a.rng_counter : 0ull);
    uint32_t it = 0;
    if (tid >= C::FWD) {
        // ================= env threads: one action each, one step ahead of the sampling =================================
        const int my_act = (tid - C::FWD) / R, row = (tid - C::FWD) % R;
        const int e = blockIdx.x * R + row;
        const bool valid = e < N;
        int elapsed = valid ? a.env_i32[e] : 0;
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
            action_noise(a.exp_noise, (size_t)a.t_begin * B + e, n, a.rng_seed, rng_base + (uint64_t)a.t_begin, (uint32_t)(e + a.rng_row_offset), q);
#pragma unroll
            for (int j = 0; j < MAX_OUT; ++j) if (j < n) qn[j * R + row] = q[j];
        }
        RW_PUBLISH_SYNC();
        for (int t = a.t_begin; t < a.t_end; ++t, ++it) {
            const uint32_t pb = it & 1u;
            double cs[4] = {s[0], s[1], s[2], s[3]};
            const bool term = cartpole_dynamics(cs, my_act);
#pragma unroll
            for (int k = 0; k < 4; ++k) cand[((pb * 2 + my_act) * 4 + k) * R + row] = cs[k];
            termf[(pb * 2 + my_act) * R + row] = term ? 1 : 0;
            Pcg64 g2 = g;
            if (my_act == 0) {
                double sr[4];
                cartpole_reset(sr, g2);
#pragma unroll
                for (int k = 0; k < 4; ++k) srs[(pb * 4 + k) * R + row] = sr[k];
            } else if (draw && t + 1 < a.t_end) {   // noise of the next step, into the other parity
                float q[MAX_OUT];
                action_noise(a.exp_noise, (size_t)(t + 1) * B + e, n, a.rng_seed, rng_base + (uint64_t)(t + 1), (uint32_t)(e + a.rng_row_offset), q);
#pragma unroll
                for (int j = 0; j < MAX_OUT; ++j) if (j < n) qn[((pb ^ 1u) * MAX_OUT + j) * R + row] = q[j];
            }
            RW_PUBLISH_SYNC();   // candidates out, action in
            const int act = act_slot[pb * R + row] & 1;
            const bool terminated = termf[(pb * 2 + act) * R + row] != 0;
            elapsed += 1;
            const bool done = terminated || (elapsed >= 500);
            const double* src = done ? srs + (size_t)pb * 4 * R : cand + (size_t)(pb * 2 + act) * 4 * R;
#pragma unroll
            for (int k = 0; k < 4; ++k) s[k] = src[k * R + row];
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
        const int warp = tid >> 5, row = tid >> 2, qd = tid & 3, cb = QCW * qd;
        const int e = blockIdx.x * R + row;
        const bool valid = e < N;
        int elapsed = valid ? a.env_i32[e] : 0;
        int len = 0;
        float ret = 0.f;
        if (valid && qd == 0) { ret = a.ep_return[e]; len = a.ep_length[e]; }
        float x[8];   // fc1 reads x[0, 4)
#pragma unroll
        for (int k = 0; k < 4; ++k) x[k] = valid ? a.policy_obs[((size_t)a.t_begin * B + e) * 4 + k] : 0.f;
        RW_PUBLISH_SYNC();   // the first step's noise is in place
        for (int t = a.t_begin; t < a.t_end; ++t, ++it) {
            const uint32_t pb = it & 1u;
            const size_t grow = (size_t)t * B + (valid ? e : 0);
            // ---- fc1 + activation + LayerNorm-1 over this quarter's 16 columns ----
            float n1[QCW], sm, sq;
            row_fc1<QCW, ACT>(x, 4, c.w1t, c.b1s, cb, a.activation_id, n1, sm, sq);
            row_sum_stats<QCW>(sm, sq);
            row_ln1_store<QCW>(n1, ln_stats(sm, sq), c.R1h, c.R1l, C::L::PANEL, row, cb);
            fence_proxy_async();
            RW_FWD_SYNC();
            {   // Z3 = n1 . W3f^T over R1 rows [0, 64), both 32-column halves b
                const uint64_t dK_A = desc_const(C::L::PANEL, 128), dK_W = desc_const(W_PANEL, 128);
                const int nb0 = (warp >> 2) * 2;   // 0: the forward threads are one warpgroup
                float z[2][16];
#pragma unroll
                for (int b = 0; b < 2; ++b)
#pragma unroll
                    for (int i = 0; i < 16; ++i) z[b][i] = 0.f;
                wgmma_fence();
#pragma unroll
                for (int pass = 0; pass < 3; ++pass) {
                    const uint32_t aa = pass == 0 ? c.aR1l : c.aR1h, bb = pass == 1 ? c.aWl : c.aWh;
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
                        for (int b = 0; b < 2; ++b)
                            wgmma_f16_n32<0, 0>(z[b], desc_at(dK_A, aa + 2 * kk * C::L::PANEL),
                                                desc_at(dK_W, bb + (nb0 + b) * 32 * 16 + 2 * kk * W_PANEL), (pass | kk) > 0);
                }
                wgmma_commit();
                wgmma_wait<0>();
                if (16 * (warp & 3) < R) {   // fragment rows 16 (warp % 4) + [0, 16): only real rows go to the staging tile
#pragma unroll
                    for (int b = 0; b < 2; ++b) frag_store<32>(z[b], c.S + 32 * (nb0 + b), S_LD);
                }
            }
            RW_FWD_SYNC();   // the staging tile is complete; the next step's stores follow its forward barrier in front of the MMAs
            float n3[QCW], s3, q3;
            row_z3<QCW>(c.S, row, cb, c.b3f, n3, s3, q3);
            row_sum_stats<QCW>(s3, q3);
            float logit[MAX_OUT];
            row_head<QCW, NOUT>(n3, ln_stats(s3, q3), c.whf, cb, n, logit);
            row_sum_head<QCW, NOUT>(logit, n);
            FOR_OUT(j) logit[j] += c.bhf[j];
            // ---- quarter 0: sampling, action outputs ----
            if (qd == 0) {
                int act = 0;
                if (valid) {
                    float q[MAX_OUT];
#pragma unroll
                    for (int j = 0; j < MAX_OUT; ++j) q[j] = 1.f;
                    if (!a.deterministic) { FOR_OUT(j) q[j] = qn[(pb * MAX_OUT + j) * R + row]; }
                    float lp;
                    act = sample_action(logit, n, a.action_masks ? a.action_masks + grow * n : nullptr, a.deterministic != 0,
                                        [&](float (&qs)[MAX_OUT]) { for (int j = 0; j < MAX_OUT; ++j) qs[j] = q[j]; }, lp);
                    a.actions[grow] = (float)act;
                    a.action_log_probs[grow] = lp;
                }
                act_slot[pb * R + row] = act;
            }
            RW_PUBLISH_SYNC();   // action out, candidates in; orders every exchange slot against the next step's writes
            // ---- commit env.step (sync_venv.py:213-218 auto-reset): every thread of the row picks the same candidate ----
            const int act = act_slot[pb * R + row] & 1;
            const bool terminated = termf[(pb * 2 + act) * R + row] != 0;
            elapsed += 1;
            const bool done = terminated || (elapsed >= 500);
            const double* src = done ? srs + (size_t)pb * 4 * R : cand + (size_t)(pb * 2 + act) * 4 * R;
#pragma unroll
            for (int k = 0; k < 4; ++k) x[k] = (float)src[k * R + row];
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
#undef RW_FWD_SYNC
#undef RW_PUBLISH_SYNC

}  // namespace

namespace orl {

// ValueNetwork.forward over `rows` rows on the tensor cores; obs widths <= 8
int launch_critic_values_tc(const float* params, int d, int activation_id, const float* obs, float* values, long long rows, cudaStream_t st) {
    const long long n_tiles = (rows + F_M - 1) / F_M;
    const int grid = (int)std::min<long long>(n_tiles, 2LL * sm_count());
    const auto kern = activation_id == 1 ? critic_values_tc_kernel<1> : critic_values_tc_kernel<-1>;
    if (int e = allow_dynamic_smem(kern, F_SMEM)) return e;
    kern<<<grid, F_NT, F_SMEM, st>>>(params, d, activation_id, obs, values, rows);
    return check_cuda(cudaGetLastError(), "critic_values_tc_kernel");
}

int launch_rollout_tc(const OrlRolloutArgs& a, cudaStream_t st) {
    const bool relu = a.activation_id == 1;
    if (a.env_kind == ORL_ENV_CARTPOLE) {
        const auto kern = relu ? rollout_cartpole_rows_kernel<1> : rollout_cartpole_rows_kernel<-1>;
        if (int e = allow_dynamic_smem(kern, RowsCfg::SMEM)) return e;
        kern<<<(a.n_envs + RowsCfg::R - 1) / RowsCfg::R, RowsCfg::NT, RowsCfg::SMEM, st>>>(a);
        return check_cuda(cudaGetLastError(), "rollout_cartpole_rows_kernel");
    }
    const auto kern = relu ? rollout_tc_kernel<1> : rollout_tc_kernel<-1>;
    if (int e = allow_dynamic_smem(kern, F_SMEM)) return e;
    kern<<<(a.n_envs + F_M - 1) / F_M, F_NT, F_SMEM, st>>>(a);
    return check_cuda(cudaGetLastError(), "rollout_tc_kernel");
}

}  // namespace orl
