// Recurrent (GRU) policy / value networks: rollout, critic pass, chunked-BPTT update, optimizer.
//
// Replaces, for cfg.use_recurrent_policy:
//   RNNLayer.forward                      openrl/modules/networks/utils/rnn.py:39-99
//   OnPolicyDriver.act / add2buffer       openrl/drivers/onpolicy_driver.py:80-152,236-279 (rnn-state carry,
//                                         zeroing on dones_env; for host-stepped envs the act is orl_rnn_act_rows
//                                         and the zeroing orl_host_insert_rnn)
//   ReplayData.recurrent_generator        openrl/buffers/replay_data.py:1062-1258 (chunks of L over f=(n*A+a)*T+t)
//   ReplayData.recurrent_generator_v3     openrl/buffers/replay_data.py:425-551 (JRPO: chunks of L over f=n*T+t, all agents)
//   PPOAlgorithm.ppo_update (BPTT part)   openrl/algorithms/ppo.py:46-458
//
// Design (DESIGN.md "recurrent path"): ONE WARP per env (rollout), per row (critic) or per chunk (update) running
// the warp-cooperative step of orl_rnn_warp.cuh — 64-vectors as two registers per lane, the net's weights staged
// once per persistent CTA in 136 KB of shared memory, mat-vecs by shuffle broadcast (shared-memory-bandwidth
// bound: one LDS per FMA).  The update writes a per-row-step tape (forward activations, local gradients);
// parameter gradients are reductions of the tape, dW = sum_rows P^T Q, by the deterministic two-stage reduction of
// orl_tape.cu.  The sequential restatement of the same step (orl_rnn_core.h, pinned to the torch oracle on the CPU)
// is compiled for the host only: the g++ reference of the CPU tests and the element-wise checker of the warp path
// (tests/debug_gru.py).
#include <algorithm>

#include "orl_adam.cuh"
#include "orl_envstep.cuh"
#include "orl_rnn_core.h"
#include "orl_rnn_warp.cuh"

namespace {
using namespace orl;
namespace rc = orl_rnn;
namespace rw = orl_rnnw;

static_assert(rc::MAXN == MAX_OUT && rw::MAXN == MAX_OUT && rw::MAXN_WIDE == MAX_OUT_WIDE, "head width limits must agree");
constexpr int LMAX = 32;     // data_chunk_length limit accepted by the host API (the chunk kernels loop over l; the tape is n_chunks * L rows)
constexpr int JOINT_A = 3;   // agents of the joint-action update (simple_spread, the multi-agent device env)

constexpr int W_NT = 512, W_WPC = W_NT / 32;   // one persistent CTA per SM, 16 warps, weights of one net in smem

// ---- rollout: one warp per env advances its A agent rows together; env.step on lane 0 ----
template <int ENV>
__global__ void __launch_bounds__(W_NT, 1) rnn_rollout_warp_kernel(const OrlRnnArgs a) {
    extern __shared__ __align__(16) float smem[];
    constexpr int A = ENV == ORL_ENV_MPE_SPREAD ? 3 : 1;
    constexpr int D = ENV == ORL_ENV_MPE_SPREAD ? 18 : 4;
    const int N = a.n_envs, B = N * A, n = a.n_actions;
    const rc::Offsets o = rc::rnn_offsets(D, n);
    const rw::SmemNet W = rw::load_net(smem, a.policy_params, o, threadIdx.x, W_NT);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* scr = smem + rw::smem_net_floats(D) + warp * A * rw::SCR;
    const EnvPtrs E = env_ptrs(a, 0);   // the env randomness is keyed by the launch's env index, like the action noise
    const uint64_t rng_base = a.rng_step_base + (a.rng_counter ? *a.rng_counter : 0ull);
    float* const no_tape[A] = {};
    for (int e = blockIdx.x * W_WPC + warp; e < N; e += gridDim.x * W_WPC) {
        for (int t = a.t_begin; t < a.t_end; ++t) {
            rw::V2 x[A], h[A], hn[A];
            float mk[A], logit[A][MAX_OUT];
            int acts[A];
#pragma unroll
            for (int ag = 0; ag < A; ++ag) {
                const size_t grow = (size_t)t * B + e * A + ag;
                const float* ob = a.policy_obs + grow * D;
                x[ag] = rw::V2{lane < D ? ob[lane] : 0.f, lane + 32 < D ? ob[lane + 32] : 0.f};
                h[ag] = rw::ldv(a.rnn_states + grow * rc::H, lane);
                mk[ag] = a.masks[grow];
            }
            rw::step_forward<A>(W, scr, D, n, a.activation_id, x, h, mk, hn, logit, no_tape, lane);
#pragma unroll
            for (int ag = 0; ag < A; ++ag) {
                const int row = e * A + ag;
                const size_t grow = (size_t)t * B + row;
                float lp;
                const int act = sample_action(logit[ag], n, nullptr, a.deterministic != 0, [&](float (&q)[MAX_OUT]) {   // identical on every lane
                    action_noise(a.exp_noise, grow, n, a.rng_seed, rng_base + (uint64_t)t, (uint32_t)row, q);
                }, lp);
                if (lane == 0) { a.actions[grow] = (float)act; a.action_log_probs[grow] = lp; }
                acts[ag] = act;
            }
            int done_i = 0;
            if (lane == 0) {
                bool done;
                if constexpr (ENV == ORL_ENV_MPE_SPREAD) {
                    done = step_insert_mpe(a, E, e, t, acts);
                } else {
                    step_insert_single(a, E, ENV, e, t, acts[0], done);
                }
                done_i = done ? 1 : 0;
            }
            done_i = __shfl_sync(0xffffffffu, done_i, 0);
#pragma unroll
            for (int ag = 0; ag < A; ++ag) {   // rnn_states[dones_env] = 0 (onpolicy_driver.py:262-269)
                const size_t r1 = (size_t)(t + 1) * B + (size_t)e * A + ag;
                rw::stv(a.rnn_states + r1 * rc::H, lane, done_i ? rw::V2{0.f, 0.f} : hn[ag]);
            }
            __syncwarp();   // lane 0's observation / mask writes are read by the whole warp in the next step
        }
    }
}

// ---- the wide head (NB = 64) of one row, on the lane-owned logits x of step_forward<R, 64> ----
// sample_action of a wide row: the first-max mode when deterministic, else argmax(probs / q) with the first index winning
// ties; q of action j is noise(j) (identical for a given j on every lane).  Returns the action on every lane.
template <typename Noise>
__device__ __forceinline__ int warp_sample_action(rw::V2 x, int n, const float* mask_row, bool deterministic, Noise&& noise,
                                                  float& lp, int lane) {
    const rw::WarpSoftmax sm = rw::warp_log_softmax(x, n, mask_row, lane);
    rw::V2 v{sm.in_a ? sm.pr(x.a) : 0.f, sm.in_b ? sm.pr(x.b) : 0.f};
    if (!deterministic) {
        if (sm.in_a) v.a = v.a / noise(lane);
        if (sm.in_b) v.b = v.b / noise(lane + 32);
    }
    const int act = rw::warp_argmax(v, sm.in_a, sm.in_b, lane);
    lp = sm.nl(rw::warp_pick(x, act));
    return act;
}
// Exp(1) noise of action j of a wide row: draw j % 4 of wide_action_noise4 (Philox lanes 0, 1 for actions 0..7, 8..21 beyond)
__device__ __forceinline__ float wide_action_noise1(const float* exp_noise, size_t grow, int n, uint64_t seed, uint64_t step,
                                                    uint32_t row, int j) {
    float q[4];
    wide_action_noise4(exp_noise, grow, n, seed, step, row, j & ~3, q);
    const int c = j & 3;
    return c == 0 ? q[0] : c == 1 ? q[1] : c == 2 ? q[2] : q[3];
}
// categorical_row of a wide row (the maths and masking of wide_categorical_row): masks x in place, then overwrites it with
// dL/dlogits (0 for the masked-out actions and for j >= n)
template <class Args>
__device__ __forceinline__ CatRow warp_categorical_row(const Args& a, rw::V2& x, int n, const float* mask_row, int act, float old_lp,
                                                       float adv, float wrow, int lane) {
    const rw::WarpSoftmax sm = rw::warp_log_softmax(x, n, mask_row, lane);
    const PgTerm pg = pg_term(sm.nl(rw::warp_pick(x, (act >= 0 && act < n) ? act : 0)), old_lp, adv, a.clip_param, a.flags,
                              a.dual_clip_coeff);
    const float pa = sm.pr(x.a), pb = sm.pr(x.b), nla = sm.nl(x.a), nlb = sm.nl(x.b);
    const float ent = -warp_sum((sm.in_a ? pa * nla : 0.f) + (sm.in_b ? pb * nlb : 0.f));
    const float dlp = pg.dlogp * wrow, went = a.entropy_coef * wrow;
    x.a = sm.live_a ? dlp * ((lane == act ? 1.f : 0.f) - pa) + went * pa * (nla + ent) : 0.f;
    x.b = sm.live_b ? dlp * ((lane + 32 == act ? 1.f : 0.f) - pb) + went * pb * (nlb + ent) : 0.f;
    return CatRow{pg.loss, ent, pg.ratio};
}
// gaussian_row of a wide row (9..64 dimensions) on the lane-owned means x (lane l: dimensions l and l + 32): the same
// per-dimension terms, each lane on its two dimensions.  Overwrites x with dL/dmean and writes dL/dlogstd to dls (0 for
// j >= n).  The row's weighted loss, weighted entropy and ratio / n are warp sums (one xor tree: the same order on every
// run), returned on every lane.
template <class Args>
__device__ __forceinline__ void warp_gaussian_row(const Args& a, rw::V2& x, int n, const float* logstd, const float* act,
                                                  const float* old_lp, float adv, float wrow, float went, rw::V2& dls,
                                                  float& loss, float& ent, float& ratio, int lane) {
    float l0 = 0.f, l1 = 0.f, l2 = 0.f;
    auto dim = [&](int j, float& m, float& ds) {
        if (j < n) {
            const float ls = logstd[j], std = expf(ls), var = std * std, diff = act[j] - m;
            const PgTerm pg = pg_term(gaussian_log_prob(diff, std, ls), old_lp[j], adv, a.clip_param, a.flags, a.dual_clip_coeff);
            l0 += pg.loss * wrow;
            l1 += gaussian_entropy(ls) * went;
            l2 += pg.ratio / (float)n;
            const float dlp = pg.dlogp * wrow;
            m = dlp * diff / var;
            ds = dlp * (diff * diff / var - 1.0f) - a.entropy_coef * went;
        } else {
            m = 0.f; ds = 0.f;
        }
    };
    dim(lane, x.a, dls.a);
    dim(lane + 32, x.b, dls.b);
    loss = warp_sum(l0); ent = warp_sum(l1); ratio = warp_sum(l2);
}

// ---- act over host-stepped rows: rows [row_begin, row_end) of slot t = t_begin, R rows per warp ----
// The host steps the env between two launches; this kernel writes actions[t], action_log_probs[t] and rnn_states[t+1]
// (orl_host_insert_rnn zeroes the rows of the envs that finish at step t).  Same staged weights, step_forward and
// sampler as rnn_rollout_warp_kernel: a row's state, logits and action depend neither on R nor on the warp that runs it.
// NB = 64: the wide head (9..64 actions), sampled by warp_sample_action with the noise keys of the feed-forward wide head.
// DX = 256: observations of 65..256 features.  HEAD = ORL_HEAD_GAUSSIAN (NB = 8): the n means out[r][0..n) go to
// gaussian_act, whose key (seed, step, row + rng_row_offset) is the feed-forward act's; the (B, n) noise table of parity
// mode is read by buffer row, the (B, n) actions and log-probs are written into slot t.  HEAD = ORL_HEAD_GAUSSIAN_WIDE
// (NB = 64, 9..64 dimensions): the lane-owned means are parked in the row's scratch and lanes 0..15 each run
// gaussian_act4 on dimensions [4 lane, 4 lane + 4), with the same key, table and slot as the 8-wide head.
template <int R, int NB, int DX, int HEAD>
__global__ void __launch_bounds__(W_NT, 1) rnn_act_rows_warp_kernel(const OrlRnnArgs a) {
    static_assert(HEAD == ORL_HEAD_CATEGORICAL || (HEAD == ORL_HEAD_GAUSSIAN && NB == MAX_OUT) ||
                      (HEAD == ORL_HEAD_GAUSSIAN_WIDE && NB == MAX_OUT_WIDE), "the DiagGaussian heads' widths");
    extern __shared__ __align__(16) float smem[];
    const int B = a.n_envs * a.n_agents, d = a.obs_dim, n = a.n_actions, t = a.t_begin;
    const rc::Offsets o = rc::rnn_offsets(d, n, HEAD != ORL_HEAD_CATEGORICAL);
    const rw::SmemNet W = rw::load_net<NB, DX>(smem, a.policy_params, o, threadIdx.x, W_NT);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* scr = smem + rw::smem_net_floats<NB, DX>(d) + warp * R * rw::SCR;
    const uint64_t step = a.rng_step_base + (a.rng_counter ? *a.rng_counter : 0ull);
    float* const no_tape[R] = {};
    const int rows = a.row_end - a.row_begin, groups = (rows + R - 1) / R;
    for (int g = blockIdx.x * W_WPC + warp; g < groups; g += gridDim.x * W_WPC) {
        typename rw::XIn<DX>::type x[R];
        rw::V2 h[R], hn[R];
        float mk[R];
        typename rw::HeadOut<NB>::type logit[R];
        int row[R];
#pragma unroll
        for (int r = 0; r < R; ++r) {
            row[r] = a.row_begin + min(g * R + r, rows - 1);   // a ragged tail recomputes the last row; its stores are skipped
            const size_t grow = (size_t)t * B + row[r];
            const float* ob = a.policy_obs + grow * d;
            if constexpr (DX == rc::H) x[r] = rw::V2{lane < d ? ob[lane] : 0.f, lane + 32 < d ? ob[lane + 32] : 0.f};
            else x[r] = ob;
            h[r] = rw::ldv(a.rnn_states + grow * rc::H, lane);
            mk[r] = a.masks[grow];
        }
        rw::step_forward<R, NB, DX>(W, scr, d, n, a.activation_id, x, h, mk, hn, logit, no_tape, lane);
        if constexpr (HEAD == ORL_HEAD_GAUSSIAN_WIDE) rw::park<R>(scr, 0, logit, lane);
#pragma unroll
        for (int r = 0; r < R; ++r) {
            if constexpr (HEAD == ORL_HEAD_GAUSSIAN_WIDE) {
                if (g * R + r < rows) {
                    const size_t grow = (size_t)t * B + row[r];
                    if (4 * lane < n)   // noise row and output slot differ: the table is (B, n), the outputs (T, B, n)
                        gaussian_act4(scr + r * rw::SCR, n, 4 * lane, a.policy_params + o.ls, a.deterministic != 0,
                                      a.exp_noise ? a.exp_noise + (size_t)row[r] * n : nullptr, a.rng_seed, step,
                                      (uint32_t)(row[r] + a.rng_row_offset), 0, a.actions + grow * n, a.action_log_probs + grow * n);
                    rw::stv(a.rnn_states + (grow + B) * rc::H, lane, hn[r]);
                }
            } else if constexpr (NB == MAX_OUT_WIDE) {
                const size_t grow = (size_t)t * B + row[r];
                float lp;
                const int act = warp_sample_action(logit[r], n, a.action_masks ? a.action_masks + grow * n : nullptr, a.deterministic != 0,
                                                   [&](int j) {
                    return wide_action_noise1(a.exp_noise, (size_t)row[r], n, a.rng_seed, step, (uint32_t)(row[r] + a.rng_row_offset), j);
                }, lp, lane);
                if (g * R + r < rows) {
                    if (lane == 0) { a.actions[grow] = (float)act; a.action_log_probs[grow] = lp; }
                    rw::stv(a.rnn_states + (grow + B) * rc::H, lane, hn[r]);
                }
            } else if constexpr (HEAD == ORL_HEAD_GAUSSIAN) {
                if (g * R + r < rows) {
                    const size_t grow = (size_t)t * B + row[r];
                    if (lane == 0)   // noise row and output slot differ: the table is (B, n), the outputs (T, B, n)
                        gaussian_act(logit[r], n, a.policy_params + o.ls, a.deterministic != 0,
                                     a.exp_noise ? a.exp_noise + (size_t)row[r] * n : nullptr, a.rng_seed, step,
                                     (uint32_t)(row[r] + a.rng_row_offset), 0, a.actions + grow * n, a.action_log_probs + grow * n);
                    rw::stv(a.rnn_states + (grow + B) * rc::H, lane, hn[r]);
                }
            } else if (g * R + r < rows) {
                const size_t grow = (size_t)t * B + row[r];
                float lp;
                const int act = sample_action(logit[r], n, a.action_masks ? a.action_masks + grow * n : nullptr, a.deterministic != 0,
                                              [&](float (&q)[MAX_OUT]) {   // identical on every lane
                    action_noise(a.exp_noise, (size_t)row[r], n, a.rng_seed, step, (uint32_t)(row[r] + a.rng_row_offset), q);
                }, lp);
                if (lane == 0) { a.actions[grow] = (float)act; a.action_log_probs[grow] = lp; }
                rw::stv(a.rnn_states + (grow + B) * rc::H, lane, hn[r]);
            }
        }
    }
}

// ---- recurrent critic over all T+1 slots: one warp per row (DX = 256: observations of 65..256 features) ----
template <int DX>
__global__ void __launch_bounds__(W_NT, 1) rnn_critic_warp_kernel(const OrlRnnArgs a) {
    extern __shared__ __align__(16) float smem[];
    const int B = a.n_envs * a.n_agents, T = a.episode_length, dc = a.critic_obs_dim;
    const rc::Offsets o = rc::rnn_offsets(dc, 1);
    const rw::SmemNet W = rw::load_net<MAX_OUT, DX>(smem, a.critic_params, o, threadIdx.x, W_NT);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* scr = smem + rw::smem_net_floats<MAX_OUT, DX>(dc) + warp * rw::SCR;
    float* const no_tape[1] = {nullptr};
    for (int row = blockIdx.x * W_WPC + warp; row < B; row += gridDim.x * W_WPC) {
        rw::V2 h[1] = {rw::ldv(a.rnn_states_critic + (size_t)row * rc::H, lane)};
        for (int t = 0; t <= T; ++t) {
            const size_t grow = (size_t)t * B + row;
            const float* ob = a.critic_obs + grow * dc;
            typename rw::XIn<DX>::type x[1];
            if constexpr (DX == rc::H) x[0] = rw::V2{lane < dc ? ob[lane] : 0.f, lane + 32 < dc ? ob[lane + 32] : 0.f};
            else x[0] = ob;
            const float mk[1] = {a.masks[grow]};
            rw::V2 hn[1]; float out[1][MAX_OUT];
            rw::step_forward<1, MAX_OUT, DX>(W, scr, dc, 1, a.activation_id, x, h, mk, hn, out, no_tape, lane);
            if (lane == 0) a.value_preds[grow] = out[0][0];
            if (t < T) {
                const float keep = a.masks[grow + B] == 0.f ? 0.f : 1.f;   // rnn_states_critic[dones_env] = 0
                h[0] = rw::V2{hn[0].a * keep, hn[0].b * keep};
                rw::stv(a.rnn_states_critic + (grow + B) * rc::H, lane, h[0]);
            }
        }
    }
}

// ---- update: one warp per R chunks; L forward steps (tape), per-step loss, L backward steps ----
// AGENT0 (the critic under ORL_PPO_JOINT_ACTION): chunks are recurrent_generator_v3 chunks over f = n*T + t and the
// critic sees agent 0's row of every step only (to_single_np, ppo.py:222-224, 254-262), buffer row t*B + n*A.
// NB = 64 (policy only): the wide head; dL/dlogits goes to the tape field TW_DLW of the wider tape rows (TAPE_WIDE).
// DX = 256: observations of 65..256 features; the rows carry the X field (tape_width_x).
// HEAD = ORL_HEAD_GAUSSIAN (policy, NB = 8): gaussian_row per row step on the row's n actions and old log-probs at bi * n;
// dL/dmean goes to TP_DLOG (the head is the same linear layer) and dL/dlogstd to the field TW_DLS of TAPE_GAUSS rows.
// HEAD = ORL_HEAD_GAUSSIAN_WIDE (policy, NB = 64): warp_gaussian_row on the lane-owned means; dL/dmean goes to TW_DLW (the
// wide head's field, zero for j >= n) and dL/dlogstd to TW_DLSW of TAPE_GAUSS_WIDE rows.
template <bool POLICY, bool AGENT0, int C_R, int NB, int DX, int HEAD>
__global__ void __launch_bounds__(W_NT, 1) rnn_chunk_warp_kernel(const OrlRnnArgs a) {
    static_assert(NB == MAX_OUT || POLICY, "the critic's head is one value");
    constexpr bool GAUSS = HEAD == ORL_HEAD_GAUSSIAN, GAUSS_W = HEAD == ORL_HEAD_GAUSSIAN_WIDE;
    static_assert(!GAUSS || (POLICY && NB == MAX_OUT && !AGENT0), "a DiagGaussian policy head has up to 8 dimensions");
    static_assert(!GAUSS_W || (POLICY && NB == MAX_OUT_WIDE && !AGENT0), "a wide DiagGaussian policy head has 9..64 dimensions");
    constexpr int TW = rw::tape_width(NB, GAUSS || GAUSS_W) + (DX == rc::H ? 0 : rw::MAXD_WIDE);
    extern __shared__ __align__(16) float smem[];
    const int B = a.n_envs * a.n_agents, T = a.episode_length, L = a.chunk_length;
    const int d = POLICY ? a.obs_dim : a.critic_obs_dim, n = POLICY ? a.n_actions : 1;
    const float* obs = POLICY ? a.policy_obs : a.critic_obs;
    const float* states = POLICY ? a.rnn_states : a.rnn_states_critic;
    const rc::Offsets o = rc::rnn_offsets(d, n, GAUSS || GAUSS_W);
    const rw::SmemNet W = rw::load_net<NB, DX>(smem, POLICY ? a.policy_params : a.critic_params, o, threadIdx.x, W_NT);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* scr = smem + rw::smem_net_floats<NB, DX>(d) + warp * C_R * rw::SCR;
    float loss0 = 0.f, loss1 = 0.f, loss2 = 0.f;   // identical on every lane; lane 0's copy is reduced

    const MbConsts mb = mb_consts(a);
    const bool pol_masks = a.flags & ORL_PPO_POLICY_ACTIVE_MASKS, val_masks = a.flags & ORL_PPO_VALUE_ACTIVE_MASKS;

    const long long n_groups = (a.n_chunks + C_R - 1) / C_R;
    for (long long grp = (long long)blockIdx.x * W_WPC + warp; grp < n_groups; grp += (long long)gridDim.x * W_WPC) {
        long long cpos[C_R], f0[C_R];
        bool valid[C_R];
        rw::V2 h[C_R];
#pragma unroll
        for (int r = 0; r < C_R; ++r) {
            valid[r] = grp * C_R + r < a.n_chunks;
            cpos[r] = valid[r] ? grp * C_R + r : grp * C_R;   // a tail slot recomputes chunk 0 of the group (same values, same addresses)
            f0[r] = a.chunk_ids[cpos[r]] * (long long)L;
            const size_t row0 = AGENT0 ? (size_t)(f0[r] / T) * a.n_agents : (size_t)(f0[r] / T);
            h[r] = rw::ldv(states + ((size_t)(f0[r] % T) * B + row0) * rc::H, lane);
        }
        for (int l = 0; l < L; ++l) {
            typename rw::XIn<DX>::type x[C_R];
            rw::V2 h2[C_R];
            float mk[C_R];
            typename rw::HeadOut<NB>::type out[C_R];
            float* tape[C_R];
            size_t bi[C_R];
#pragma unroll
            for (int r = 0; r < C_R; ++r) {
                const long long f = f0[r] + l, row = AGENT0 ? f / T * a.n_agents : f / T, t = f % T;
                bi[r] = (size_t)t * B + row;
                const float* ob = obs + bi[r] * d;
                if constexpr (DX == rc::H) x[r] = rw::V2{lane < d ? ob[lane] : 0.f, lane + 32 < d ? ob[lane + 32] : 0.f};
                else x[r] = ob;
                mk[r] = a.masks[bi[r]];
                tape[r] = a.tape + ((size_t)cpos[r] * L + l) * TW;
            }
            rw::step_forward<C_R, NB, DX, GAUSS || GAUSS_W>(W, scr, d, n, a.activation_id, x, h, mk, h2, out, tape, lane);
#pragma unroll
            for (int r = 0; r < C_R; ++r) {
                h[r] = h2[r];
                if constexpr (GAUSS_W) {
                    // the entropy weight of the 8-wide head: active / sum(active) per dimension, else 1 / (rows n)
                    const float active = a.active_masks[bi[r]];
                    const float keep = valid[r] ? 1.f : 0.f;
                    const float wrow = mb.weight(pol_masks, active), went = pol_masks ? active * mb.inv_act : mb.inv_rows / (float)n;
                    rw::V2 dls;
                    float l0, l1, l2;
                    warp_gaussian_row(a, out[r], n, a.policy_params + o.ls, a.actions + bi[r] * n, a.action_log_probs + bi[r] * n,
                                      apply_adv_norm(mb.adv, a.advantages[bi[r]]), wrow, went, dls, l0, l1, l2, lane);
                    loss0 += keep * l0; loss1 += keep * l1; loss2 += keep * l2;
                    rw::stv(tape[r] + rw::TW_DLW, lane, out[r]);
                    rw::stv(tape[r] + rw::TW_DLSW, lane, dls);
                } else if constexpr (NB == MAX_OUT_WIDE) {
                    const float keep = valid[r] ? 1.f : 0.f;
                    const float wrow = mb.weight(pol_masks, a.active_masks[bi[r]]);
                    const CatRow c = warp_categorical_row(a, out[r], n, a.action_masks ? a.action_masks + bi[r] * n : nullptr,
                                                          (int)a.actions[bi[r]], a.action_log_probs[bi[r]],
                                                          apply_adv_norm(mb.adv, a.advantages[bi[r]]), wrow, lane);
                    loss0 += keep * c.loss * wrow; loss1 += keep * c.ent * wrow; loss2 += keep * c.ratio;
                    rw::stv(tape[r] + rw::TW_DLW, lane, out[r]);
                } else if constexpr (GAUSS) {
                    // the entropy is the mean over rows and dimensions (act.py:150-158): active / sum(active) per dimension
                    // with the active-mask option, else 1 / (rows n)
                    const float active = a.active_masks[bi[r]];
                    const float keep = valid[r] ? 1.f : 0.f;
                    const float wrow = mb.weight(pol_masks, active), went = pol_masks ? active * mb.inv_act : mb.inv_rows / (float)n;
                    float dl[MAX_OUT], dls[MAX_OUT], l0 = 0.f, l1 = 0.f, l2 = 0.f;
#pragma unroll
                    for (int j = 0; j < MAX_OUT; ++j) { dl[j] = 0.f; dls[j] = 0.f; }
                    gaussian_row(a, out[r], n, a.policy_params + o.ls, a.actions + bi[r] * n, a.action_log_probs + bi[r] * n,
                                 apply_adv_norm(mb.adv, a.advantages[bi[r]]), wrow, went, dl, dls, l0, l1, l2);
                    loss0 += keep * l0; loss1 += keep * l1; loss2 += keep * l2;
                    float mine = 0.f, mine_ls = 0.f;   // lane m < 8 stores dL/dmean[m] and dL/dlogstd[m]
#pragma unroll
                    for (int j = 0; j < MAX_OUT; ++j) if (lane == j) { mine = dl[j]; mine_ls = dls[j]; }
                    if (lane < MAX_OUT) { tape[r][rc::TP_DLOG + lane] = mine; tape[r][rw::TW_DLS + lane] = mine_ls; }
                } else {
                    float dl[MAX_OUT];
#pragma unroll
                    for (int j = 0; j < MAX_OUT; ++j) dl[j] = 0.f;
                    const float active = a.active_masks[bi[r]];
                    const float keep = valid[r] ? 1.f : 0.f;
                    if (POLICY) {
                        const float wrow = mb.weight(pol_masks, active);
                        const CatRow c = categorical_row(a, out[r], n, a.action_masks ? a.action_masks + bi[r] * n : nullptr,
                                                         (int)a.actions[bi[r]], a.action_log_probs[bi[r]],
                                                         apply_adv_norm(mb.adv, a.advantages[bi[r]]), wrow, dl);
                        loss0 += keep * c.loss * wrow; loss1 += keep * c.ent * wrow; loss2 += keep * c.ratio;
                    } else {
                        const float ret = a.returns[bi[r]];
                        const float target = (a.flags & ORL_PPO_VALUENORM) ? (ret - mb.vn_mean) / mb.vn_std : ret;
                        const ValueTerm vt = value_term(out[r][0], a.value_preds[bi[r]], target, a.clip_param, a.huber_delta, a.flags);
                        const float wrow = mb.weight(val_masks, active);
                        loss0 += keep * vt.loss * wrow;
                        dl[0] = a.value_loss_coef * wrow * vt.dv;
                    }
                    float mine = 0.f;   // lane m < 8 stores dL/dout[m]
#pragma unroll
                    for (int j = 0; j < MAX_OUT; ++j) if (lane == j) mine = dl[j];
                    if (lane < MAX_OUT) tape[r][rc::TP_DLOG + lane] = mine;
                }
            }
        }
        __syncwarp();   // tape scalars (lane 0) and dL/dout (lanes < 8) are read by every lane below
        rw::V2 dh[C_R];
#pragma unroll
        for (int r = 0; r < C_R; ++r) dh[r] = rw::V2{0.f, 0.f};
        for (int l = L - 1; l >= 0; --l) {
            float* tape[C_R];
#pragma unroll
            for (int r = 0; r < C_R; ++r) tape[r] = a.tape + ((size_t)cpos[r] * L + l) * TW;
            rw::step_backward<C_R, NB>(W, scr, n, a.activation_id, tape, dh, lane);
        }
    }
    __shared__ float red[3][W_WPC];
    if (lane == 0) { red[0][warp] = loss0; red[1][warp] = loss1; red[2][warp] = loss2; }
    __syncthreads();
    if (threadIdx.x < 3) {
        float s = 0.f;
        for (int w = 0; w < W_WPC; ++w) s += red[threadIdx.x][w];
        if (POLICY) atomicAdd(a.loss_acc + threadIdx.x, s);
        else if (threadIdx.x == 0) atomicAdd(a.loss_acc + 3, s);
    }
}

// ---- joint-action policy update (ORL_PPO_JOINT_ACTION, JRPO): one warp per recurrent_generator_v3 chunk ----
// A v3 sample is one (env, step) pair f = n*T + t carrying all A agents (replay_data.py:425-551); the warp advances
// the A agent rows of its chunk together (step_forward<A> / step_backward<A>, the rollout's row grouping).  Per step
// (one group): ratio = exp(sum_a logp_a - sum_a old_logp_a) with agent 0's advantage, weighted by agent 0's active
// mask over the agent-0 active sum (mb_stats[2]) or 1/groups; every agent row receives the same dL/dlogp.  The
// entropy stays per agent row, weighted by every agent's active mask over the all-agent active sum (mb_stats[5]) or
// 1/(groups*A) (ppo.py:254-319).  Tape row of (chunk c, step l, agent ag): (c*L + l)*A + ag.
template <int A>
__global__ void __launch_bounds__(W_NT, 1) rnn_joint_policy_warp_kernel(const OrlRnnArgs a) {
    extern __shared__ __align__(16) float smem[];
    const int B = a.n_envs * A, T = a.episode_length, L = a.chunk_length;
    const int d = a.obs_dim, n = a.n_actions;
    const rc::Offsets o = rc::rnn_offsets(d, n);
    const rw::SmemNet W = rw::load_net(smem, a.policy_params, o, threadIdx.x, W_NT);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* scr = smem + rw::smem_net_floats(d) + warp * A * rw::SCR;
    float loss0 = 0.f, loss1 = 0.f, loss2 = 0.f;   // identical on every lane; lane 0's copy is reduced

    const double groups_d = loss_rows(a);
    const float inv_groups = (float)(1.0 / groups_d), inv_rows = (float)(1.0 / (groups_d * A));
    const float inv_act0 = (float)(1.0 / a.mb_stats[2]), inv_act_all = (float)(1.0 / a.mb_stats[5]);
    const bool pol_masks = a.flags & ORL_PPO_POLICY_ACTIVE_MASKS;
    const AdvNorm advn = make_adv_norm(a.gae_stats, a.flags & ORL_PPO_ADV_NORMALIZE);

    for (long long c = (long long)blockIdx.x * W_WPC + warp; c < a.n_chunks; c += (long long)gridDim.x * W_WPC) {
        const long long f0 = a.chunk_ids[c] * (long long)L;
        const size_t s0 = (size_t)(f0 % T) * B + (size_t)(f0 / T) * A;   // agent 0 of the chunk's first sample
        rw::V2 h[A];
#pragma unroll
        for (int ag = 0; ag < A; ++ag) h[ag] = rw::ldv(a.rnn_states + (s0 + ag) * rc::H, lane);
        for (int l = 0; l < L; ++l) {
            const long long f = f0 + l;
            const size_t base = (size_t)(f % T) * B + (size_t)(f / T) * A;
            rw::V2 x[A], h2[A];
            float mk[A], out[A][MAX_OUT];
            float* tape[A];
#pragma unroll
            for (int ag = 0; ag < A; ++ag) {
                const float* ob = a.policy_obs + (base + ag) * d;
                x[ag] = rw::V2{lane < d ? ob[lane] : 0.f, lane + 32 < d ? ob[lane + 32] : 0.f};
                mk[ag] = a.masks[base + ag];
                tape[ag] = a.tape + (((size_t)c * L + l) * A + ag) * rw::TAPE_W;
            }
            rw::step_forward<A>(W, scr, d, n, a.activation_id, x, h, mk, h2, out, tape, lane);
            float joint = 0.f, joint_old = 0.f;   // summed in agent order, like the reference's reshape(-1, A).sum
#pragma unroll
            for (int ag = 0; ag < A; ++ag) {
                h[ag] = h2[ag];
                float nl[MAX_OUT], pr[MAX_OUT];
                log_softmax_n(out[ag], n, nl, pr);
                joint += log_prob_of(nl, n, (int)a.actions[base + ag]);
                joint_old += a.action_log_probs[base + ag];
            }
            const float adv = apply_adv_norm(advn, a.advantages[base]);
            const PgTerm pg = pg_term(joint, joint_old, adv, a.clip_param, a.flags, a.dual_clip_coeff);
            const float wgrp = pol_masks ? a.active_masks[base] * inv_act0 : inv_groups;
            loss0 += pg.loss * wgrp; loss2 += pg.ratio;
            const float dlp = pg.dlogp * wgrp;
#pragma unroll
            for (int ag = 0; ag < A; ++ag) {
                float nl[MAX_OUT], pr[MAX_OUT], dl[MAX_OUT] = {};
                log_softmax_n(out[ag], n, nl, pr);
                const float went_w = pol_masks ? a.active_masks[base + ag] * inv_act_all : inv_rows;
                const float ent = categorical_entropy(nl, pr, n);
                loss1 += ent * went_w;
                categorical_dlogits(dlp, a.entropy_coef * went_w, (int)a.actions[base + ag], n, 0u, nl, pr, ent, dl);
                float mine = 0.f;   // lane m < 8 stores dL/dout[m]
#pragma unroll
                for (int j = 0; j < MAX_OUT; ++j) if (lane == j) mine = dl[j];
                if (lane < MAX_OUT) tape[ag][rc::TP_DLOG + lane] = mine;
            }
        }
        __syncwarp();   // tape scalars (lane 0) and dL/dout (lanes < 8) are read by every lane below
        rw::V2 dh[A];
#pragma unroll
        for (int ag = 0; ag < A; ++ag) dh[ag] = rw::V2{0.f, 0.f};
        for (int l = L - 1; l >= 0; --l) {
            float* tape[A];
#pragma unroll
            for (int ag = 0; ag < A; ++ag) tape[ag] = a.tape + (((size_t)c * L + l) * A + ag) * rw::TAPE_W;
            rw::step_backward<A>(W, scr, n, a.activation_id, tape, dh, lane);
        }
    }
    __shared__ float red[3][W_WPC];
    if (lane == 0) { red[0][warp] = loss0; red[1][warp] = loss1; red[2][warp] = loss2; }
    __syncthreads();
    if (threadIdx.x < 3) {
        float s = 0.f;
        for (int w = 0; w < W_WPC; ++w) s += red[threadIdx.x][w];
        atomicAdd(a.loss_acc + threadIdx.x, s);
    }
}

// ---- parameter gradients of one net from its tape (orl::reduce_tape); every job fits the gemm tiles: TQ_X + 64 <= TAPE_W ----
// A wide head (n > 8) reads dL/dlogits from the appended field TW_DLW of its TAPE_WIDE rows; a DiagGaussian head adds the
// logstd column sum over TW_DLS (TW_DLSW for n > 8).  A wide observation (d > 64) has no W1 job here: its gradient comes
// from w1_panel_jobs.
TapeJobs make_jobs(int d, int n, bool gauss) {
    const rc::Offsets o = rc::rnn_offsets(d, n, gauss);
    TapeJobs t; int g = 0, c = 0;
    auto gemm = [&](int p, int M, int q, int N, int out) { t.gemm[g++] = TapeJob{p, M, q, N, out}; };
    auto col = [&](int p, int M, int out) { t.col[c++] = TapeJob{p, M, -1, 1, out}; };
    if (d <= rc::MAXD) gemm(rc::TP_DZ1, rc::H, rc::TQ_X, d, o.w1);
    col(rc::TP_DZ1, rc::H, o.b1);
    col(rc::TS_DY1N1, rc::H, o.g1);                  col(rc::TS_DY1, rc::H, o.be1);
    gemm(rc::TP_DZ3, rc::H, rc::TQ_Y1, rc::H, o.w3); col(rc::TP_DZ3, rc::H, o.b3);
    col(rc::TS_DY3N3, rc::H, o.g3);                  col(rc::TS_DY3, rc::H, o.be3);
    gemm(rc::TP_DGI, rc::G3, rc::TQ_Y3, rc::H, o.wih); gemm(rc::TP_DGH, rc::G3, rc::TQ_HM, rc::H, o.whh);
    col(rc::TP_DGI, rc::G3, o.bih);                  col(rc::TP_DGH, rc::G3, o.bhh);
    col(rc::TS_DONO, rc::H, o.gr);                   col(rc::TS_DO, rc::H, o.ber);
    const int dlog = n > MAX_OUT ? rw::TW_DLW : rc::TP_DLOG;
    gemm(dlog, n, rc::TQ_O, rc::H, o.wh);            col(dlog, n, o.bh);
    if (gauss) col(n > MAX_OUT ? rw::TW_DLSW : rw::TW_DLS, n, o.ls);
    t.n_gemm = g; t.n_col = c;
    return t;
}

// dW1 of a wide observation (d > 64) as 64-column panels sum_rows dZ1^T X_p over the X field: panel p lands at
// W1P_PANEL * p as [64][min(64, d - 64 p)], in a panel buffer of W1P_FLOATS that w1_scatter_kernel unpacks into W1's [64][d]
constexpr int W1P_PANEL = rc::H * 64, W1P_FLOATS = W1P_PANEL * rw::MAXD_WIDE / 64;
TapeJobs w1_panel_jobs(int d, int n, bool gauss) {
    TapeJobs t; t.n_gemm = 0; t.n_col = 0;
    for (int p = 0; 64 * p < d; ++p)
        t.gemm[t.n_gemm++] = TapeJob{rc::TP_DZ1, rc::H, rw::tape_width(n, gauss) + 64 * p, std::min(64, d - 64 * p), W1P_PANEL * p};
    return t;
}
__global__ void w1_scatter_kernel(const float* __restrict__ panels, int d, float* __restrict__ w1) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rc::H * d) return;
    const int m = i / d, k = i % d, p = k / 64, np = min(64, d - 64 * p);
    w1[i] = panels[W1P_PANEL * p + m * np + (k - 64 * p)];
}
// the update's workspace: the larger of the two nets' tapes, the reduction partials and, with a wide observation, the panel
// buffer.  JRPO sizes it with rows = its policy tape's A rows per chunk step, the larger tape there.
long long ws_floats(long long rows, int grads_stride, int n_actions, int obs_dim, int critic_obs_dim, bool gauss = false) {
    const long long tw = std::max(rw::tape_width_x(n_actions, obs_dim, gauss), rw::tape_width_x(1, critic_obs_dim));
    const bool wide = obs_dim > rc::MAXD || critic_obs_dim > rc::MAXD;
    return rows * tw + (rows + TAPE_ROW_BLOCK - 1) / TAPE_ROW_BLOCK * grads_stride + (wide ? W1P_FLOATS : 0);
}

// ---- optimizer: per-net global-norm clip + Adam on the true-layout gradients (one CTA per net) ----
// HEAD = ORL_HEAD_GAUSSIAN: the policy's total includes logstd, so it is in the clip norm and takes its Adam step
// (clip_grad_norm_ over every policy parameter, ppo.py:120-158)
template <int HEAD>
__global__ void __launch_bounds__(1024) rnn_apply_kernel(const OrlRnnArgs a) {
    const int net = blockIdx.x;
    const int total = net == 0 ? rc::rnn_offsets(a.obs_dim, a.n_actions, HEAD == ORL_HEAD_GAUSSIAN).total
                               : rc::rnn_offsets(a.critic_obs_dim, 1).total;
    const float* grads = a.grads + (size_t)net * a.grads_stride;
    float sq = 0.f;
    for (int i = threadIdx.x; i < total; i += blockDim.x) sq = fmaf(grads[i], grads[i], sq);
    const float norm = block_l2_norm(sq);
    adam_step(a, net, net == 0 ? a.policy_params : a.critic_params, net == 0 ? a.policy_adam_m : a.critic_adam_m,
              net == 0 ? a.policy_adam_v : a.critic_adam_v, grads, total, clip_factor(a, norm));
    if (threadIdx.x == 0) {
        if (net == 0) add_policy_info(a, a.loss_acc, norm);
        else add_value_info(a, a.loss_acc[3], norm);
    }
}

// weights of one net staged by load_net<NB, DX> + the per-warp mat-vec scratch of R rows
template <int NB, int DX>
constexpr size_t w_smem(int d, int rows_per_warp) {
    return (size_t)(rw::smem_net_floats<NB, DX>(d) + rw::smem_scratch_floats(W_WPC, rows_per_warp)) * sizeof(float);
}
static_assert(w_smem<MAX_OUT_WIDE, rc::H>(rc::MAXD, 2) <= 227 * 1024, "the wide policy's weights and scratch fit the opt-in shared memory");
// A wide observation (d > 64): W1 at w1_ld(d).  Rows per warp: two where the weights, the scratch and the chunk kernel's
// 192 B of static loss slots fit the 227 KB opt-in limit, else one.  Only the wide head's net at d > 240 needs one.
constexpr size_t SMEM_OPTIN = 227 * 1024, CHUNK_STATIC_SMEM = 3 * W_WPC * sizeof(float);
template <int NB>
constexpr int wide_rows_per_warp(int d) { return w_smem<NB, rw::MAXD_WIDE>(d, 2) + CHUNK_STATIC_SMEM <= SMEM_OPTIN ? 2 : 1; }
static_assert(wide_rows_per_warp<MAX_OUT>(rw::MAXD_WIDE) == 2, "a narrow-head net of any width runs two rows per warp");
static_assert(wide_rows_per_warp<MAX_OUT_WIDE>(240) == 2 && wide_rows_per_warp<MAX_OUT_WIDE>(241) == 1, "the R switch");
static_assert(w_smem<MAX_OUT_WIDE, rw::MAXD_WIDE>(rw::MAXD_WIDE, 1) + CHUNK_STATIC_SMEM <= SMEM_OPTIN, "every width fits at one row per warp");
// the only bounds at which two rows per warp may not fit (the static_asserts above)
template <int NB, int DX>
constexpr bool may_need_one_row = NB == MAX_OUT_WIDE && DX == rw::MAXD_WIDE;

int warp_grid(long long units) {   // persistent CTAs: one per SM, never more than the work needs
    const long long need = (units + W_WPC - 1) / W_WPC;
    return (int)std::max(1LL, std::min<long long>(need, orl::sm_count()));
}
// every launch of a dynamic-shared-memory kernel here: `units` warp work items (envs, rows, row pairs, chunks)
int launch(void (*kern)(OrlRnnArgs), long long units, size_t smem, const OrlRnnArgs& a, cudaStream_t st) {
    if (int e = orl::allow_dynamic_smem(kern, smem)) return e;
    kern<<<warp_grid(units), W_NT, smem, st>>>(a);
    return 0;
}

// max_obs: 64 for the device-env rollout, 256 (MAXD_WIDE) for the host-stepped entries
int check_common(const OrlRnnArgs& a, int max_obs = rc::MAXD) {
    ORL_CHECK_ARG(a.n_envs > 0 && a.n_agents > 0 && a.episode_length > 0, "n_envs / n_agents / episode_length");
    if (max_obs == rc::MAXD) {
        ORL_CHECK_ARG(a.obs_dim > 0 && a.obs_dim <= rc::MAXD && a.critic_obs_dim > 0 && a.critic_obs_dim <= rc::MAXD, "obs dims (<= 64)");
    } else {
        ORL_CHECK_ARG(a.obs_dim > 0 && a.obs_dim <= max_obs && a.critic_obs_dim > 0 && a.critic_obs_dim <= max_obs,
                      "obs dims must be in 1..256");
    }
    ORL_CHECK_ARG(a.n_actions > 0 && a.n_actions <= MAX_OUT_WIDE, "n_actions must be in 1..64");
    ORL_CHECK_ARG(a.activation_id >= 0 && a.activation_id <= 3, "activation_id");
    ORL_CHECK_ARG(a.head_kind == ORL_HEAD_CATEGORICAL || a.head_kind == ORL_HEAD_GAUSSIAN || a.head_kind == ORL_HEAD_GAUSSIAN_WIDE,
                  "head_kind must be ORL_HEAD_CATEGORICAL, ORL_HEAD_GAUSSIAN or ORL_HEAD_GAUSSIAN_WIDE");
    ORL_CHECK_ARG(a.head_kind != ORL_HEAD_GAUSSIAN || a.n_actions <= MAX_OUT, "ORL_HEAD_GAUSSIAN is built for 1..8 dimensions");
    ORL_CHECK_ARG(a.head_kind != ORL_HEAD_GAUSSIAN_WIDE || a.n_actions > MAX_OUT,
                  "head_kind ORL_HEAD_GAUSSIAN_WIDE is built for 9..64 dimensions (ORL_HEAD_GAUSSIAN for 1..8)");
    return 0;
}

// the act over `rows` host-stepped rows: one row per warp while the rows leave warps of the persistent grid idle, else
// two (every weight read feeds both) where they fit
template <int NB, int DX, int HEAD = ORL_HEAD_CATEGORICAL>
int launch_act_rows(const OrlRnnArgs& a, int rows, cudaStream_t st) {
    const bool one = rows <= orl::sm_count() * W_WPC || (may_need_one_row<NB, DX> && wide_rows_per_warp<NB>(a.obs_dim) == 1);
    return one ? launch(rnn_act_rows_warp_kernel<1, NB, DX, HEAD>, rows, w_smem<NB, DX>(a.obs_dim, 1), a, st)
               : launch(rnn_act_rows_warp_kernel<2, NB, DX, HEAD>, (rows + 1) / 2, w_smem<NB, DX>(a.obs_dim, 2), a, st);
}

// the chunk kernel of one net of d features: two chunks per warp (every weight read feeds both) where they fit
template <bool POLICY, bool AGENT0, int NB, int DX, int HEAD = ORL_HEAD_CATEGORICAL>
int launch_chunks(const OrlRnnArgs& a, int d, cudaStream_t st) {
    if constexpr (may_need_one_row<NB, DX>) {
        if (wide_rows_per_warp<NB>(d) == 1)
            return launch(rnn_chunk_warp_kernel<POLICY, AGENT0, 1, NB, DX, HEAD>, a.n_chunks, w_smem<NB, DX>(d, 1), a, st);
    }
    return launch(rnn_chunk_warp_kernel<POLICY, AGENT0, 2, NB, DX, HEAD>, (a.n_chunks + 1) / 2, w_smem<NB, DX>(d, 2), a, st);
}

// the forward / backward pass of one net over its chunks, writing its tape; JRPO (joint): the joint policy kernel, and the
// critic on agent 0's rows
int launch_net(const OrlRnnArgs& a, int net, bool joint, cudaStream_t st) {
    const int d = net == 0 ? a.obs_dim : a.critic_obs_dim;
    const bool wide_obs = d > rc::MAXD, wide_head = a.n_actions > MAX_OUT;
    constexpr int XW = rw::MAXD_WIDE;
    if (net == 1) {
        if (joint) return launch_chunks<false, true, MAX_OUT, rc::H>(a, d, st);
        return wide_obs ? launch_chunks<false, false, MAX_OUT, XW>(a, d, st) : launch_chunks<false, false, MAX_OUT, rc::H>(a, d, st);
    }
    if (joint) return launch(rnn_joint_policy_warp_kernel<JOINT_A>, a.n_chunks, w_smem<MAX_OUT, rc::H>(d, JOINT_A), a, st);
    if (a.head_kind == ORL_HEAD_GAUSSIAN)
        return wide_obs ? launch_chunks<true, false, MAX_OUT, XW, ORL_HEAD_GAUSSIAN>(a, d, st)
                        : launch_chunks<true, false, MAX_OUT, rc::H, ORL_HEAD_GAUSSIAN>(a, d, st);
    if (a.head_kind == ORL_HEAD_GAUSSIAN_WIDE)
        return wide_obs ? launch_chunks<true, false, MAX_OUT_WIDE, XW, ORL_HEAD_GAUSSIAN_WIDE>(a, d, st)
                        : launch_chunks<true, false, MAX_OUT_WIDE, rc::H, ORL_HEAD_GAUSSIAN_WIDE>(a, d, st);
    if (wide_obs)
        return wide_head ? launch_chunks<true, false, MAX_OUT_WIDE, XW>(a, d, st) : launch_chunks<true, false, MAX_OUT, XW>(a, d, st);
    return wide_head ? launch_chunks<true, false, MAX_OUT_WIDE, rc::H>(a, d, st) : launch_chunks<true, false, MAX_OUT, rc::H>(a, d, st);
}

}  // namespace

extern "C" {

int orl_rnn_param_count(int obs_dim, int n_out) { return rc::rnn_offsets(obs_dim, n_out).total; }
int orl_rnn_param_count_head(int obs_dim, int n_out, int head_kind) {
    return rc::rnn_offsets(obs_dim, n_out, head_kind == ORL_HEAD_GAUSSIAN || head_kind == ORL_HEAD_GAUSSIAN_WIDE).total;
}
int orl_rnn_tape_width(void) { return rw::TAPE_W; }
long long orl_rnn_workspace_floats_wide_obs(long long rows, int grads_stride, int n_actions, int obs_dim, int critic_obs_dim) {
    return ws_floats(rows, grads_stride, n_actions, obs_dim, critic_obs_dim);
}
long long orl_rnn_workspace_floats_head(long long rows, int grads_stride, int n_actions, int obs_dim, int critic_obs_dim, int head_kind) {
    return ws_floats(rows, grads_stride, n_actions, obs_dim, critic_obs_dim,
                     head_kind == ORL_HEAD_GAUSSIAN || head_kind == ORL_HEAD_GAUSSIAN_WIDE);
}
long long orl_rnn_workspace_floats(long long rows, int grads_stride) { return ws_floats(rows, grads_stride, 1, rc::MAXD, rc::MAXD); }
long long orl_rnn_workspace_floats_for(long long rows, int grads_stride, int n_actions) {
    return ws_floats(rows, grads_stride, n_actions, rc::MAXD, rc::MAXD);
}

int orl_rnn_rollout(const OrlRnnArgs* ap, void* stream) {
    ORL_CHECK_ARG(ap, "args");
    const OrlRnnArgs& a = *ap;
    if (int e = check_common(a)) return e;
    ORL_CHECK_ARG(a.env_kind != ORL_ENV_NONE, "ORL_ENV_NONE: the act of host-stepped rows is orl_rnn_act_rows");
    ORL_CHECK_ARG(a.n_actions <= MAX_OUT, "n_actions must be in 1..8 for the device envs (they have at most 5 actions)");
    ORL_CHECK_ARG(a.head_kind == ORL_HEAD_CATEGORICAL, "the device envs are Discrete: orl_rnn_rollout takes ORL_HEAD_CATEGORICAL only");
    ORL_CHECK_ARG(a.policy_params && a.policy_obs && a.rnn_states && a.actions && a.action_log_probs && a.masks, "null rollout buffer");
    ORL_CHECK_ARG(a.t_begin >= 0 && a.t_end <= a.episode_length && a.t_begin <= a.t_end, "t range");
    ORL_CHECK_ARG(a.critic_obs && a.rewards && a.active_masks, "null rollout buffer");
    ORL_CHECK_ARG(a.env_kind == ORL_ENV_MPE_SPREAD || a.env_kind == ORL_ENV_CARTPOLE || a.env_kind == ORL_ENV_GRIDWORLD,
                  "unknown env kind");
    ORL_CHECK_ARG(a.ep_return && a.ep_length && a.episode_stats, "episode statistics buffers");
    if (a.env_kind == ORL_ENV_MPE_SPREAD) {
        ORL_CHECK_ARG(a.n_agents == 3 && a.obs_dim == 18 && a.critic_obs_dim == 54 && a.env_f64 && a.env_u64 && a.env_i32,
                      "simple_spread shapes / state");
    } else {
        ORL_CHECK_ARG(a.n_agents == 1 && a.obs_dim == 4, "single-agent env shapes");
        ORL_CHECK_ARG(single_obs_aligned(a), "policy_obs and critic_obs must be 16-byte aligned");
    }
    if (a.t_end > a.t_begin) {
        const bool mpe = a.env_kind == ORL_ENV_MPE_SPREAD;
        void (*const kern)(OrlRnnArgs) = mpe ? rnn_rollout_warp_kernel<ORL_ENV_MPE_SPREAD>
                                         : a.env_kind == ORL_ENV_CARTPOLE ? rnn_rollout_warp_kernel<ORL_ENV_CARTPOLE>
                                                                          : rnn_rollout_warp_kernel<ORL_ENV_GRIDWORLD>;
        if (int e = launch(kern, a.n_envs, w_smem<MAX_OUT, rc::H>(a.obs_dim, mpe ? 3 : 1), a, (cudaStream_t)stream)) return e;
    }
    if (int e = orl::check_cuda(cudaGetLastError(), "rnn_rollout_warp_kernel launch")) return e;
    return orl::bump_rng_counter(a.rng_counter, a.t_end - a.t_begin, (cudaStream_t)stream);
}

int orl_rnn_act_rows(const OrlRnnArgs* ap, void* stream) {
    ORL_CHECK_ARG(ap, "args");
    const OrlRnnArgs& a = *ap;
    if (int e = check_common(a, rw::MAXD_WIDE)) return e;
    ORL_CHECK_ARG(a.policy_params && a.policy_obs && a.rnn_states && a.actions && a.action_log_probs && a.masks, "null act buffer");
    ORL_CHECK_ARG(a.t_begin >= 0 && a.t_begin < a.episode_length, "slot t_begin");
    ORL_CHECK_ARG(a.row_begin >= 0 && a.row_begin <= a.row_end && (long long)a.row_end <= (long long)a.n_envs * a.n_agents, "row range");
    cudaStream_t st = (cudaStream_t)stream;
    const int rows = a.row_end - a.row_begin;
    if (rows > 0) {
        constexpr int XW = rw::MAXD_WIDE;
        const bool wide_obs = a.obs_dim > rc::MAXD, wide_head = a.n_actions > MAX_OUT;
        int e = a.head_kind == ORL_HEAD_GAUSSIAN
                    ? (wide_obs ? launch_act_rows<MAX_OUT, XW, ORL_HEAD_GAUSSIAN>(a, rows, st)
                                : launch_act_rows<MAX_OUT, rc::H, ORL_HEAD_GAUSSIAN>(a, rows, st))
              : a.head_kind == ORL_HEAD_GAUSSIAN_WIDE
                    ? (wide_obs ? launch_act_rows<MAX_OUT_WIDE, XW, ORL_HEAD_GAUSSIAN_WIDE>(a, rows, st)
                                : launch_act_rows<MAX_OUT_WIDE, rc::H, ORL_HEAD_GAUSSIAN_WIDE>(a, rows, st))
              : wide_obs ? (wide_head ? launch_act_rows<MAX_OUT_WIDE, XW>(a, rows, st) : launch_act_rows<MAX_OUT, XW>(a, rows, st))
                         : (wide_head ? launch_act_rows<MAX_OUT_WIDE, rc::H>(a, rows, st) : launch_act_rows<MAX_OUT, rc::H>(a, rows, st));
        if (e) return e;
        if ((e = orl::check_cuda(cudaGetLastError(), "rnn_act_rows_warp_kernel launch"))) return e;
    }
    return orl::bump_rng_counter(a.rng_counter, 1, st);
}

int orl_rnn_critic(const OrlRnnArgs* ap, void* stream) {
    ORL_CHECK_ARG(ap, "args");
    const OrlRnnArgs& a = *ap;
    if (int e = check_common(a, rw::MAXD_WIDE)) return e;
    ORL_CHECK_ARG(a.critic_params && a.critic_obs && a.rnn_states_critic && a.masks && a.value_preds, "null critic buffer");
    const int B = a.n_envs * a.n_agents, dc = a.critic_obs_dim;
    const int e = dc > rc::MAXD ? launch(rnn_critic_warp_kernel<rw::MAXD_WIDE>, B, w_smem<MAX_OUT, rw::MAXD_WIDE>(dc, 1), a, (cudaStream_t)stream)
                                : launch(rnn_critic_warp_kernel<rc::H>, B, w_smem<MAX_OUT, rc::H>(dc, 1), a, (cudaStream_t)stream);
    return e ? e : orl::check_cuda(cudaGetLastError(), "rnn_critic_warp_kernel launch");
}

int orl_rnn_fwdbwd(const OrlRnnArgs* ap, void* stream) {
    ORL_CHECK_ARG(ap, "args");
    const OrlRnnArgs& a = *ap;
    if (int e = check_common(a, rw::MAXD_WIDE)) return e;
    ORL_CHECK_ARG(a.chunk_length >= 1 && a.chunk_length <= LMAX, "chunk_length (data_chunk_length) must be in [1, 32]");
    ORL_CHECK_ARG(a.n_chunks > 0 && a.chunk_ids, "chunks");
    ORL_CHECK_ARG(a.policy_params && a.critic_params && a.policy_obs && a.critic_obs && a.rnn_states && a.rnn_states_critic &&
                      a.actions && a.action_log_probs && a.masks && a.active_masks && a.value_preds && a.returns && a.advantages,
                  "null update buffer");
    ORL_CHECK_ARG(a.gae_stats && a.mb_stats && a.tape && a.grads && a.loss_acc, "stats / workspace");
    const bool gauss = a.head_kind == ORL_HEAD_GAUSSIAN || a.head_kind == ORL_HEAD_GAUSSIAN_WIDE;
    ORL_CHECK_ARG(a.grads_stride >= rc::rnn_offsets(a.obs_dim, a.n_actions, gauss).total &&
                      a.grads_stride >= rc::rnn_offsets(a.critic_obs_dim, 1).total, "grads_stride");
    if (a.flags & ORL_PPO_VALUENORM) { ORL_CHECK_ARG(a.vn_state, "vn_state"); }
    // ORL_PPO_JOINT_ACTION: v3 chunks; the policy tape holds A rows per chunk step, the critic's one (agent 0)
    const bool joint = a.flags & ORL_PPO_JOINT_ACTION;
    if (joint) {
        ORL_CHECK_ARG(a.n_agents == JOINT_A, "ORL_PPO_JOINT_ACTION is built for 3 agents (simple_spread)");
        ORL_CHECK_ARG(a.n_chunks * a.chunk_length <= (long long)a.n_envs * a.episode_length, "v3 chunks exceed the N*T samples");
        ORL_CHECK_ARG(!a.action_masks, "ORL_PPO_JOINT_ACTION takes no action_masks (simple_spread reports none)");
        ORL_CHECK_ARG(a.n_actions <= MAX_OUT, "ORL_PPO_JOINT_ACTION is built for up to 8 actions");
        ORL_CHECK_ARG(!gauss, "ORL_PPO_JOINT_ACTION is built for Discrete action spaces (ORL_HEAD_CATEGORICAL)");
        ORL_CHECK_ARG(a.obs_dim <= rc::MAXD && a.critic_obs_dim <= rc::MAXD, "ORL_PPO_JOINT_ACTION is built for obs dims 1..64");
    }
    cudaStream_t st = (cudaStream_t)stream;
    int e = orl::check_cuda(cudaMemsetAsync(a.loss_acc, 0, 8 * sizeof(float), st), "memset loss_acc");
    if (e) return e;
    const long long steps = a.n_chunks * a.chunk_length;
    const long long net_rows[2] = {joint ? steps * JOINT_A : steps, steps};
    const int tw[2] = {rw::tape_width_x(a.n_actions, a.obs_dim, gauss), rw::tape_width_x(1, a.critic_obs_dim)};
    float* partials = a.tape + std::max(net_rows[0] * tw[0], net_rows[1] * tw[1]);   // after the larger of the two tapes
    float* panels = partials + (std::max(net_rows[0], net_rows[1]) + TAPE_ROW_BLOCK - 1) / TAPE_ROW_BLOCK * a.grads_stride;
    for (int net = 0; net < 2; ++net) {
        const int d = net == 0 ? a.obs_dim : a.critic_obs_dim, n = net == 0 ? a.n_actions : 1;
        if ((e = launch_net(a, net, joint, st))) return e;
        const bool g = net == 0 && gauss;
        const rc::Offsets o = rc::rnn_offsets(d, n, g);
        float* grads = a.grads + (size_t)net * a.grads_stride;
        if ((e = orl::reduce_tape(a.tape, tw[net], net_rows[net], make_jobs(d, n, g), partials, a.grads_stride, o.total, grads, st))) return e;
        if (d > rc::MAXD) {   // W1's entries of the first reduction are overwritten here
            const int last = (d - 1) / 64, used = W1P_PANEL * last + rc::H * (d - 64 * last);
            if ((e = orl::reduce_tape(a.tape, tw[net], net_rows[net], w1_panel_jobs(d, n, g), partials, W1P_FLOATS, used, panels, st))) return e;
            w1_scatter_kernel<<<(rc::H * d + 255) / 256, 256, 0, st>>>(panels, d, grads + o.w1);
        }
    }
    return orl::check_cuda(cudaGetLastError(), "rnn update launches");
}

int orl_rnn_apply(const OrlRnnArgs* ap, void* stream) {
    ORL_CHECK_ARG(ap, "args");
    const OrlRnnArgs& a = *ap;
    if (int e = check_common(a, rw::MAXD_WIDE)) return e;
    ORL_CHECK_ARG(a.policy_params && a.critic_params && a.grads && a.loss_acc && a.policy_adam_m && a.policy_adam_v &&
                      a.critic_adam_m && a.critic_adam_v && a.adam_steps && a.lrs && a.train_info && a.mb_stats, "null optimizer buffer");
    ORL_CHECK_ARG(a.n_chunks > 0 && a.chunk_length >= 1, "chunks");
    if (a.flags & ORL_PPO_VALUENORM) { ORL_CHECK_ARG(a.vn_state, "vn_state"); }
    // the wide DiagGaussian head has the 8-wide one's layout (logstd after the head): it runs as that
    if (a.head_kind == ORL_HEAD_GAUSSIAN || a.head_kind == ORL_HEAD_GAUSSIAN_WIDE)
        rnn_apply_kernel<ORL_HEAD_GAUSSIAN><<<2, 1024, 0, (cudaStream_t)stream>>>(a);
    else rnn_apply_kernel<ORL_HEAD_CATEGORICAL><<<2, 1024, 0, (cudaStream_t)stream>>>(a);
    return orl::check_cuda(cudaGetLastError(), "rnn_apply_kernel launch");
}

}  // extern "C"
