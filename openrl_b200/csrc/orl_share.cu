// cfg.use_share_model: ONE policy-value network (reference: PolicyValueNetwork, policy_value_network.py:33-174) with one
// optimiser — rollout, value pass and the PPO update (ppo.py:46-176 with `_use_share_model`: both losses back-propagate
// into the same parameters, both clip_grad_norm_ calls see all of them, one Adam step).
//
// Correctness-first implementation (this option is not on the benchmarked configs): one thread per row runs the
// sequential core of orl_deep_core.h (verified on the CPU against torch autograd of the oracle, tests/test_deep_core_cpu.py);
// the update writes a per-row tape and the parameter gradients are deterministic tape reductions dW = sum_rows P^T Q.
// Discrete actions take a Categorical head (device envs or ORL_ENV_NONE); Box(n <= 8) actions take a DiagGaussian head
// (ORL_ENV_NONE: host-stepped envs).  The kernels are templates on the head, so the Categorical instances are exactly
// the kernels built before the Gaussian head existed.
#include <algorithm>

#include "orl_adam.cuh"
#include "orl_deep_core.h"
#include "orl_envstep.cuh"

namespace {
using namespace orl;
namespace dc = orl_deep;

constexpr int S_NT = 128;

__device__ __forceinline__ void load_obs_row(const float* __restrict__ obs, size_t row, int d, float* x) {
    for (int k = 0; k < d; ++k) x[k] = obs[row * d + k];
}

// ---- rollout (single-agent device envs, or ENV_NONE = act only): one thread per env for all steps ----
// HEAD = ORL_HEAD_GAUSSIAN: the DiagGaussian act of gaussian_act (the noise of the FFMA rollout_kernel's act for the same
// (seed, step, row)); device envs are all Discrete, so only the ENV_NONE instance has it.
template <int ENV, int HEAD>
__global__ void __launch_bounds__(S_NT) share_rollout_kernel(const OrlRolloutArgs a) {
    static_assert(HEAD == ORL_HEAD_CATEGORICAL || ENV == ORL_ENV_NONE, "Box actions act on host-stepped envs only");
    const int N = a.n_envs, B = N * a.n_agents, d = a.obs_dim, n = a.n_actions;
    const int e = blockIdx.x * S_NT + threadIdx.x;
    if (e >= B) return;
    const dc::Offsets o = dc::deep_offsets(d, n, HEAD == ORL_HEAD_GAUSSIAN);
    const uint64_t rng_base = a.rng_step_base + (a.rng_counter ? *a.rng_counter : 0ull);
    float x[dc::MAXD];
    load_obs_row(a.policy_obs, (size_t)a.t_begin * B + e, d, x);
    for (int t = a.t_begin; t < a.t_end; ++t) {
        float logit[MAX_OUT];
#pragma unroll
        for (int j = 0; j < MAX_OUT; ++j) logit[j] = 0.f;
        dc::deep_forward(a.policy_params, o, a.activation_id, x, nullptr, logit, nullptr, nullptr);
        const size_t grow = (size_t)t * B + e;
        if constexpr (HEAD == ORL_HEAD_GAUSSIAN) {
            gaussian_act(logit, n, a.policy_params + dc::logstd_offset(o), a.deterministic != 0, a.exp_noise, a.rng_seed,
                         rng_base + (uint64_t)t, (uint32_t)(e + a.rng_row_offset), grow, a.actions, a.action_log_probs);
        } else {
            float lp;
            const int act = sample_action(logit, n, a.action_masks ? a.action_masks + grow * n : nullptr, a.deterministic != 0,
                                          [&](float (&q)[MAX_OUT]) {
                                              action_noise(a.exp_noise, grow, n, a.rng_seed, rng_base + (uint64_t)t, (uint32_t)(e + a.rng_row_offset), q);
                                          }, lp);
            a.actions[grow] = (float)act;
            a.action_log_probs[grow] = lp;
            if constexpr (ENV != ORL_ENV_NONE) {
                bool done;
                const float4 o = step_insert_single(a, env_ptrs(a, a.rng_row_offset / a.n_agents), ENV, e, t, act, done);
                x[0] = o.x; x[1] = o.y; x[2] = o.z; x[3] = o.w;
            }
        }
    }
}

__global__ void __launch_bounds__(S_NT) share_values_kernel(const float* __restrict__ params, int d, int n, int activation_id,
                                                            const float* __restrict__ obs, float* __restrict__ values, long long rows) {
    const long long r = (long long)blockIdx.x * S_NT + threadIdx.x;
    if (r >= rows) return;
    const dc::Offsets o = dc::deep_offsets(d, n);
    float x[dc::MAXD];
    load_obs_row(obs, (size_t)r, d, x);
    float v;
    dc::deep_forward(params, o, activation_id, x, &v, nullptr, nullptr, nullptr);
    values[r] = v;
}

// ---- update: forward + both losses + backward of one minibatch row per thread -> tape row; loss sums -> loss_acc ----
// HEAD = ORL_HEAD_GAUSSIAN: gaussian_row's per-dimension loss, dL/dmean into the backward and the row's dL/dlogstd into
// the tape field TS_DLS of the wider Gaussian tape.
template <int HEAD>
__global__ void __launch_bounds__(S_NT) share_fwdbwd_kernel(const OrlPpoArgs a, float* __restrict__ tape, float* __restrict__ loss_part) {
    constexpr bool GAUSS = HEAD == ORL_HEAD_GAUSSIAN;
    const long long r = (long long)blockIdx.x * S_NT + threadIdx.x;
    const int d = a.obs_dim, n = a.n_actions;
    const dc::Offsets o = dc::deep_offsets(d, n, GAUSS);
    float l_pol = 0.f, l_ent = 0.f, l_ratio = 0.f, l_val = 0.f;
    if (r < a.batch_rows) {
        const long long gi = a.indices ? a.indices[r] : a.row_begin + r;
        const bool pol_masks = a.flags & ORL_PPO_POLICY_ACTIVE_MASKS, val_masks = a.flags & ORL_PPO_VALUE_ACTIVE_MASKS;
        const MbConsts mb = mb_consts(a);
        float x[dc::MAXD];
        load_obs_row(a.policy_obs, (size_t)gi, d, x);
        dc::Save sv;
        float value, logit[MAX_OUT];
#pragma unroll
        for (int j = 0; j < MAX_OUT; ++j) logit[j] = 0.f;
        float* tp = tape + (size_t)r * dc::tape_width(GAUSS);
        dc::deep_forward(a.policy_params, o, a.activation_id, x, &value, logit, &sv, tp);
        const float active = a.active_masks[gi];
        // policy loss (ppo.py:300-319) + entropy (act.py:150-168)
        const float wrow = mb.weight(pol_masks, active);
        float dl[MAX_OUT] = {};
        if constexpr (GAUSS) {
            // the entropy is the mean over rows and dimensions (act.py:150-158): weight active / sum(active) per dimension
            // with the active-mask option, else 1 / (rows n)
            const float went = pol_masks ? active * mb.inv_act : mb.inv_rows / (float)n;
            float dls[MAX_OUT] = {};
            gaussian_row(a, logit, n, a.policy_params + dc::logstd_offset(o), a.actions + gi * n, a.old_log_probs + gi * n,
                         apply_adv_norm(mb.adv, a.advantages[gi]), wrow, went, dl, dls, l_pol, l_ent, l_ratio);
#pragma unroll
            for (int j = 0; j < MAX_OUT; ++j) tp[dc::TS_DLS + j] = dls[j];
        } else {
            const CatRow c = categorical_row(a, logit, n, a.action_masks ? a.action_masks + gi * n : nullptr, (int)a.actions[gi],
                                             a.old_log_probs[gi], apply_adv_norm(mb.adv, a.advantages[gi]), wrow, dl);
            l_pol = c.loss * wrow; l_ent = c.ent * wrow; l_ratio = c.ratio;
        }
        // value loss (ppo.py:178-220)
        const float ret = a.returns[gi];
        const float target = (a.flags & ORL_PPO_VALUENORM) ? (ret - mb.vn_mean) / mb.vn_std : ret;
        const ValueTerm vt = value_term(value, a.value_preds[gi], target, a.clip_param, a.huber_delta, a.flags);
        const float wv = mb.weight(val_masks, active);
        l_val = vt.loss * wv;
        dc::deep_backward(a.policy_params, o, a.activation_id, sv, a.value_loss_coef * wv * vt.dv, dl, tp);
    }
    // block sums -> loss_part[block][slot], summed over the blocks by share_loss_sum_kernel
    __shared__ float red[4][S_NT / 32];
    float v[4] = {l_pol, l_ent, l_ratio, l_val};
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 4; ++k) { const float s = warp_sum(v[k]); if (lane == 0) red[k][warp] = s; }
    __syncthreads();
    if (threadIdx.x < 4) {
        float s = 0.f;
        for (int w = 0; w < S_NT / 32; ++w) s += red[threadIdx.x][w];
        loss_part[(size_t)blockIdx.x * 4 + threadIdx.x] = s;
    }
}

// The four loss sums over the update's blocks, in double and in a fixed order (deterministic).  One float atomic per
// block and slot drifted by up to 2e-5 relative at C2's 4096 blocks: the entropy's nearly equal block sums round alike
// against the growing total.  One CTA of S_NT threads per slot.
__global__ void __launch_bounds__(S_NT) share_loss_sum_kernel(const float* __restrict__ loss_part, int blocks, float* __restrict__ out) {
    const int k = blockIdx.x;
    double s = 0.0;
    for (int b = threadIdx.x; b < blocks; b += S_NT) s += (double)loss_part[(size_t)b * 4 + k];
    __shared__ double red[S_NT];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int w = S_NT / 2; w > 0; w >>= 1) {
        if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[k] = (float)red[0];
}

// ---- parameter gradients from the tape (orl::reduce_tape).  Every gemm job fits its tiles: the Q tiles end by TQ_Y7 + 64
// <= TAPE, the P tile of the M = 1 value head is TP_DV + 16 <= TAPE.  A Gaussian head adds the logstd column sum ----
TapeJobs make_share_jobs(int d, int n, bool gaussian) {
    const dc::Offsets o = dc::deep_offsets(d, n, gaussian);
    TapeJobs t; int g = 0, c = 0;
    auto gemm = [&](int p, int M, int q, int N, int out) { t.gemm[g++] = TapeJob{p, M, q, N, out}; };
    auto col = [&](int p, int M, int out) { t.col[c++] = TapeJob{p, M, -1, 1, out}; };
    gemm(dc::TP_DZ1, dc::H, dc::TQ_X, d, o.w1);       col(dc::TP_DZ1, dc::H, o.b1);  col(dc::TS_DY1N1, dc::H, o.g1); col(dc::TS_DY1, dc::H, o.be1);
    gemm(dc::TP_DZ3, dc::H, dc::TQ_Y1, dc::H, o.w3);  col(dc::TP_DZ3, dc::H, o.b3);  col(dc::TS_DY3N3, dc::H, o.g3); col(dc::TS_DY3, dc::H, o.be3);
    gemm(dc::TP_DZ5, dc::H, dc::TQ_Y3, dc::H, o.w5);  col(dc::TP_DZ5, dc::H, o.b5);  col(dc::TS_DY5N5, dc::H, o.g5); col(dc::TS_DY5, dc::H, o.be5);
    gemm(dc::TP_DZ7, dc::H, dc::TQ_Y5, dc::H, o.w7);  col(dc::TP_DZ7, dc::H, o.b7);  col(dc::TS_DY7N7, dc::H, o.g7); col(dc::TS_DY7, dc::H, o.be7);
    gemm(dc::TP_DV, 1, dc::TQ_Y7, dc::H, o.wv);       col(dc::TP_DV, 1, o.bv);
    gemm(dc::TP_DLOG, n, dc::TQ_Y7, dc::H, o.wa);     col(dc::TP_DLOG, n, o.ba);
    if (gaussian) col(dc::TS_DLS, n, dc::logstd_offset(o));
    t.n_gemm = g; t.n_col = c;
    return t;
}

// ---- optimiser: ppo.py:120-158 with a shared model — clip_grad_norm_(all) twice, one Adam step (lr = lrs[0]) ----
template <int HEAD>
__global__ void __launch_bounds__(1024) share_apply_kernel(const OrlPpoArgs a, const float* __restrict__ loss_acc) {
    const int total = dc::deep_offsets(a.obs_dim, a.n_actions, HEAD == ORL_HEAD_GAUSSIAN).total;
    float sq = 0.f;
    for (int i = threadIdx.x; i < total; i += blockDim.x) sq = fmaf(a.grads[i], a.grads[i], sq);
    const float norm1 = block_l2_norm(sq);   // actor_grad_norm: norm before the first clip
    const float c1 = clip_factor(a, norm1);
    const float norm2 = norm1 * c1;          // critic_grad_norm: what the second clip_grad_norm_ measures
    adam_step(a, 0, a.policy_params, a.policy_adam_m, a.policy_adam_v, a.grads, total, c1 * clip_factor(a, norm2));
    if (threadIdx.x == 0) {
        add_value_info(a, loss_acc[3], norm2);
        add_policy_info(a, loss_acc, norm1);
    }
}

}  // namespace

extern "C" {

int orl_share_param_count(int obs_dim, int n_actions) { return dc::deep_offsets(obs_dim, n_actions).total; }
int orl_share_param_count_head(int obs_dim, int n_actions, int head_kind) {
    return dc::deep_offsets(obs_dim, n_actions, head_kind == ORL_HEAD_GAUSSIAN).total;
}
int orl_share_tape_width(void) { return dc::TAPE; }
/* floats of the update workspace for a minibatch of `rows` rows: tape rows, then reduction partials, then the loss sums
 * of each share_fwdbwd_kernel block */
long long orl_share_workspace_floats_head(long long rows, int obs_dim, int n_actions, int head_kind) {
    const bool g = head_kind == ORL_HEAD_GAUSSIAN;
    const long long rb = (rows + TAPE_ROW_BLOCK - 1) / TAPE_ROW_BLOCK;
    return rows * dc::tape_width(g) + rb * (long long)((dc::deep_offsets(obs_dim, n_actions, g).total + 3) & ~3) +
           4 * ((rows + S_NT - 1) / S_NT);
}
long long orl_share_workspace_floats(long long rows, int obs_dim, int n_actions) {
    return orl_share_workspace_floats_head(rows, obs_dim, n_actions, ORL_HEAD_CATEGORICAL);
}

int orl_share_rollout(const OrlRolloutArgs* ap, void* stream) {
    ORL_CHECK_ARG(ap, "args");
    const OrlRolloutArgs& a = *ap;
    ORL_CHECK_ARG(a.n_envs > 0 && a.obs_dim > 0 && a.obs_dim <= dc::MAXD && a.n_actions > 0 && a.n_actions <= MAX_OUT, "shapes");
    ORL_CHECK_ARG(a.t_begin >= 0 && a.t_begin < a.t_end, "step range");
    ORL_CHECK_ARG(a.policy_params && a.policy_obs && a.actions && a.action_log_probs, "null buffer");
    ORL_CHECK_ARG(a.head_kind == ORL_HEAD_CATEGORICAL || (a.head_kind == ORL_HEAD_GAUSSIAN && a.env_kind == ORL_ENV_NONE),
                  "head_kind: Categorical, or DiagGaussian on host-stepped envs (ORL_ENV_NONE)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int B = a.n_envs * a.n_agents;
    const int grid = (B + S_NT - 1) / S_NT;
    const char* aligned = "policy_obs (and a separate critic_obs) must be 16-byte aligned";
    if (a.env_kind == ORL_ENV_NONE) {
        ORL_CHECK_ARG(a.t_end == a.t_begin + 1, "ORL_ENV_NONE acts for one step per call");
        if (a.head_kind == ORL_HEAD_GAUSSIAN) share_rollout_kernel<ORL_ENV_NONE, ORL_HEAD_GAUSSIAN><<<grid, S_NT, 0, st>>>(a);
        else share_rollout_kernel<ORL_ENV_NONE, ORL_HEAD_CATEGORICAL><<<grid, S_NT, 0, st>>>(a);
    } else if (a.env_kind == ORL_ENV_CARTPOLE) {
        ORL_CHECK_ARG(a.n_agents == 1 && a.obs_dim == 4 && a.n_actions == 2 && a.env_f64 && a.env_u64 && a.env_i32, "CartPole shapes / state");
        ORL_CHECK_ARG(single_obs_aligned(a), aligned);
        share_rollout_kernel<ORL_ENV_CARTPOLE, ORL_HEAD_CATEGORICAL><<<grid, S_NT, 0, st>>>(a);
    } else if (a.env_kind == ORL_ENV_GRIDWORLD) {
        ORL_CHECK_ARG(a.n_agents == 1 && a.obs_dim == 4 && a.n_actions == 5 && a.env_i32, "GridWorld shapes / state");
        ORL_CHECK_ARG(single_obs_aligned(a), aligned);
        share_rollout_kernel<ORL_ENV_GRIDWORLD, ORL_HEAD_CATEGORICAL><<<grid, S_NT, 0, st>>>(a);
    } else {
        orl::set_last_error("orl_share_rollout: env_kind %d is not built for the shared model (single-agent device envs and ORL_ENV_NONE are)", a.env_kind);
        return ORL_ERR_UNSUPPORTED;
    }
    ORL_LAUNCH_CHECK("share_rollout_kernel");
    return orl::bump_rng_counter(a.rng_counter, a.t_end - a.t_begin, st);
}

int orl_share_values(const float* params, int obs_dim, int n_actions, int activation_id, const float* obs, float* values, long long rows,
                     void* stream) {
    ORL_CHECK_ARG(params && obs && values && rows > 0, "null buffer / rows");
    ORL_CHECK_ARG(obs_dim > 0 && obs_dim <= dc::MAXD && n_actions > 0 && n_actions <= MAX_OUT, "shapes");
    share_values_kernel<<<(unsigned)((rows + S_NT - 1) / S_NT), S_NT, 0, reinterpret_cast<cudaStream_t>(stream)>>>(params, obs_dim, n_actions,
                                                                                                               activation_id, obs, values, rows);
    ORL_LAUNCH_CHECK("share_values_kernel");
    return 0;
}

/* forward + losses + backward + deterministic gradient reduction: args->policy_* = the shared model, args->partials =
 * workspace (orl_share_workspace_floats), args->grads = true gradients (out), args->folded[0..3] = loss sums (out) */
int orl_share_fwdbwd(const OrlPpoArgs* ap, void* stream) {
    ORL_CHECK_ARG(ap, "args");
    const OrlPpoArgs& a = *ap;
    ORL_CHECK_ARG(a.obs_dim > 0 && a.obs_dim <= dc::MAXD && a.n_actions > 0 && a.n_actions <= MAX_OUT && a.batch_rows > 0, "shapes");
    ORL_CHECK_ARG(a.policy_params && a.partials && a.folded && a.grads && a.policy_obs && a.actions && a.old_log_probs && a.advantages &&
                      a.value_preds && a.returns && a.active_masks && a.gae_stats && a.mb_stats, "null buffer");
    ORL_CHECK_ARG(a.head_kind == ORL_HEAD_CATEGORICAL || a.head_kind == ORL_HEAD_GAUSSIAN, "head_kind");
    ORL_CHECK_ARG(!(a.flags & ORL_PPO_VALUENORM) || a.vn_state, "vn_state required with VALUENORM");   // read by mb_consts
    ORL_CHECK_ARG(a.indices || (a.row_begin >= 0 && a.row_begin + a.batch_rows <= a.total_rows), "row range");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const bool g = a.head_kind == ORL_HEAD_GAUSSIAN;
    const int width = dc::tape_width(g);
    float* tape = a.partials;
    const long long rows = a.batch_rows;
    const int total = dc::deep_offsets(a.obs_dim, a.n_actions, g).total, stride = (total + 3) & ~3;
    float* partials = tape + (size_t)rows * width;
    const unsigned grid = (unsigned)((rows + S_NT - 1) / S_NT);
    float* loss_part = partials + (size_t)((rows + TAPE_ROW_BLOCK - 1) / TAPE_ROW_BLOCK) * stride;
    int e = orl::check_cuda(cudaMemsetAsync(a.folded, 0, 8 * sizeof(float), st), "memset loss sums");
    if (e) return e;
    if (g) share_fwdbwd_kernel<ORL_HEAD_GAUSSIAN><<<grid, S_NT, 0, st>>>(a, tape, loss_part);
    else share_fwdbwd_kernel<ORL_HEAD_CATEGORICAL><<<grid, S_NT, 0, st>>>(a, tape, loss_part);
    ORL_LAUNCH_CHECK("share_fwdbwd_kernel");
    share_loss_sum_kernel<<<4, S_NT, 0, st>>>(loss_part, (int)grid, a.folded);
    ORL_LAUNCH_CHECK("share_loss_sum_kernel");
    return orl::reduce_tape(tape, width, rows, make_share_jobs(a.obs_dim, a.n_actions, g), partials, stride, total, a.grads, st);
}

int orl_share_apply(const OrlPpoArgs* ap, void* stream) {
    ORL_CHECK_ARG(ap, "args");
    const OrlPpoArgs& a = *ap;
    ORL_CHECK_ARG(a.policy_params && a.policy_adam_m && a.policy_adam_v && a.adam_steps && a.lrs && a.grads && a.folded && a.train_info && a.mb_stats,
                  "null buffer");
    ORL_CHECK_ARG(a.head_kind == ORL_HEAD_CATEGORICAL || a.head_kind == ORL_HEAD_GAUSSIAN, "head_kind");
    ORL_CHECK_ARG(!(a.flags & ORL_PPO_VALUENORM) || a.vn_state, "vn_state required with VALUENORM");   // written by add_value_info
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (a.head_kind == ORL_HEAD_GAUSSIAN) share_apply_kernel<ORL_HEAD_GAUSSIAN><<<1, 1024, 0, st>>>(a, a.folded);
    else share_apply_kernel<ORL_HEAD_CATEGORICAL><<<1, 1024, 0, st>>>(a, a.folded);
    ORL_LAUNCH_CHECK("share_apply_kernel");
    return 0;
}

}  // extern "C"
