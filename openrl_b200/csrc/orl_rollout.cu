// Fused rollout kernel: policy MLP forward + action sampling (categorical, or DiagGaussian on host-stepped envs) +
// device env.step + in-place buffer insert, for steps [t_begin, t_end) of one rollout of simple_spread or of host-stepped
// envs (ORL_ENV_NONE: act only; CartPole and GridWorld run the tensor-core rollouts of orl_fwd_tc.cu), plus env reset and
// the FFMA row-batch forward of the critic values (obs_dim > 8) and the policy eval.  See include/openrl_b200.h for the
// reference functions this replaces.
//
// Mapping: a CTA of 128 threads owns ROWS = 32 consecutive rows (env, agent) for the whole step
// range — envs never interact, so there is no grid-wide dependency and ONE launch covers all T
// steps; the policy weights (folded, 37 KB) stay resident in shared memory.  Per step the trunk is
// two register-tiled tile GEMMs (32x64xd, 32x64x64; see orl_mlp.cuh), then 4 lanes per row compute
// the logits, one lane samples and steps the env, writing slot t / t+1 of the buffers directly.
// The step chain is latency-bound (T sequential steps); the grid is N*A/32 CTAs.
#include "orl_envstep.cuh"

namespace {
using namespace orl;

constexpr int R_NT = 128;  // threads per CTA; rows per CTA R_M is a template parameter (8 / 16 / 32)


__global__ void env_step_mpe_kernel(int N, EnvPtrs E, const float* __restrict__ actions, float* __restrict__ obs_out,
                                    float* __restrict__ critic_obs_out, float* __restrict__ rewards_out,
                                    float* __restrict__ dones_out) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= N) return;
    const int acts[3] = {(int)actions[e * 3], (int)actions[e * 3 + 1], (int)actions[e * 3 + 2]};
    float ob[3][18], reward; bool done;
    env_step_mpe(E, e, N, acts, ob, reward, done);
    for (int ag = 0; ag < 3; ++ag) {
        mpe_insert_obs(ob[ag], ag, (size_t)e * 3, obs_out, critic_obs_out);
        rewards_out[e * 3 + ag] = reward;
        dones_out[e * 3 + ag] = done ? 1.f : 0.f;
    }
}

__global__ void env_step_kernel(int kind, int N, EnvPtrs E, const float* __restrict__ actions, float* __restrict__ obs_out,
                                float* __restrict__ rewards_out, float* __restrict__ dones_out, float* __restrict__ final_obs_out) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= N) return;
    float ob[4], fin[4], reward; bool done;
    env_step_single(E, kind, e, N, (int)actions[e], ob, reward, done, fin);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        obs_out[(size_t)e * 4 + k] = ob[k];
        if (final_obs_out) final_obs_out[(size_t)e * 4 + k] = fin[k];
    }
    rewards_out[e] = reward;
    dones_out[e] = done ? 1.f : 0.f;
}


// ENV of the host act (ORL_ENV_NONE) for observations of 65..256 features: fc1 in panels (orl_mlp.cuh, fc1_panels) in
// the buffers of the d = 64 layout
constexpr int ENV_NONE_WIDE_OBS = -1;

// NB: head width bound (orl_mlp.cuh); NB = 64 is the wide Categorical head of host-stepped envs (ORL_ENV_NONE), whose
// logits tile reuses N1s once the trunk is done with it.
template <int R_M, int ENV, int NB = MAX_OUT>
__global__ void __launch_bounds__(R_NT) rollout_kernel(const OrlRolloutArgs a) {
    constexpr bool PANELS = ENV == ENV_NONE_WIDE_OBS;
    extern __shared__ __align__(16) float smem[];
    const int N = a.n_envs, A = a.n_agents, B = N * A, d = a.obs_dim, n = a.n_actions;
    const int ldx = PANELS ? LDX_PANEL : pad4(d) + 4;
    float* p = smem;
    SmemWeights w = carve_weights<NB>(p, PANELS ? OBS_PANEL : d, false);
    float* Xs = p;  p += R_M * ldx;
    float* N1s = p; p += R_M * LDA;
    float* N3s = p; p += R_M * LDA;
    int* act_s = reinterpret_cast<int*>(p); p += R_M;

    // rows of this CTA: whole envs only
    const int envs_per_cta = R_M / A;
    const int env0 = blockIdx.x * envs_per_cta;
    const int n_env_here = min(envs_per_cta, N - env0);
    const int row0 = env0 * A;
    const int rows_here = n_env_here * A;
    const int tid = threadIdx.x;

    load_weights_folded<R_NT, NB, PANELS>(w, a.policy_params, d, n, false);   // (the logstd tail, if any, is read directly)

    // stage obs of slot t_begin (zero padding for the k tail and for idle rows); a panelled fc1 stages its own
    if constexpr (!PANELS) {
        for (int i = tid; i < R_M * ldx; i += R_NT) {
            const int r = i / ldx, k = i % ldx;
            Xs[i] = (r < rows_here && k < d) ? a.policy_obs[((size_t)a.t_begin * B + row0 + r) * d + k] : 0.f;
        }
        __syncthreads();
    }

    constexpr int PPR = R_NT / R_M;
    const int hrow = tid / PPR, hpart = tid % PPR;
    const uint64_t rng_base = a.rng_step_base + (a.rng_counter ? *a.rng_counter : 0ull);

    for (int t = a.t_begin; t < a.t_end; ++t) {
        float mu1[R_M / (R_NT / 16)], rstd1[R_M / (R_NT / 16)], rstd3[R_M / (R_NT / 16)];
        unsigned pm;
        if constexpr (PANELS) {   // ORL_ENV_NONE: t == t_begin, the one step of the call
            float acc[R_M / (R_NT / 16)][4];
            fc1_panels<R_M, R_NT>(w, a.policy_params + net_offsets(d, n).w1, d, Xs, [&](int r) -> const float* {
                return r < rows_here ? a.policy_obs + ((size_t)t * B + row0 + r) * d : nullptr;
            }, acc);
            trunk_from_z1<R_M, R_NT, false>(w, acc, a.activation_id, N1s, N3s, mu1, rstd1, rstd3, pm);
        } else {
            trunk_forward<R_M, R_NT, false>(w, Xs, ldx, d, a.activation_id, N1s, N3s, mu1, rstd1, rstd3, pm);
        }
        __syncthreads();
        if constexpr (NB == MAX_OUT_WIDE) {
            static_assert(ENV == ORL_ENV_NONE || PANELS, "wide heads act on host-stepped envs");
            head_tile<R_M, R_NT>(w, N3s, N1s);
            __syncthreads();
            if (tid < rows_here) {   // one thread per row
                const size_t grow = (size_t)t * B + row0 + tid;
                const uint64_t step = rng_base + (uint64_t)t;
                const uint32_t grow32 = (uint32_t)(row0 + tid + a.rng_row_offset);
                float lp;
                const int act = wide_sample_action(N1s + tid * LDA, n, a.action_masks ? a.action_masks + grow * n : nullptr,
                                                   a.deterministic != 0, [&](int j0, float (&q)[4]) {
                                                       wide_action_noise4(a.exp_noise, grow, n, a.rng_seed, step, grow32, j0, q);
                                                   }, lp);
                a.actions[grow] = (float)act;
                a.action_log_probs[grow] = lp;
            }
            __syncthreads();
            continue;
        }
        float logit[MAX_OUT];
        head_dots<R_M, R_NT>(w, N3s, n, logit);
        if (hpart == 0 && hrow < rows_here && a.head_kind == ORL_HEAD_GAUSSIAN)
            gaussian_act(logit, n, a.policy_params + net_offsets(d, n, 1).ls, a.deterministic != 0, a.exp_noise, a.rng_seed,
                         rng_base + (uint64_t)t, (uint32_t)(row0 + hrow + a.rng_row_offset), (size_t)t * B + row0 + hrow, a.actions,
                         a.action_log_probs);
        if (hpart == 0 && hrow < rows_here && a.head_kind != ORL_HEAD_GAUSSIAN) {
            const size_t grow = (size_t)t * B + row0 + hrow;
            float lp;
            const int act = sample_action(logit, n, a.action_masks ? a.action_masks + grow * n : nullptr, a.deterministic != 0,
                                          [&](float (&q)[MAX_OUT]) {
                                              action_noise(a.exp_noise, grow, n, a.rng_seed, rng_base + (uint64_t)t,
                                                           (uint32_t)(row0 + hrow + a.rng_row_offset), q);
                                          }, lp);
            a.actions[grow] = (float)act;
            a.action_log_probs[grow] = lp;
            act_s[hrow] = act;
        }
        __syncthreads();

        // ---- env.step for the envs of this CTA (one thread per env) ----
        if constexpr (ENV == ORL_ENV_MPE_SPREAD) {
            if (tid < n_env_here) {
                const int acts[3] = {act_s[tid * 3], act_s[tid * 3 + 1], act_s[tid * 3 + 2]};
                step_insert_mpe(a, env_ptrs(a, a.rng_row_offset / A), env0 + tid, t, acts,
                                [&](int ag, int k, float v) { Xs[(tid * 3 + ag) * ldx + k] = v; });
            }
        }
        __syncthreads();
    }
}

__global__ void env_reset_kernel(int env_kind, int N, double* env_f64, uint64_t* env_u64, int32_t* env_i32,
                                 const int32_t* env_table, int env_table_len, uint64_t seed, float* obs_out,
                                 float* critic_obs_out) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= N) return;
    if (env_kind == ORL_ENV_MPE_SPREAD) {
        MpeState s;
        Pcg64 g = pcg_load(env_u64, e, N);
        mpe_reset(s, g);
        pcg_store(env_u64, e, N, g);
        mpe_store(env_f64, e, N, s);
        env_i32[e] = 0;
        for (int ag = 0; ag < 3; ++ag) {
            float o[18];
            mpe_obs(s, ag, o);
            mpe_insert_obs(o, ag, (size_t)e * 3, obs_out, critic_obs_out);
        }
        return;
    }
    if (env_kind == ORL_ENV_CARTPOLE) {
        double s[4];
        Pcg64 g = pcg_load(env_u64, e, N);
        cartpole_reset(s, g);
        pcg_store(env_u64, e, N, g);
#pragma unroll
        for (int k = 0; k < 4; ++k) { env_f64[(size_t)k * N + e] = s[k]; obs_out[(size_t)e * 4 + k] = (float)s[k]; }
        env_i32[e] = 0;
    } else if (env_kind == ORL_ENV_GRIDWORLD) {
        int x, y, nreset = env_i32[3 * N + e];
        gridworld_reset(x, y, e, nreset, seed, env_table, env_table_len, 10, 10);
        env_i32[0 * N + e] = x; env_i32[1 * N + e] = y; env_i32[2 * N + e] = 0; env_i32[3 * N + e] = nreset + 1;
        obs_out[(size_t)e * 4 + 0] = (float)x; obs_out[(size_t)e * 4 + 1] = (float)y;
        obs_out[(size_t)e * 4 + 2] = 1.f; obs_out[(size_t)e * 4 + 3] = 1.f;
    }
}

// ---- FFMA row-batch forward: the MLP of one net over a flat batch of rows ------------------------------------------------
// Persistent CTAs of C_NT threads walk tiles of C_M rows (grid-stride); per tile the trunk and the n head dots, then
// epilogue(g, out) on the thread that owns row g, with out[0..n) the head outputs of that row.
constexpr int C_M = 128, C_NT = 256;

// NB = 64 (wide Categorical heads): the logits go to a tile in N1s and epilogue(g, x) gets the row's logits x[0..n) there.
// PANELS: observations of 65..256 features, fc1 in panels (orl_mlp.cuh, fc1_panels) in the buffers of the d = 64 layout.
template <int NB = MAX_OUT, bool PANELS = false, typename Epilogue>
__device__ __forceinline__ void rows_forward(const float* __restrict__ params, int d, int n, int activation_id,
                                             const float* __restrict__ obs, long long rows, Epilogue&& epilogue) {
    extern __shared__ __align__(16) float smem[];
    const int ldx = PANELS ? LDX_PANEL : pad4(d) + 4;
    float* p = smem;
    SmemWeights w = carve_weights<NB>(p, PANELS ? OBS_PANEL : d, false);
    float* Xs = p;  p += C_M * ldx;
    float* N1s = p; p += C_M * LDA;
    float* N3s = p; p += C_M * LDA;
    const int tid = threadIdx.x;
    load_weights_folded<C_NT, NB, PANELS>(w, params, d, n, false);
    const long long n_tiles = (rows + C_M - 1) / C_M;
    for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const long long r0 = tile * C_M;
        const int rows_here = (int)min((long long)C_M, rows - r0);
        float mu1[C_M / (C_NT / 16)], rstd1[C_M / (C_NT / 16)], rstd3[C_M / (C_NT / 16)];
        unsigned pm;
        if constexpr (PANELS) {
            float acc[C_M / (C_NT / 16)][4];
            fc1_panels<C_M, C_NT>(w, params + net_offsets(d, n).w1, d, Xs,
                                  [&](int r) -> const float* { return r < rows_here ? obs + (r0 + r) * d : nullptr; }, acc);
            trunk_from_z1<C_M, C_NT, false>(w, acc, activation_id, N1s, N3s, mu1, rstd1, rstd3, pm);
        } else {
            for (int i = tid; i < C_M * ldx; i += C_NT) {
                const int r = i / ldx, k = i % ldx;
                Xs[i] = (r < rows_here && k < d) ? obs[(r0 + r) * d + k] : 0.f;
            }
            __syncthreads();
            trunk_forward<C_M, C_NT, false>(w, Xs, ldx, d, activation_id, N1s, N3s, mu1, rstd1, rstd3, pm);
        }
        __syncthreads();
        if constexpr (NB == MAX_OUT_WIDE) {
            head_tile<C_M, C_NT>(w, N3s, N1s);
            __syncthreads();
            if (tid < rows_here) epilogue(r0 + tid, N1s + tid * LDA);
        } else {
            float out[MAX_OUT];
            head_dots<C_M, C_NT>(w, N3s, n, out);
            constexpr int PPR = C_NT / C_M;
            if (tid % PPR == 0 && tid / PPR < rows_here) epilogue(r0 + tid / PPR, out);
        }
        __syncthreads();
    }
}

// ValueNetwork.forward (value_network.py:113-136)
template <bool PANELS>
__device__ __forceinline__ void critic_values_body(const float* __restrict__ params, int d, int activation_id,
                                                   const float* __restrict__ obs, float* __restrict__ values, long long rows) {
    rows_forward<MAX_OUT, PANELS>(params, d, 1, activation_id, obs, rows, [&](long long g, float (&out)[MAX_OUT]) { values[g] = out[0]; });
}
__global__ void __launch_bounds__(C_NT) critic_values_kernel(const float* __restrict__ params, int d, int activation_id,
                                                             const float* __restrict__ obs, float* __restrict__ values,
                                                             long long rows) {
    critic_values_body<false>(params, d, activation_id, obs, values, rows);
}
__global__ void __launch_bounds__(C_NT) critic_values_wide_obs_kernel(const float* __restrict__ params, int d, int activation_id,
                                                                      const float* __restrict__ obs, float* __restrict__ values,
                                                                      long long rows) {
    critic_values_body<true>(params, d, activation_id, obs, values, rows);
}

// PolicyNetwork.eval_actions (policy_network.py:164-203, act.py:160-168 / 150-158): the log-prob of the given action and
// the entropy of the action distribution per row (the caller takes the masked mean); per dimension for a Gaussian head.
template <bool PANELS>
__device__ __forceinline__ void policy_eval_body(const float* __restrict__ params, int d, int n, int activation_id, int head_kind,
                                                 const float* __restrict__ obs, const float* __restrict__ actions,
                                                 const float* __restrict__ action_masks, float* __restrict__ logp_out,
                                                 float* __restrict__ entropy_out, long long rows) {
    const float* logstd = params + net_offsets(d, n, 1).ls;
    rows_forward<MAX_OUT, PANELS>(params, d, n, activation_id, obs, rows, [&](long long g, float (&out)[MAX_OUT]) {
        if (head_kind == ORL_HEAD_GAUSSIAN) {
            for (int j = 0; j < n; ++j) {
                const float ls = logstd[j];
                logp_out[g * n + j] = gaussian_log_prob(actions[g * n + j] - out[j], expf(ls), ls);
                entropy_out[g * n + j] = gaussian_entropy(ls);
            }
        } else {
            float nl[MAX_OUT], pr[MAX_OUT];
            masked_log_softmax(out, n, action_masks ? action_masks + g * n : nullptr, nl, pr);
            logp_out[g] = log_prob_of(nl, n, (int)actions[g]);
            entropy_out[g] = categorical_entropy(nl, pr, n);
        }
    });
}
__global__ void __launch_bounds__(C_NT) policy_eval_kernel(const float* __restrict__ params, int d, int n, int activation_id, int head_kind,
                                                           const float* __restrict__ obs, const float* __restrict__ actions,
                                                           const float* __restrict__ action_masks, float* __restrict__ logp_out,
                                                           float* __restrict__ entropy_out, long long rows) {
    policy_eval_body<false>(params, d, n, activation_id, head_kind, obs, actions, action_masks, logp_out, entropy_out, rows);
}
__global__ void __launch_bounds__(C_NT) policy_eval_wide_obs_kernel(const float* __restrict__ params, int d, int n, int activation_id,
                                                                    int head_kind, const float* __restrict__ obs,
                                                                    const float* __restrict__ actions, const float* __restrict__ action_masks,
                                                                    float* __restrict__ logp_out, float* __restrict__ entropy_out, long long rows) {
    policy_eval_body<true>(params, d, n, activation_id, head_kind, obs, actions, action_masks, logp_out, entropy_out, rows);
}

// policy_eval_kernel of a wide Categorical head (9..64 actions)
template <bool PANELS>
__device__ __forceinline__ void policy_eval_wide_body(const float* __restrict__ params, int d, int n, int activation_id,
                                                      const float* __restrict__ obs, const float* __restrict__ actions,
                                                      const float* __restrict__ action_masks, float* __restrict__ logp_out,
                                                      float* __restrict__ entropy_out, long long rows) {
    rows_forward<MAX_OUT_WIDE, PANELS>(params, d, n, activation_id, obs, rows, [&](long long g, float* x) {
        const WideSoftmax sm = wide_log_softmax(x, n, action_masks ? action_masks + g * n : nullptr);
        logp_out[g] = wide_log_prob_of(sm, x, n, (int)actions[g]);
        entropy_out[g] = wide_entropy(sm, x, n);
    });
}
__global__ void __launch_bounds__(C_NT) policy_eval_wide_kernel(const float* __restrict__ params, int d, int n, int activation_id,
                                                                const float* __restrict__ obs, const float* __restrict__ actions,
                                                                const float* __restrict__ action_masks, float* __restrict__ logp_out,
                                                                float* __restrict__ entropy_out, long long rows) {
    policy_eval_wide_body<false>(params, d, n, activation_id, obs, actions, action_masks, logp_out, entropy_out, rows);
}
__global__ void __launch_bounds__(C_NT) policy_eval_wide_wide_obs_kernel(const float* __restrict__ params, int d, int n, int activation_id,
                                                                         const float* __restrict__ obs, const float* __restrict__ actions,
                                                                         const float* __restrict__ action_masks, float* __restrict__ logp_out,
                                                                         float* __restrict__ entropy_out, long long rows) {
    policy_eval_wide_body<true>(params, d, n, activation_id, obs, actions, action_masks, logp_out, entropy_out, rows);
}

// ---- insert of one host env.step into the rollout buffer (OnPolicyDriver.add2buffer, onpolicy_driver.py:80-152) -----------
// staged = [obs (B*d) (| critic obs (B*dc)) | rewards (B) | dones (B) (| action masks (B*n))] as uploaded from the host in
// ONE copy; one thread per row.  Row r of the insert; returns whether every agent of the row's env is done.  The critic
// section is present (and critic_obs_next non-null) only for envs with a Dict {"policy", "critic"} observation space.  The
// masks block is present (and action_masks_next non-null) only when the envs reported masks for this step; otherwise slot
// t+1 keeps what it held.
__device__ __forceinline__ bool host_insert_row(const float* __restrict__ staged, int n_envs, int n_agents, int d, int r,
                                                float* __restrict__ obs_next, float* __restrict__ rewards,
                                                float* __restrict__ masks_next, float* __restrict__ active_next,
                                                float* __restrict__ action_masks_next, int n,
                                                float* __restrict__ critic_next, int dc) {
    const int B = n_envs * n_agents;
    const float* so = staged;
    const float* sr = staged + (size_t)B * d;
    if (critic_next) {
        const float* sc = sr;
        for (int k = 0; k < dc; ++k) critic_next[(size_t)r * dc + k] = sc[(size_t)r * dc + k];
        sr += (size_t)B * dc;
    }
    const float* sd = sr + B;
    for (int k = 0; k < d; ++k) obs_next[(size_t)r * d + k] = so[(size_t)r * d + k];
    if (action_masks_next) {
        const float* sm = sd + B;
        for (int k = 0; k < n; ++k) action_masks_next[(size_t)r * n + k] = sm[(size_t)r * n + k];
    }
    rewards[r] = sr[r];
    const int e = r / n_agents;
    bool all_done = true;
    for (int a = 0; a < n_agents; ++a) all_done = all_done && (sd[e * n_agents + a] != 0.f);
    const bool done = sd[r] != 0.f;
    masks_next[r] = all_done ? 0.f : 1.f;                    // masks[dones_env] = 0
    active_next[r] = (done && !all_done) ? 0.f : 1.f;        // active[dones] = 0, active[dones_env] = 1
    return all_done;
}

__global__ void host_insert_kernel(const float* __restrict__ staged, int n_envs, int n_agents, int d, float* __restrict__ obs_next,
                                   float* __restrict__ rewards, float* __restrict__ masks_next, float* __restrict__ active_next,
                                   float* __restrict__ action_masks_next, int n, float* __restrict__ critic_next, int dc) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_envs * n_agents) return;
    host_insert_row(staged, n_envs, n_agents, d, r, obs_next, rewards, masks_next, active_next, action_masks_next, n,
                    critic_next, dc);
}

// the same insert for a recurrent policy: rnn_states[t+1] of every agent of a finished env is zeroed (onpolicy_driver.py:262-269)
constexpr int RNN_HIDDEN = 64;   // OrlRnnArgs.rnn_states rows
__global__ void host_insert_rnn_kernel(const float* __restrict__ staged, int n_envs, int n_agents, int d, float* __restrict__ obs_next,
                                       float* __restrict__ rewards, float* __restrict__ masks_next, float* __restrict__ active_next,
                                       float* __restrict__ rnn_next, float* __restrict__ action_masks_next, int n,
                                       float* __restrict__ critic_next, int dc) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_envs * n_agents) return;
    if (host_insert_row(staged, n_envs, n_agents, d, r, obs_next, rewards, masks_next, active_next, action_masks_next, n,
                        critic_next, dc)) {
        float4* h = reinterpret_cast<float4*>(rnn_next + (size_t)r * RNN_HIDDEN);
#pragma unroll
        for (int k = 0; k < RNN_HIDDEN / 4; ++k) h[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

// launch of a row-batch forward kernel over `rows` rows of obs_dim d: grid = min(tiles, 2 x SMs).  A panelled kernel
// (d > 64) takes the layout of d = 64.
template <int NB = MAX_OUT, typename... Params, typename... Args>
int launch_rows_forward(void (*kern)(Params...), const char* name, int d, long long rows, cudaStream_t st, Args... args) {
    d = std::min(d, OBS_PANEL);
    const int ldx = pad4(d) + 4;
    const size_t smem = sizeof(float) * (smem_weights_floats<NB>(d, false) + C_M * ldx + 2 * C_M * LDA);
    if (int e = allow_dynamic_smem(kern, 200 * 1024)) return e;
    const long long n_tiles = (rows + C_M - 1) / C_M;
    const int grid = (int)std::min<long long>(n_tiles, 2LL * sm_count());
    kern<<<grid, C_NT, smem, st>>>(args...);
    ORL_LAUNCH_CHECK(name);
    return 0;
}

}  // namespace

namespace orl {
int launch_rollout_tc(const OrlRolloutArgs& a, cudaStream_t st);
int launch_critic_values_tc(const float* params, int d, int activation_id, const float* obs, float* values, long long rows, cudaStream_t st);
}  // namespace orl

extern "C" int orl_env_reset(int env_kind, int n_envs, int n_agents, double* env_f64, uint64_t* env_u64,
                             int32_t* env_i32, const int32_t* env_table, int env_table_len, uint64_t rng_seed,
                             float* policy_obs_out, float* critic_obs_out, void* stream) {
    ORL_CHECK_ARG(n_envs > 0 && n_agents > 0, "n_envs/n_agents");
    ORL_CHECK_ARG(policy_obs_out, "policy_obs_out");
    if (env_kind == ORL_ENV_CARTPOLE) ORL_CHECK_ARG(env_f64 && env_u64 && env_i32 && n_agents == 1, "cartpole state");
    else if (env_kind == ORL_ENV_GRIDWORLD) ORL_CHECK_ARG(env_i32 && n_agents == 1, "gridworld state");
    else if (env_kind == ORL_ENV_MPE_SPREAD) ORL_CHECK_ARG(env_f64 && env_u64 && env_i32 && n_agents == 3, "simple_spread state");
    else { orl::set_last_error("orl_env_reset: unsupported env_kind %d", env_kind); return ORL_ERR_UNSUPPORTED; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    env_reset_kernel<<<(n_envs + 127) / 128, 128, 0, st>>>(env_kind, n_envs, env_f64, env_u64, env_i32, env_table,
                                                          env_table_len, rng_seed, policy_obs_out, critic_obs_out);
    ORL_LAUNCH_CHECK("env_reset_kernel");
    return 0;
}


extern "C" int orl_env_step(int env_kind, int n_envs, int n_agents, double* env_f64, uint64_t* env_u64, int32_t* env_i32,
                            const int32_t* env_table, int env_table_len, uint64_t rng_seed, float* ep_return,
                            int32_t* ep_length, double* episode_stats, const float* actions, float* obs_out,
                            float* rewards_out, float* dones_out, float* final_obs_out, void* stream) {
    ORL_CHECK_ARG(n_envs > 0, "n_envs");
    ORL_CHECK_ARG(actions && obs_out && rewards_out && dones_out && ep_return && ep_length && episode_stats, "null buffer");
    if (env_kind == ORL_ENV_MPE_SPREAD) {
        ORL_CHECK_ARG(n_agents == 3 && env_f64 && env_u64 && env_i32, "simple_spread state");
        EnvPtrs Em{env_f64, env_u64, env_i32, env_table, env_table_len, rng_seed, ep_return, ep_length, episode_stats};
        // final_obs_out doubles as the critic observation output (B, 54) for this env kind
        env_step_mpe_kernel<<<(n_envs + 127) / 128, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
            n_envs, Em, actions, obs_out, final_obs_out, rewards_out, dones_out);
        ORL_LAUNCH_CHECK("env_step_mpe_kernel");
        return 0;
    }
    ORL_CHECK_ARG(n_agents == 1, "n_agents");
    if (env_kind == ORL_ENV_CARTPOLE) ORL_CHECK_ARG(env_f64 && env_u64 && env_i32, "cartpole state");
    else if (env_kind == ORL_ENV_GRIDWORLD) ORL_CHECK_ARG(env_i32, "gridworld state");
    else { orl::set_last_error("orl_env_step: unsupported env_kind %d", env_kind); return ORL_ERR_UNSUPPORTED; }
    EnvPtrs E{env_f64, env_u64, env_i32, env_table, env_table_len, rng_seed, ep_return, ep_length, episode_stats};
    env_step_kernel<<<(n_envs + 127) / 128, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        env_kind, n_envs, E, actions, obs_out, rewards_out, dones_out, final_obs_out);
    ORL_LAUNCH_CHECK("env_step_kernel");
    return 0;
}

extern "C" int orl_rollout(const OrlRolloutArgs* args, void* stream) {
    ORL_CHECK_ARG(args, "args");
    const OrlRolloutArgs& a = *args;
    ORL_CHECK_ARG(a.n_envs > 0 && a.n_agents > 0 && a.n_agents <= 32, "n_envs / n_agents");
    ORL_CHECK_ARG(a.obs_dim > 0 && a.obs_dim <= orl::MAX_OBS_WIDE, "obs_dim must be in 1..256");
    ORL_CHECK_ARG(a.obs_dim <= orl::OBS_PANEL || a.env_kind == ORL_ENV_NONE,
                  "obs_dim must be in 1..64 (65..256: host-stepped envs, ORL_ENV_NONE)");
    ORL_CHECK_ARG(a.n_actions > 0 && a.n_actions <= orl::MAX_OUT_WIDE, "n_actions must be in 1..64");
    ORL_CHECK_ARG(a.n_actions <= orl::MAX_OUT || (a.env_kind == ORL_ENV_NONE && a.head_kind == ORL_HEAD_CATEGORICAL),
                  "n_actions must be in 1..8 (9..64: Categorical heads on host-stepped envs, ORL_ENV_NONE)");
    ORL_CHECK_ARG(a.t_begin >= 0 && a.t_begin < a.t_end && a.t_end <= a.episode_length, "step range");
    ORL_CHECK_ARG(a.activation_id >= 0 && a.activation_id <= 3, "activation_id");
    ORL_CHECK_ARG(a.policy_params && a.policy_obs && a.actions && a.action_log_probs, "null buffer");
    ORL_CHECK_ARG(a.head_kind == ORL_HEAD_CATEGORICAL || (a.head_kind == ORL_HEAD_GAUSSIAN && a.env_kind == ORL_ENV_NONE),
                  "Gaussian heads act on host-stepped envs (ORL_ENV_NONE)");
    if (a.env_kind == ORL_ENV_NONE) {
        ORL_CHECK_ARG(a.t_end == a.t_begin + 1, "ORL_ENV_NONE acts for one step per call");
    } else if (a.env_kind == ORL_ENV_CARTPOLE) {
        ORL_CHECK_ARG(a.n_agents == 1 && a.obs_dim == 4 && a.n_actions == 2, "CartPole shapes");
        ORL_CHECK_ARG(a.env_f64 && a.env_u64 && a.env_i32 && a.rewards && a.masks && a.active_masks && a.ep_return &&
                          a.ep_length && a.episode_stats, "CartPole state buffers");
    } else if (a.env_kind == ORL_ENV_GRIDWORLD) {
        ORL_CHECK_ARG(a.n_agents == 1 && a.obs_dim == 4 && a.n_actions == 5, "GridWorld shapes");
        ORL_CHECK_ARG(a.env_i32 && a.rewards && a.masks && a.active_masks && a.ep_return && a.ep_length &&
                          a.episode_stats, "GridWorld state buffers");
    } else if (a.env_kind == ORL_ENV_MPE_SPREAD) {
        ORL_CHECK_ARG(a.n_agents == 3 && a.obs_dim == 18 && a.critic_obs_dim == 54 && a.n_actions == 5, "simple_spread shapes");
        ORL_CHECK_ARG(a.env_f64 && a.env_u64 && a.env_i32 && a.rewards && a.masks && a.active_masks && a.ep_return &&
                          a.ep_length && a.episode_stats && a.critic_obs, "simple_spread state buffers");
    } else {
        orl::set_last_error("orl_rollout: unsupported env_kind %d", a.env_kind);
        return ORL_ERR_UNSUPPORTED;
    }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (a.env_kind == ORL_ENV_CARTPOLE || a.env_kind == ORL_ENV_GRIDWORLD) {   // the tensor-core rollouts (orl_fwd_tc.cu)
        // both store each observation as one float4; only rollout_tc_kernel (GridWorld) writes a separate critic_obs
        ORL_CHECK_ARG(a.env_kind == ORL_ENV_CARTPOLE ? (reinterpret_cast<uintptr_t>(a.policy_obs) & 15) == 0 : orl::single_obs_aligned(a),
                      "CartPole / GridWorld: policy_obs (and GridWorld's separate critic_obs) must be 16-byte aligned");
        if (int e = orl::launch_rollout_tc(a, st)) return e;
        return orl::bump_rng_counter(a.rng_counter, a.t_end - a.t_begin, st);
    }
    // rows per CTA: the step chain is latency-bound, so prefer many small CTAs (>= ~4 per SM) and
    // only grow the tile when there are enough rows to keep that many CTAs anyway
    const long long B = (long long)a.n_envs * a.n_agents;
    const long long want = 4LL * orl::sm_count();
    int rm = 32;
    if (B / 32 < want) rm = 16;
    if (B / 16 < want) rm = 8;
    while (rm < a.n_agents) rm *= 2;
    const int envs_per_cta = rm / a.n_agents;
    const int grid = (a.n_envs + envs_per_cta - 1) / envs_per_cta;
    const int ds = std::min(a.obs_dim, orl::OBS_PANEL);   // a panelled fc1 takes the layout of d = 64
    const int ldx = orl::pad4(ds) + 4;
    const bool mpe = a.env_kind == ORL_ENV_MPE_SPREAD, wide = a.n_actions > orl::MAX_OUT, wide_obs = a.obs_dim > orl::OBS_PANEL;
    const size_t smem = sizeof(float) * ((wide ? orl::smem_weights_floats<orl::MAX_OUT_WIDE>(ds, false)
                                               : orl::smem_weights_floats(ds, false)) + rm * ldx + 2 * rm * orl::LDA + rm);
    void (*const kern)(OrlRolloutArgs) =
        wide_obs ? (wide ? (rm == 8 ? rollout_kernel<8, ENV_NONE_WIDE_OBS, orl::MAX_OUT_WIDE>
                            : rm == 16 ? rollout_kernel<16, ENV_NONE_WIDE_OBS, orl::MAX_OUT_WIDE>
                                       : rollout_kernel<32, ENV_NONE_WIDE_OBS, orl::MAX_OUT_WIDE>)
                         : (rm == 8 ? rollout_kernel<8, ENV_NONE_WIDE_OBS>
                            : rm == 16 ? rollout_kernel<16, ENV_NONE_WIDE_OBS> : rollout_kernel<32, ENV_NONE_WIDE_OBS>))
        : wide ? (rm == 8 ? rollout_kernel<8, ORL_ENV_NONE, orl::MAX_OUT_WIDE>
                : rm == 16 ? rollout_kernel<16, ORL_ENV_NONE, orl::MAX_OUT_WIDE> : rollout_kernel<32, ORL_ENV_NONE, orl::MAX_OUT_WIDE>)
        : rm == 8 ? (mpe ? rollout_kernel<8, ORL_ENV_MPE_SPREAD> : rollout_kernel<8, ORL_ENV_NONE>)
        : rm == 16 ? (mpe ? rollout_kernel<16, ORL_ENV_MPE_SPREAD> : rollout_kernel<16, ORL_ENV_NONE>)
                   : (mpe ? rollout_kernel<32, ORL_ENV_MPE_SPREAD> : rollout_kernel<32, ORL_ENV_NONE>);
    if (int e = orl::allow_dynamic_smem(kern, 200 * 1024)) return e;
    kern<<<grid, R_NT, smem, st>>>(a);
    ORL_LAUNCH_CHECK("rollout_kernel");
    return orl::bump_rng_counter(a.rng_counter, a.t_end - a.t_begin, st);
}

extern "C" int orl_critic_values(const float* critic_params, int obs_dim, int activation_id, const float* obs,
                                 float* values, long long rows, void* stream) {
    ORL_CHECK_ARG(critic_params && obs && values, "null buffer");
    ORL_CHECK_ARG(obs_dim > 0 && obs_dim <= orl::MAX_OBS_WIDE, "obs_dim must be in 1..256");
    ORL_CHECK_ARG(rows > 0, "rows");
    ORL_CHECK_ARG(activation_id >= 0 && activation_id <= 3, "activation_id");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (obs_dim <= 8)   // tensor-core forward (orl_fwd_tc.cu)
        return orl::launch_critic_values_tc(critic_params, obs_dim, activation_id, obs, values, rows, st);
    if (obs_dim > orl::OBS_PANEL)
        return launch_rows_forward(critic_values_wide_obs_kernel, "critic_values_wide_obs_kernel", obs_dim, rows, st, critic_params,
                                   obs_dim, activation_id, obs, values, rows);
    return launch_rows_forward(critic_values_kernel, "critic_values_kernel", obs_dim, rows, st, critic_params, obs_dim,
                               activation_id, obs, values, rows);
}

extern "C" int orl_policy_eval(const float* policy_params, int obs_dim, int n_actions, int activation_id, int head_kind,
                               const float* obs, const float* actions, const float* action_masks, float* log_probs,
                               float* entropy, long long rows, void* stream) {
    ORL_CHECK_ARG(policy_params && obs && actions && log_probs && entropy, "null buffer");
    ORL_CHECK_ARG(obs_dim > 0 && obs_dim <= orl::MAX_OBS_WIDE, "obs_dim must be in 1..256");
    ORL_CHECK_ARG(n_actions > 0 && n_actions <= orl::MAX_OUT_WIDE, "n_actions must be in 1..64");
    ORL_CHECK_ARG(rows > 0 && activation_id >= 0 && activation_id <= 3, "rows / activation_id");
    ORL_CHECK_ARG(head_kind == ORL_HEAD_CATEGORICAL || head_kind == ORL_HEAD_GAUSSIAN, "head_kind");
    ORL_CHECK_ARG(n_actions <= orl::MAX_OUT || head_kind == ORL_HEAD_CATEGORICAL,
                  "n_actions must be in 1..8 for Gaussian heads (1..64 for Categorical heads)");
    const bool wide_obs = obs_dim > orl::OBS_PANEL;
    if (n_actions > orl::MAX_OUT && wide_obs)
        return launch_rows_forward<orl::MAX_OUT_WIDE>(policy_eval_wide_wide_obs_kernel, "policy_eval_wide_wide_obs_kernel", obs_dim,
                                                      rows, reinterpret_cast<cudaStream_t>(stream), policy_params, obs_dim, n_actions,
                                                      activation_id, obs, actions, action_masks, log_probs, entropy, rows);
    if (wide_obs)
        return launch_rows_forward(policy_eval_wide_obs_kernel, "policy_eval_wide_obs_kernel", obs_dim, rows,
                                   reinterpret_cast<cudaStream_t>(stream), policy_params, obs_dim, n_actions, activation_id, head_kind,
                                   obs, actions, action_masks, log_probs, entropy, rows);
    if (n_actions > orl::MAX_OUT)
        return launch_rows_forward<orl::MAX_OUT_WIDE>(policy_eval_wide_kernel, "policy_eval_wide_kernel", obs_dim, rows,
                                                      reinterpret_cast<cudaStream_t>(stream), policy_params, obs_dim, n_actions,
                                                      activation_id, obs, actions, action_masks, log_probs, entropy, rows);
    return launch_rows_forward(policy_eval_kernel, "policy_eval_kernel", obs_dim, rows, reinterpret_cast<cudaStream_t>(stream),
                               policy_params, obs_dim, n_actions, activation_id, head_kind, obs, actions, action_masks,
                               log_probs, entropy, rows);
}

// the two feed-forward inserts: critic sections of 1..max_critic features
static int host_insert(const float* staged, int n_envs, int n_agents, int obs_dim, float* policy_obs_next, float* rewards,
                       float* masks_next, float* active_masks_next, float* action_masks_next, int n_actions,
                       float* critic_obs_next, int critic_obs_dim, void* stream, int max_critic) {
    ORL_CHECK_ARG(staged && policy_obs_next && rewards && masks_next && active_masks_next, "null buffer");
    ORL_CHECK_ARG(n_envs > 0 && n_agents > 0 && obs_dim > 0, "shapes");
    ORL_CHECK_ARG(!action_masks_next || (n_actions > 0 && n_actions <= orl::MAX_OUT_WIDE), "n_actions must be in 1..64");
    ORL_CHECK_ARG(!critic_obs_next || (critic_obs_dim > 0 && critic_obs_dim <= max_critic),
                  max_critic == orl::OBS_PANEL ? "critic_obs_dim must be in 1..64 (orl_host_insert_wide_obs: 1..256)"
                                               : "critic_obs_dim must be in 1..256");
    const int B = n_envs * n_agents;
    host_insert_kernel<<<(B + 255) / 256, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(staged, n_envs, n_agents, obs_dim, policy_obs_next,
                                                                                         rewards, masks_next, active_masks_next,
                                                                                         action_masks_next, n_actions,
                                                                                         critic_obs_next, critic_obs_dim);
    ORL_LAUNCH_CHECK("host_insert_kernel");
    return 0;
}

extern "C" int orl_host_insert(const float* staged, int n_envs, int n_agents, int obs_dim, float* policy_obs_next, float* rewards,
                               float* masks_next, float* active_masks_next, float* action_masks_next, int n_actions,
                               float* critic_obs_next, int critic_obs_dim, void* stream) {
    return host_insert(staged, n_envs, n_agents, obs_dim, policy_obs_next, rewards, masks_next, active_masks_next, action_masks_next,
                       n_actions, critic_obs_next, critic_obs_dim, stream, orl::OBS_PANEL);
}

extern "C" int orl_host_insert_wide_obs(const float* staged, int n_envs, int n_agents, int obs_dim, float* policy_obs_next,
                                        float* rewards, float* masks_next, float* active_masks_next, float* action_masks_next,
                                        int n_actions, float* critic_obs_next, int critic_obs_dim, void* stream) {
    return host_insert(staged, n_envs, n_agents, obs_dim, policy_obs_next, rewards, masks_next, active_masks_next, action_masks_next,
                       n_actions, critic_obs_next, critic_obs_dim, stream, orl::MAX_OBS_WIDE);
}

// the three GRU inserts: masks of 1..max_actions actions, critic sections of 1..max_critic features
static int host_insert_rnn(const float* staged, int n_envs, int n_agents, int obs_dim, float* policy_obs_next, float* rewards,
                           float* masks_next, float* active_masks_next, float* rnn_states_next, float* action_masks_next,
                           int n_actions, float* critic_obs_next, int critic_obs_dim, void* stream, int max_actions,
                           int max_critic = orl::OBS_PANEL) {
    ORL_CHECK_ARG(staged && policy_obs_next && rewards && masks_next && active_masks_next && rnn_states_next, "null buffer");
    ORL_CHECK_ARG(n_envs > 0 && n_agents > 0 && obs_dim > 0, "shapes");
    ORL_CHECK_ARG(!action_masks_next || (n_actions > 0 && n_actions <= max_actions),
                  max_actions == orl::MAX_OUT ? "n_actions must be in 1..8 (orl_host_insert_rnn_wide: 1..64)"
                                              : "n_actions must be in 1..64");
    ORL_CHECK_ARG(!critic_obs_next || (critic_obs_dim > 0 && critic_obs_dim <= max_critic),
                  max_critic == orl::OBS_PANEL ? "critic_obs_dim must be in 1..64" : "critic_obs_dim must be in 1..256");
    ORL_CHECK_ARG(reinterpret_cast<uintptr_t>(rnn_states_next) % 16 == 0, "rnn_states_next must be 16-byte aligned");
    const int B = n_envs * n_agents;
    host_insert_rnn_kernel<<<(B + 255) / 256, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        staged, n_envs, n_agents, obs_dim, policy_obs_next, rewards, masks_next, active_masks_next, rnn_states_next,
        action_masks_next, n_actions, critic_obs_next, critic_obs_dim);
    ORL_LAUNCH_CHECK("host_insert_rnn_kernel");
    return 0;
}

extern "C" int orl_host_insert_rnn(const float* staged, int n_envs, int n_agents, int obs_dim, float* policy_obs_next, float* rewards,
                                   float* masks_next, float* active_masks_next, float* rnn_states_next, float* action_masks_next,
                                   int n_actions, float* critic_obs_next, int critic_obs_dim, void* stream) {
    return host_insert_rnn(staged, n_envs, n_agents, obs_dim, policy_obs_next, rewards, masks_next, active_masks_next, rnn_states_next,
                           action_masks_next, n_actions, critic_obs_next, critic_obs_dim, stream, orl::MAX_OUT);
}

extern "C" int orl_host_insert_rnn_wide(const float* staged, int n_envs, int n_agents, int obs_dim, float* policy_obs_next,
                                        float* rewards, float* masks_next, float* active_masks_next, float* rnn_states_next,
                                        float* action_masks_next, int n_actions, float* critic_obs_next, int critic_obs_dim,
                                        void* stream) {
    return host_insert_rnn(staged, n_envs, n_agents, obs_dim, policy_obs_next, rewards, masks_next, active_masks_next, rnn_states_next,
                           action_masks_next, n_actions, critic_obs_next, critic_obs_dim, stream, orl::MAX_OUT_WIDE);
}

extern "C" int orl_host_insert_rnn_wide_obs(const float* staged, int n_envs, int n_agents, int obs_dim, float* policy_obs_next,
                                            float* rewards, float* masks_next, float* active_masks_next, float* rnn_states_next,
                                            float* action_masks_next, int n_actions, float* critic_obs_next, int critic_obs_dim,
                                            void* stream) {
    return host_insert_rnn(staged, n_envs, n_agents, obs_dim, policy_obs_next, rewards, masks_next, active_masks_next, rnn_states_next,
                           action_masks_next, n_actions, critic_obs_next, critic_obs_dim, stream, orl::MAX_OUT_WIDE, orl::MAX_OBS_WIDE);
}
