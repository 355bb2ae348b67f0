// Device-side env.step wrappers (auto-reset + episode statistics), the env step-and-insert of the device rollouts and the
// action sampler (noise, masking, sampling, log-prob) shared by every rollout kernel.
#pragma once
#include "orl_envs.cuh"
#include "orl_loss.cuh"

namespace orl {

struct EnvPtrs {
    double* f64; uint64_t* u64; int32_t* i32; const int32_t* table; int table_len; uint64_t seed;
    float* ep_return; int32_t* ep_length; double* episode_stats;
    int env_offset = 0;   // first GLOBAL env index of this shard: Philox-keyed env randomness is drawn per global env
};

// One env.step of a single-agent, 4-wide-observation env (CartPole-v1 / GridWorldEnv) with the
// reference's auto-reset (sync_venv.py:213-218): on done the returned obs is the reset obs and the
// terminal obs goes to `fin` (info["final_observation"]).
__device__ __forceinline__ void env_step_single(const EnvPtrs& E, int kind, int e, int N, int act, float (&ob)[4],
                                                float& reward, bool& done, float (&fin)[4]) {
    if (kind == ORL_ENV_CARTPOLE) {
        double s[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) s[k] = E.f64[(size_t)k * N + e];
        int elapsed = E.i32[e];
        const bool terminated = cartpole_dynamics(s, act);
        elapsed += 1;
        done = terminated || (elapsed >= 500);
        reward = 1.0f;
        float ret = E.ep_return[e] + 1.0f;
        int len = E.ep_length[e] + 1;
#pragma unroll
        for (int k = 0; k < 4; ++k) fin[k] = (float)s[k];
        if (done) {
            Pcg64 g = pcg_load(E.u64, e, N);
            cartpole_reset(s, g);
            pcg_store(E.u64, e, N, g);
            elapsed = 0;
            atomicAdd(E.episode_stats + 0, (double)ret);
            atomicAdd(E.episode_stats + 1, (double)len);
            atomicAdd(E.episode_stats + 2, 1.0);
            ret = 0.f; len = 0;
        }
        E.ep_return[e] = ret; E.ep_length[e] = len;
        E.i32[e] = elapsed;
#pragma unroll
        for (int k = 0; k < 4; ++k) { E.f64[(size_t)k * N + e] = s[k]; ob[k] = (float)s[k]; }
    } else {  // ORL_ENV_GRIDWORLD
        int x = E.i32[0 * N + e], y = E.i32[1 * N + e], steps = E.i32[2 * N + e];
        int nreset = E.i32[3 * N + e];
        const int nrow = 10, ncol = 10;
        if (act == 1) x -= 1; else if (act == 2) x += 1; else if (act == 3) y -= 1; else if (act == 4) y += 1;
        x = min(max(x, 0), nrow - 1); y = min(max(y, 0), ncol - 1);
        done = false;
        if (x == 1 && y == 1) { reward = 10.f; done = true; } else reward = -1.f;
        if (steps == 100) { done = true; reward -= 10.f; } else steps += 1;  // gridworld_env.py:68-72
        float ret = E.ep_return[e] + reward;
        int len = E.ep_length[e] + 1;
        fin[0] = (float)x; fin[1] = (float)y; fin[2] = 1.f; fin[3] = 1.f;
        if (done) {
            gridworld_reset(x, y, e, nreset, E.seed, E.table, E.table_len, nrow, ncol, e + E.env_offset);
            nreset += 1; steps = 0;
            atomicAdd(E.episode_stats + 0, (double)ret);
            atomicAdd(E.episode_stats + 1, (double)len);
            atomicAdd(E.episode_stats + 2, 1.0);
            ret = 0.f; len = 0;
        }
        E.ep_return[e] = ret; E.ep_length[e] = len;
        E.i32[0 * N + e] = x; E.i32[1 * N + e] = y; E.i32[2 * N + e] = steps; E.i32[3 * N + e] = nreset;
        ob[0] = (float)x; ob[1] = (float)y; ob[2] = 1.f; ob[3] = 1.f;
    }
}

// One simple_spread env.step (3 agents) with auto-reset at world_length = 25.
__device__ __forceinline__ void env_step_mpe(const EnvPtrs& E, int e, int N, const int (&acts)[3], float (&ob)[3][18],
                                             float& reward, bool& done) {
    MpeState s;
    mpe_load(E.f64, e, N, s);
    int step = E.i32[e] + 1;
    mpe_world_step(s, acts);
    const double r = mpe_shared_reward(s);
    reward = (float)r;
    done = step >= 25;
    float ret = E.ep_return[e] + reward;
    int len = E.ep_length[e] + 1;
    if (done) {
        Pcg64 g = pcg_load(E.u64, e, N);
        mpe_reset(s, g);
        pcg_store(E.u64, e, N, g);
        step = 0;
        atomicAdd(E.episode_stats + 0, (double)ret);
        atomicAdd(E.episode_stats + 1, (double)len);
        atomicAdd(E.episode_stats + 2, 1.0);
        ret = 0.f; len = 0;
    }
    E.ep_return[e] = ret; E.ep_length[e] = len;
    E.i32[e] = step;
    mpe_store(E.f64, e, N, s);
#pragma unroll
    for (int ag = 0; ag < 3; ++ag) mpe_obs(s, ag, ob[ag]);
}

// ---- env.step + in-place buffer insert of the device rollouts (onpolicy_driver.py:80-152 for device envs) ---------------
// EnvPtrs of an OrlRolloutArgs or an OrlRnnArgs (the two share the field names)
template <typename Args>
__device__ __forceinline__ EnvPtrs env_ptrs(const Args& a, int env_offset) {
    return EnvPtrs{a.env_f64, a.env_u64, a.env_i32, a.env_table, a.env_table_len, a.rng_seed,
                   a.ep_return, a.ep_length, a.episode_stats, env_offset};
}

// agent ag's observation of a simple_spread env whose agent 0 is buffer row r0: to its policy row and, when critic_obs is
// given, to columns [18 ag, +18) of all three agents' 54-wide critic rows (the concatenated observation)
__device__ __forceinline__ void mpe_insert_obs(const float (&o)[18], int ag, size_t r0, float* policy_obs, float* critic_obs) {
#pragma unroll
    for (int k = 0; k < 18; ++k) {
        policy_obs[(r0 + ag) * 18 + k] = o[k];
        if (critic_obs) {
#pragma unroll
            for (int dst = 0; dst < 3; ++dst) critic_obs[(r0 + dst) * 54 + ag * 18 + k] = o[k];
        }
    }
}

// step_insert_single stores an observation as one float4: policy_obs and a separate critic_obs must be 16-byte aligned
template <typename Args>
inline bool single_obs_aligned(const Args& a) {
    return ((reinterpret_cast<uintptr_t>(a.policy_obs) | reinterpret_cast<uintptr_t>(a.critic_obs)) & 15) == 0;
}

// env.step of single-agent env e (CartPole-v1 / GridWorldEnv) on the action of slot t, then the insert: obs[t+1] (and a
// separate critic_obs[t+1]), rewards[t], masks[t+1] and active_masks[t+1] = 1 (onpolicy_driver.py:118-124 with one
// agent).  Returns obs[t+1]; `done` tells whether the env finished and was reset.
template <typename Args>
__device__ __forceinline__ float4 step_insert_single(const Args& a, const EnvPtrs& E, int kind, int e, int t, int act, bool& done) {
    const int N = a.n_envs;
    float ob[4], fin[4], reward;
    env_step_single(E, kind, e, N, act, ob, reward, done, fin);
    const float4 o = make_float4(ob[0], ob[1], ob[2], ob[3]);
    const size_t o1 = (size_t)(t + 1) * N + e;
    reinterpret_cast<float4*>(a.policy_obs)[o1] = o;
    if (a.critic_obs && a.critic_obs != a.policy_obs) reinterpret_cast<float4*>(a.critic_obs)[o1] = o;
    a.rewards[(size_t)t * N + e] = reward;
    a.masks[o1] = done ? 0.f : 1.f;
    a.active_masks[o1] = 1.f;
    return o;
}

// no copy of the observations besides the buffers (the default `keep` of step_insert_mpe)
struct NoKeep {
    __device__ __forceinline__ void operator()(int, int, float) const {}
};

// the same for a simple_spread env: its three agent rows, which finish together.  keep(ag, k, v) receives obs[t+1] for a
// kernel's own shared-memory copy, ahead of every buffer store: so the compiler can merge those shared stores into
// vector stores (it cannot move them across the global ones), and the FFMA rollout stays within its registers without
// spilling.  Returns done.
template <typename Args, typename Keep = NoKeep>
__device__ __forceinline__ bool step_insert_mpe(const Args& a, const EnvPtrs& E, int e, int t, const int (&acts)[3],
                                                Keep keep = {}) {
    const int N = a.n_envs, B = N * a.n_agents;   // n_agents == 3
    float ob[3][18], reward; bool done;
    env_step_mpe(E, e, N, acts, ob, reward, done);
#pragma unroll
    for (int ag = 0; ag < 3; ++ag)
#pragma unroll
        for (int k = 0; k < 18; ++k) keep(ag, k, ob[ag][k]);
    const size_t r1 = (size_t)(t + 1) * B + (size_t)e * 3;
#pragma unroll
    for (int ag = 0; ag < 3; ++ag) {
        mpe_insert_obs(ob[ag], ag, r1, a.policy_obs, a.critic_obs);
        a.rewards[(size_t)t * B + (size_t)e * 3 + ag] = reward;
        a.masks[r1 + ag] = done ? 0.f : 1.f;
        a.active_masks[r1 + ag] = 1.f;
    }
    return done;
}

// ---- the action sampler of every rollout kernel ------------------------------------------------------------------------
// Philox4x32-10 block `lane` of the action randomness of (step, row): key = seed, counter = (step lo, step hi, row, lane).
// The row is the GLOBAL row (local row + rng_row_offset) wherever the kernel knows it, so an env-sharded run draws the
// same noise as the unsharded one.
__device__ __forceinline__ uint4 action_philox(uint64_t seed, uint64_t step, uint32_t row, uint32_t lane) {
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    return philox4x32_10(make_uint4((uint32_t)step, (uint32_t)(step >> 32), row, lane), key);
}

// Exp(1) noise q[0..n) of (step, row): the reference-order table exp_noise[grow * n + j] when one is given (parity mode),
// else -log U of the 8 draws of Philox lanes `lane`, `lane + 1`.
// Lanes of one (step, row): 0, 1 the noise of actions 0..7 (wide_action_noise4 keeps them for those actions); 2..33 the
// DiagGaussian normals, dimensions [4k, 4k + 4) by Box-Muller of u1 from lane 2 + 2k and u2 from lane 3 + 2k (k = 0, 1:
// gaussian_act's lanes 2..5; k = 0..15: gaussian_noise4 of a wide head), and in the self-play rollout 2, 3 the opponent's
// noise and 4 its pick; 8..21 the noise of actions 8..63 of a wide Categorical head, action j from draw (j - 8) % 4 of
// lane 8 + (j - 8) / 4.  A row has one head, so no two uses of one draw meet within a row.
__device__ __forceinline__ void action_noise(const float* exp_noise, size_t grow, int n, uint64_t seed, uint64_t step,
                                             uint32_t row, float (&q)[MAX_OUT], uint32_t lane = 0u) {
    if (exp_noise) {
#pragma unroll
        for (int j = 0; j < MAX_OUT; ++j) q[j] = (j < n) ? exp_noise[grow * n + j] : 1.f;
    } else {
        const uint4 r0 = action_philox(seed, step, row, lane), r1 = action_philox(seed, step, row, lane + 1u);
        const uint32_t rr[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
        for (int j = 0; j < MAX_OUT; ++j) q[j] = -logf(u32_to_unit_open(rr[j]));
    }
}

// Categorical action of one row and its log-prob: the first-max mode when deterministic, else torch.multinomial(probs, 1)
// == argmax(probs / q) (first index wins ties) over the Exp(1) noise q that `noise(q)` writes.  The noise is asked for
// only on the stochastic branch, after the log-softmax, so a kernel that draws it there keeps q short-lived.
template <typename Noise>
__device__ __forceinline__ int sample_action(float (&logit)[MAX_OUT], int n, const float* mask_row, bool deterministic,
                                             Noise&& noise, float& lp) {
    float nl[MAX_OUT], pr[MAX_OUT];
    masked_log_softmax(logit, n, mask_row, nl, pr);
    int act;
    if (deterministic) {
        act = 0;
#pragma unroll
        for (int j = 1; j < MAX_OUT; ++j) if (j < n && pr[j] > pr[act]) act = j;
    } else {
        float q[MAX_OUT];
        noise(q);
        int best = 0;
        float bv = pr[0] / q[0];
#pragma unroll
        for (int j = 1; j < MAX_OUT; ++j)
            if (j < n) { const float v = pr[j] / q[j]; if (v > bv) { bv = v; best = j; } }
        act = best;
    }
    lp = log_prob_of(nl, n, act);
    return act;
}

// Exp(1) noise q[0..4) of actions j0..j0+3 (j0 % 4 == 0) of a wide head's row: the table entries j < n in parity mode,
// else -log U of Philox lane j0 / 4 (actions 0..7, the draws action_noise gives them) or 8 + (j0 - 8) / 4.
__device__ __forceinline__ void wide_action_noise4(const float* exp_noise, size_t grow, int n, uint64_t seed, uint64_t step,
                                                   uint32_t row, int j0, float (&q)[4]) {
    if (exp_noise) {
#pragma unroll
        for (int c = 0; c < 4; ++c) q[c] = (j0 + c < n) ? exp_noise[grow * n + j0 + c] : 1.f;
    } else {
        const uint4 r = action_philox(seed, step, row, j0 < 8 ? (uint32_t)(j0 / 4) : 8u + (uint32_t)((j0 - 8) / 4));
        q[0] = -logf(u32_to_unit_open(r.x)); q[1] = -logf(u32_to_unit_open(r.y));
        q[2] = -logf(u32_to_unit_open(r.z)); q[3] = -logf(u32_to_unit_open(r.w));
    }
}

// sample_action of a wide head's row x[0..n) in shared memory (masked in place): the first-max mode when deterministic,
// else argmax(probs / q) with the first index winning ties, q from noise4(j0, q[4]) four actions at a time.
template <typename Noise4>
__device__ __forceinline__ int wide_sample_action(float* x, int n, const float* mask_row, bool deterministic, Noise4&& noise4,
                                                  float& lp) {
    const WideSoftmax sm = wide_log_softmax(x, n, mask_row);
    int act = 0;
    float bv = sm.pr(x, 0);
    if (deterministic) {
        for (int j = 1; j < n; ++j) { const float v = sm.pr(x, j); if (v > bv) { bv = v; act = j; } }
    } else {
        for (int j0 = 0; j0 < n; j0 += 4) {
            float q[4];
            noise4(j0, q);
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const int j = j0 + c;
                if (j < n) {
                    const float v = sm.pr(x, j) / q[c];
                    if (j == 0 || v > bv) { bv = v; act = j; }
                }
            }
        }
    }
    lp = wide_log_prob_of(sm, x, n, act);
    return act;
}

// DiagGaussian act of one row (distributions.py:75-98): action = noise * std + mean (the mean when deterministic) and
// the per-dimension log-probs, written to actions / log_probs [grow * n + j].  The N(0, 1) noise is the reference-order
// table noise_table[grow * n + j] when one is given (parity mode), else Box-Muller over Philox lanes 2..5 of
// (step, row): 8 normals from the 16 uniforms of the lane pairs (2, 3) and (4, 5).
__device__ __forceinline__ void gaussian_act(const float (&mean)[MAX_OUT], int n, const float* logstd, bool deterministic,
                                             const float* noise_table, uint64_t seed, uint64_t step, uint32_t row, size_t grow,
                                             float* actions, float* log_probs) {
    uint32_t rr[8];
    if (!noise_table && !deterministic) {
        const uint4 r0 = action_philox(seed, step, row, 2u), r1 = action_philox(seed, step, row, 3u);
        const uint4 r2 = action_philox(seed, step, row, 4u), r3 = action_philox(seed, step, row, 5u);
        const uint32_t u1[8] = {r0.x, r0.y, r0.z, r0.w, r2.x, r2.y, r2.z, r2.w};
        const uint32_t u2[8] = {r1.x, r1.y, r1.z, r1.w, r3.x, r3.y, r3.z, r3.w};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float rad = sqrtf(-2.0f * logf(u32_to_unit_open(u1[j])));
            rr[j] = __float_as_uint(rad * cospif(2.0f * u32_to_unit_open(u2[j])));
        }
    }
#pragma unroll
    for (int j = 0; j < MAX_OUT; ++j) {
        if (j < n) {
            const float ls = logstd[j], std = expf(ls);
            float act = mean[j];
            if (!deterministic) {
                const float eps = noise_table ? noise_table[grow * n + j] : __uint_as_float(rr[j]);
                act = __fadd_rn(__fmul_rn(eps, std), mean[j]);
            }
            actions[grow * n + j] = act;
            log_probs[grow * n + j] = gaussian_log_prob(act - mean[j], std, ls);
        }
    }
}

// N(0, 1) noise eps[0..4) of dimensions j0..j0+3 (j0 % 4 == 0) of a wide DiagGaussian head's row: Box-Muller of u1 from
// Philox lane 2 + j0 / 2 and u2 from lane 3 + j0 / 2, gaussian_act's expression, so dimensions 0..7 draw what
// gaussian_act draws for them, bit for bit
__device__ __forceinline__ void gaussian_noise4(uint64_t seed, uint64_t step, uint32_t row, int j0, float (&eps)[4]) {
    const uint32_t lane = 2u + (uint32_t)(j0 / 2);
    const uint4 r1 = action_philox(seed, step, row, lane), r2 = action_philox(seed, step, row, lane + 1u);
    const uint32_t u1[4] = {r1.x, r1.y, r1.z, r1.w}, u2[4] = {r2.x, r2.y, r2.z, r2.w};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const float rad = sqrtf(-2.0f * logf(u32_to_unit_open(u1[c])));
        eps[c] = rad * cospif(2.0f * u32_to_unit_open(u2[c]));
    }
}

// DiagGaussian act of dimensions j0..j0+3 (those < n) of one row of a wide head (1..64 dimensions): gaussian_act's
// arithmetic on the means mean[0..n) of the row, in shared memory.  The noise is the table entries in parity mode, else
// gaussian_noise4; deterministic calls return the mean.
__device__ __forceinline__ void gaussian_act4(const float* mean, int n, int j0, const float* logstd, bool deterministic,
                                              const float* noise_table, uint64_t seed, uint64_t step, uint32_t row, size_t grow,
                                              float* actions, float* log_probs) {
    float eps[4] = {0.f, 0.f, 0.f, 0.f};
    if (!noise_table && !deterministic) gaussian_noise4(seed, step, row, j0, eps);
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const int j = j0 + c;
        if (j < n) {
            const float ls = logstd[j], std = expf(ls);
            float act = mean[j];
            if (!deterministic) {
                const float e = noise_table ? noise_table[grow * n + j] : eps[c];
                act = __fadd_rn(__fmul_rn(e, std), mean[j]);
            }
            actions[grow * n + j] = act;
            log_probs[grow * n + j] = gaussian_log_prob(act - mean[j], std, ls);
        }
    }
}

}  // namespace orl
