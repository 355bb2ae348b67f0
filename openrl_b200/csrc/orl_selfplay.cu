// Self-play on the device (BASELINE configs[3]: "GridWorld self-play PPO, 2 players, opponent-pool sampling"): a
// two-player GridWorld whose second player is driven by a policy snapshot drawn from an OPPONENT POOL that lives in HBM.
// Replaces, for this env, the reference's self-play control flow (SURVEY.md §3.5):
//   OpponentPoolWrapper.reset / get_opponent_action / on_episode_end   openrl/selfplay/wrappers/opponent_pool_wrapper.py:30-120
//   RandomOpponent / LastOpponent sampling                             openrl/selfplay/sample_strategy/{random,last}_opponent.py:24-28
//   SelfplayCallback snapshot cadence                                  openrl/selfplay/callbacks/selfplay_callback.py:124-144
// (the pool server, TrueSkill rating and opponent files of the reference's Ray/HTTP control plane are out of scope; the
// pool here is a ring of parameter snapshots written by the host every `save_freq` iterations).
//
// The game (new env: the reference ships no 2-player GridWorld, SURVEY.md §8f-2 — no reference parity possible; the rules
// are restated in oracle/selfplay.py and the device step is checked bit-exactly against it):
//   10 x 10 grid, goal cell (1, 1) (GridWorldEnv's, gridworld_env.py:21-36).  Both players start on distinct non-goal cells
//   (Philox keyed by (seed, GLOBAL env, #reset), or a host table in tests).  Each step both pick an action of
//   GridWorldEnv's set {0 stay, 1 x-1, 2 x+1, 3 y-1, 4 y+1}, move simultaneously, positions clipped to the grid (cells may be
//   shared).  Exactly one player on the goal: it wins — learner reward +10 / -10, episode ends.  Both on the goal: draw,
//   reward 0, ends.  Otherwise reward -1; after 100 steps the episode ends as a draw with reward -11 (GridWorldEnv's
//   time-out penalty).  The learner observes (x0, y0, x1, y1); the opponent observes (x1, y1, x0, y0).
//
// One thread per env for all T steps (envs are independent): learner forward + sample, opponent forward with ITS
// snapshot's weights (read through L1/L2; snapshots are 20 KB) + sample, env step, in-place buffer insert.  At every
// episode start the env draws its opponent: uniform over the pool (RandomOpponent) or the newest snapshot (LastOpponent);
// with an empty pool the opponent acts uniformly at random (opponent_pool_wrapper.py:70-81).
#include "orl_envstep.cuh"
#include "orl_rnn_core.h"

namespace {
using namespace orl;

constexpr int SP_NT = 128, SP_ROWS = 10, SP_COLS = 10, SP_MAX_STEPS = 100;

// policy forward of one row (net_offsets layout): logits[n].  A real call: the kernel keeps one call frame instead of
// inlining both forwards.
__device__ __noinline__ void sp_forward(const float* __restrict__ P, int n, int activation_id, const float (&x)[4], float* logits) {
    const NetOffsets o = net_offsets(4, n);
    float y[H];
    orl_rnn::trunk_forward(P, o, activation_id, x, y);
    for (int j = 0; j < n; ++j) {
        float s = P[o.bh + j];
        for (int k = 0; k < H; ++k) s = fmaf(P[o.wh + j * H + k], y[k], s);
        logits[j] = s;
    }
}

__device__ __forceinline__ void sp_move(int& x, int& y, int act) {
    if (act == 1) x -= 1; else if (act == 2) x += 1; else if (act == 3) y -= 1; else if (act == 4) y += 1;
    x = min(max(x, 0), SP_ROWS - 1); y = min(max(y, 0), SP_COLS - 1);
}

// start cells of both players: distinct, non-goal; Philox keyed by (seed, global env, #reset) or a host table
// table[(env * table_len + k) * 4 + {0..3}] = x0, y0, x1, y1 of reset k
__device__ __forceinline__ void sp_reset_cells(int& x0, int& y0, int& x1, int& y1, int env, int env_key, int nreset, uint64_t seed,
                                               const int* __restrict__ table, int table_len) {
    if (table) {
        const int k = min(nreset, table_len - 1);
        const int* t = table + ((size_t)env * table_len + k) * 4;
        x0 = t[0]; y0 = t[1]; x1 = t[2]; y1 = t[3];
        return;
    }
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    uint4 c = make_uint4((uint32_t)env_key, (uint32_t)nreset, 0x53706c79u, 0u);
    x0 = 0; y0 = 0; x1 = 0; y1 = 2;
    for (int it = 0; it < 16; ++it) {
        c.w = it;
        const uint4 r = philox4x32_10(c, key);
        const int a0 = (int)(((uint64_t)r.x * SP_ROWS) >> 32), b0 = (int)(((uint64_t)r.y * SP_COLS) >> 32);
        const int a1 = (int)(((uint64_t)r.z * SP_ROWS) >> 32), b1 = (int)(((uint64_t)r.w * SP_COLS) >> 32);
        if (!(a0 == 1 && b0 == 1) && !(a1 == 1 && b1 == 1) && !(a0 == a1 && b0 == b1)) { x0 = a0; y0 = b0; x1 = a1; y1 = b1; return; }
    }
}

// opponent of a new episode: index into the pool ring, or -1 (random-action opponent) while the pool is empty
__device__ __forceinline__ int sp_pick_opponent(int strategy, int pool_count, int pool_cap, int env_key, int nreset, uint64_t seed) {
    const int avail = min(pool_count, pool_cap);
    if (avail <= 0) return -1;
    if (strategy == ORL_SP_LAST) return (pool_count - 1) % pool_cap;                       // last_opponent.py:24-27
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    const uint4 r = philox4x32_10(make_uint4((uint32_t)env_key, (uint32_t)nreset, 0x4f70706fu, 0u), key);
    return (int)(((uint64_t)r.x * (uint64_t)avail) >> 32);                                // random.randint(0, len - 1), random_opponent.py:25-28
}

// env_i32 layout [8][N]: x0, y0, x1, y1, steps, nreset, opponent index, (unused)
__global__ void __launch_bounds__(SP_NT) selfplay_reset_kernel(const OrlSelfPlayArgs s, float* __restrict__ obs_out) {
    const OrlRolloutArgs& a = s.rollout;
    const int N = a.n_envs, e = blockIdx.x * SP_NT + threadIdx.x;
    if (e >= N) return;
    const int env_key = e + a.rng_row_offset;
    int x0, y0, x1, y1, nreset = a.env_i32[5 * N + e];
    sp_reset_cells(x0, y0, x1, y1, e, env_key, nreset, a.rng_seed, a.env_table, a.env_table_len);
    a.env_i32[0 * N + e] = x0; a.env_i32[1 * N + e] = y0; a.env_i32[2 * N + e] = x1; a.env_i32[3 * N + e] = y1;
    a.env_i32[4 * N + e] = 0;
    a.env_i32[6 * N + e] = sp_pick_opponent(s.strategy, *s.pool_count, s.pool_capacity, env_key, nreset, a.rng_seed);
    a.env_i32[5 * N + e] = nreset + 1;
    obs_out[(size_t)e * 4 + 0] = (float)x0; obs_out[(size_t)e * 4 + 1] = (float)y0;
    obs_out[(size_t)e * 4 + 2] = (float)x1; obs_out[(size_t)e * 4 + 3] = (float)y1;
}

__global__ void __launch_bounds__(SP_NT) selfplay_rollout_kernel(const OrlSelfPlayArgs s) {
    const OrlRolloutArgs& a = s.rollout;
    const int N = a.n_envs, n = a.n_actions, e = blockIdx.x * SP_NT + threadIdx.x;
    if (e >= N) return;
    const int env_key = e + a.rng_row_offset;
    const uint64_t rng_base = a.rng_step_base + (a.rng_counter ? *a.rng_counter : 0ull);
    const int pool_count = *s.pool_count;
    int x0 = a.env_i32[0 * N + e], y0 = a.env_i32[1 * N + e], x1 = a.env_i32[2 * N + e], y1 = a.env_i32[3 * N + e];
    int steps = a.env_i32[4 * N + e], nreset = a.env_i32[5 * N + e], opp = a.env_i32[6 * N + e];
    float ep_ret = a.ep_return[e];
    int ep_len = a.ep_length[e];
    for (int t = a.t_begin; t < a.t_end; ++t) {
        const uint64_t step = rng_base + (uint64_t)t;
        const size_t grow = (size_t)t * N + e;
        // ---- learner: forward + sample (deterministic bit 1: greedy, bit 2: scripted from exp_noise) ----
        // Philox lanes of (step, env_key): 0/1 learner, 2/3 opponent policy, 4 random opponent
        const float xl[4] = {(float)x0, (float)y0, (float)x1, (float)y1};
        float logits[MAX_OUT], lp;
        sp_forward(a.policy_params, n, a.activation_id, xl, logits);
        int act0 = sample_action(logits, n, nullptr, a.deterministic & 1, [&](float (&q)[MAX_OUT]) {
            action_noise(nullptr, 0, n, a.rng_seed, step, (uint32_t)env_key, q);
        }, lp);
        if ((a.deterministic & 2) && a.exp_noise) {   // scripted learner action (vec-env step API, tests): log-prob of THAT action
            act0 = (int)a.exp_noise[grow * 2 + 0];
            float nl[MAX_OUT], pr[MAX_OUT];
            masked_log_softmax(logits, n, nullptr, nl, pr);
            lp = log_prob_of(nl, n, act0);
        }
        // ---- opponent: its snapshot's policy on the mirrored observation, or a uniformly random action ----
        int act1;
        if ((a.deterministic & 4) && a.exp_noise) {
            act1 = (int)a.exp_noise[grow * 2 + 1];
        } else if (opp >= 0) {
            const float xo[4] = {(float)x1, (float)y1, (float)x0, (float)y0};
            float lo[MAX_OUT], lpo;
            sp_forward(s.pool_params + (size_t)opp * s.pool_stride, n, a.activation_id, xo, lo);
            act1 = sample_action(lo, n, nullptr, false, [&](float (&q)[MAX_OUT]) {
                action_noise(nullptr, 0, n, a.rng_seed, step, (uint32_t)env_key, q, 2u);
            }, lpo);
        } else {
            act1 = (int)(((uint64_t)action_philox(a.rng_seed, step, (uint32_t)env_key, 4u).x * (uint64_t)n) >> 32);
        }
        a.actions[grow] = (float)act0;
        a.action_log_probs[grow] = lp;
        // ---- env step ----
        sp_move(x0, y0, act0);
        sp_move(x1, y1, act1);
        const bool g0 = (x0 == 1 && y0 == 1), g1 = (x1 == 1 && y1 == 1);
        float reward; bool done = false; int outcome = -1;   // 0 win, 1 loss, 2 draw (from the learner's side)
        if (g0 && !g1) { reward = 10.f; done = true; outcome = 0; }
        else if (g1 && !g0) { reward = -10.f; done = true; outcome = 1; }
        else if (g0 && g1) { reward = 0.f; done = true; outcome = 2; }
        else reward = -1.f;
        if (!done) {
            if (steps == SP_MAX_STEPS) { done = true; reward -= 10.f; outcome = 2; } else steps += 1;
        }
        ep_ret += reward; ep_len += 1;
        if (done) {
            // bookkeeping of the finished episode against this opponent (opponent_pool_wrapper.py:91-120): slot = pool index, last slot = random opponent
            const int slot = opp >= 0 ? opp : s.pool_capacity;
            atomicAdd(s.pool_stats + (size_t)slot * 3 + outcome, 1);
            atomicAdd(a.episode_stats + 0, (double)ep_ret);
            atomicAdd(a.episode_stats + 1, (double)ep_len);
            atomicAdd(a.episode_stats + 2, 1.0);
            ep_ret = 0.f; ep_len = 0;
            sp_reset_cells(x0, y0, x1, y1, e, env_key, nreset, a.rng_seed, a.env_table, a.env_table_len);
            opp = sp_pick_opponent(s.strategy, pool_count, s.pool_capacity, env_key, nreset, a.rng_seed);
            nreset += 1; steps = 0;
        }
        const size_t o1 = (size_t)(t + 1) * N + e;
        *reinterpret_cast<float4*>(a.policy_obs + o1 * 4) = make_float4((float)x0, (float)y0, (float)x1, (float)y1);
        a.rewards[grow] = reward;
        a.masks[o1] = done ? 0.f : 1.f;
        a.active_masks[o1] = 1.f;
    }
    a.env_i32[0 * N + e] = x0; a.env_i32[1 * N + e] = y0; a.env_i32[2 * N + e] = x1; a.env_i32[3 * N + e] = y1;
    a.env_i32[4 * N + e] = steps; a.env_i32[5 * N + e] = nreset; a.env_i32[6 * N + e] = opp;
    a.ep_return[e] = ep_ret; a.ep_length[e] = ep_len;
}

int check_selfplay(const OrlSelfPlayArgs& s) {
    const OrlRolloutArgs& a = s.rollout;
    ORL_CHECK_ARG(a.n_envs > 0 && a.n_agents == 1 && a.obs_dim == 4 && a.n_actions == 5, "the 2-player GridWorld has obs (x0,y0,x1,y1) and 5 actions");
    ORL_CHECK_ARG(a.env_i32 && s.pool_count && s.pool_stats, "env state / pool buffers");
    ORL_CHECK_ARG(s.pool_capacity >= 0 && (s.pool_capacity == 0 || (s.pool_params && s.pool_stride > 0)), "pool");
    ORL_CHECK_ARG(s.strategy == ORL_SP_RANDOM || s.strategy == ORL_SP_LAST, "strategy");
    ORL_CHECK_ARG(a.head_kind != ORL_HEAD_GAUSSIAN_WIDE, "the self-play rollout acts with Categorical heads");
    return 0;
}

}  // namespace

extern "C" int orl_selfplay_reset(const OrlSelfPlayArgs* sp, float* policy_obs_out, void* stream) {
    ORL_CHECK_ARG(sp && policy_obs_out, "args");
    if (int e = check_selfplay(*sp)) return e;
    const int N = sp->rollout.n_envs;
    selfplay_reset_kernel<<<(N + SP_NT - 1) / SP_NT, SP_NT, 0, reinterpret_cast<cudaStream_t>(stream)>>>(*sp, policy_obs_out);
    ORL_LAUNCH_CHECK("selfplay_reset_kernel");
    return 0;
}

extern "C" int orl_selfplay_rollout(const OrlSelfPlayArgs* sp, void* stream) {
    ORL_CHECK_ARG(sp, "args");
    if (int e = check_selfplay(*sp)) return e;
    const OrlRolloutArgs& a = sp->rollout;
    ORL_CHECK_ARG(a.t_begin >= 0 && a.t_begin < a.t_end, "step range");
    ORL_CHECK_ARG(a.policy_params && a.policy_obs && a.actions && a.action_log_probs && a.rewards && a.masks && a.active_masks &&
                      a.ep_return && a.ep_length && a.episode_stats, "null buffer");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    selfplay_rollout_kernel<<<(a.n_envs + SP_NT - 1) / SP_NT, SP_NT, 0, st>>>(*sp);
    ORL_LAUNCH_CHECK("selfplay_rollout_kernel");
    return orl::bump_rng_counter(a.rng_counter, a.t_end - a.t_begin, st);
}
