/*
 * openrl_b200.h — C-ABI of libopenrl_b200.so (hand-written sm_90a CUDA).
 *
 * Drop-in boundary for OpenRL's rollout-collection + PPO/MAPPO-update hot path.
 * The reference has no FFI: its seams are Python constructor-injection points
 * (SURVEY.md §8b).  Every entry point below replaces the inner loop of one
 * reference function; the Python host package `openrl_b200` binds them with ctypes
 * (openrl_b200/lib.py) and INTEGRATION.md shows the stub a reference maintainer
 * would add.
 *
 * Conventions
 *   - plain pointers and sizes only; all pointers are DEVICE pointers unless the
 *     name ends in _host; the caller owns all memory (torch tensors in practice);
 *   - every call is asynchronous on `stream` (a cudaStream_t passed as void*);
 *   - return value: 0 = ok, otherwise a cudaError_t or ORL_ERR_*; the message is
 *     available from orl_last_error();
 *   - all floating-point buffers are float32, row-major, laid out like the
 *     reference's ReplayData arrays with the (env, agent) axes flattened:
 *     element (t, n, a, k) of a (T[+1], N, A, K) array is at ((t*N + n)*A + a)*K + k;
 *     B = N*A is the number of "rows" (columns of the time scan).
 */
#ifndef OPENRL_B200_H
#define OPENRL_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ORL_ABI_VERSION 1

#define ORL_ERR_BAD_ARG 10001
#define ORL_ERR_UNSUPPORTED 10002

/* library / device --------------------------------------------------------------- */
int orl_abi_version(void);
const char* orl_last_error(void);
/* number of SMs of the current device (grids are sized from it) */
int orl_device_sm_count(int* sm_count_out);

/* ---- GAE / returns ---------------------------------------------------------------
 * Replaces ReplayData.compute_returns (openrl/buffers/replay_data.py:320-423, all 8
 * branches) and, fused behind it, the advantage construction of
 * PPOAlgorithm.train_ppo (openrl/algorithms/ppo.py:384-399) plus the moments needed
 * by its normalisation (ppo.py:402-409) and by ValueNorm.update on a full-buffer
 * minibatch (openrl/modules/utils/valuenorm.py:59-76).
 *
 * flags: */
#define ORL_GAE_USE_GAE 1            /* cfg.use_gae */
#define ORL_GAE_PROPER_TIME_LIMITS 2 /* cfg.use_proper_time_limits (reads bad_masks) */
#define ORL_GAE_DENORM 4             /* (use_popart|use_valuenorm) and normalizer given */
/*
 * rewards      (T,   B)   in
 * value_preds  (T+1, B)   in/out: row T is overwritten with next_value when USE_GAE
 * masks        (T+1, B)   in
 * bad_masks    (T+1, B)   in   (may be NULL unless PROPER_TIME_LIMITS)
 * active_masks (T+1, B)   in   (may be NULL: treated as all ones; only used for stats)
 * next_value   (B)        in   bootstrap value of slot T
 * vn_state     (3)        in   ValueNorm {running_mean, running_mean_sq, debiasing_term}
 *                              (valuenorm.py:27-35); required iff ORL_GAE_DENORM
 * returns      (T+1, B)   out  (row T = next_value when !USE_GAE, untouched otherwise)
 * advantages   (T,   B)   out  returns[:-1] - denorm(value_preds[:-1]); may be NULL
 * stats        (ORL_GAE_NSTATS doubles) out, may be NULL; ZEROED by the call, then
 *              accumulated: see ORL_GS_* indices.
 * gamma, gae_lambda are passed as double because the reference multiplies the two
 * Python floats in double before the product meets the float32 arrays.
 * Bit-exact with the reference's numpy float32 evaluation order (no FMA contraction).
 */
#define ORL_GAE_NSTATS 8
#define ORL_GS_ADV_SUM 0      /* sum adv            over all (t<T, b)            */
#define ORL_GS_ADV_SQSUM 1    /* sum adv^2                                        */
#define ORL_GS_COUNT 2        /* T*B                                              */
#define ORL_GS_ADV_ACT_SUM 3  /* sum adv   where active_masks[t] != 0             */
#define ORL_GS_ADV_ACT_SQSUM 4
#define ORL_GS_RET_SUM 5      /* sum returns[t<T]       } {5,6,7} is the mb_stats triple  */
#define ORL_GS_RET_SQSUM 6    /* sum returns[t<T]^2     } of orl_ppo_* for a minibatch    */
#define ORL_GS_ACT_COUNT 7    /* number of active elements } covering the whole buffer    */
int orl_gae(const float* rewards, float* value_preds, const float* masks,
            const float* bad_masks, const float* active_masks, const float* next_value,
            const float* vn_state, float* returns, float* advantages, double* stats,
            int T, int B, double gamma, double gae_lambda, int flags, void* stream);


/* ---- device-resident vectorised envs -------------------------------------------------
 * Replace SyncVectorEnv/AsyncVectorEnv stepping (openrl/envs/vec_env/sync_venv.py:129-247,
 * async_venv.py:316-430,731-875) + the per-env wrappers Single2MultiAgentWrapper /
 * RemoveTruncated (openrl/envs/wrappers/multiagent_wrapper.py:33-79,
 * extra_wrappers.py:122-134) for the simple gym-class envs.  State lives in caller-owned
 * device arrays (SoA over envs):
 *   CARTPOLE : env_f64 [4][N] (x, x_dot, theta, theta_dot) float64 like gymnasium;
 *              env_i32 [1][N] elapsed steps (TimeLimit 500);
 *              env_u64 [4][N] numpy-PCG64 {state_hi, state_lo, inc_hi, inc_lo} of the env's
 *              np_random (seeded seed + i*10086 by the host, sync_venv.py:137).
 *   GRIDWORLD: env_i32 [4][N] (x, y, steps, resets); env_table optional int32
 *              [N][env_table_len][2] start cells for parity runs; else Philox(rng_seed).
 *   NONE     : no device env (host env.step, e.g. MuJoCo): orl_rollout only acts.
 */
#define ORL_HEAD_CATEGORICAL 0
#define ORL_HEAD_GAUSSIAN 1
/* DiagGaussian head of 1..64 dimensions (Box(n) with n up to 64): the parameter layout, actions and log-probs of
 * ORL_HEAD_GAUSSIAN, run on the 64-wide head tile.  Taken by orl_rollout (ORL_ENV_NONE only), orl_policy_eval,
 * orl_ppo_fwdbwd, orl_ppo_reduce, orl_ppo_apply and their peer variants; ORL_ERR_BAD_ARG on the tensor-core update,
 * the orl_share_* entries, the self-play rollout and every device env.  ORL_HEAD_GAUSSIAN keeps 1..8.  The GRU entries
 * (OrlRnnArgs.head_kind) take it for 9..64 dimensions only. */
#define ORL_HEAD_GAUSSIAN_WIDE 2
#define ORL_ENV_NONE 0
#define ORL_ENV_CARTPOLE 1
#define ORL_ENV_GRIDWORLD 2
#define ORL_ENV_MPE_SPREAD 3

/* Draw initial states (env.reset()) and write the observations of slot `obs_out` (B, d).
 * Mirrors SyncVectorEnv._reset (sync_venv.py:129-169).  RNG streams must already be seeded. */
int orl_env_reset(int env_kind, int n_envs, int n_agents, double* env_f64, uint64_t* env_u64,
                  int32_t* env_i32, const int32_t* env_table, int env_table_len,
                  uint64_t rng_seed, float* policy_obs_out, float* critic_obs_out, void* stream);

/* One vectorised env.step outside the fused rollout (the BaseVecEnv.step duck type used by
 * evaluation loops): actions (B) float -> obs (B,d), rewards (B), dones (B) as 0/1 floats and,
 * optionally, the pre-reset terminal observation (info["final_observation"], sync_venv.py:213-218). */
int orl_env_step(int env_kind, int n_envs, int n_agents, double* env_f64, uint64_t* env_u64,
                 int32_t* env_i32, const int32_t* env_table, int env_table_len, uint64_t rng_seed,
                 float* ep_return, int32_t* ep_length, double* episode_stats, const float* actions,
                 float* obs_out, float* rewards_out, float* dones_out, float* final_obs_out,
                 void* stream);

/* ---- fused rollout: policy forward + sampling + env.step + buffer insert -----------------
 * Replaces the body of OnPolicyDriver.actor_rollout for steps [t_begin, t_end)
 * (openrl/drivers/onpolicy_driver.py:154-203): act() :236-279 (policy half:
 * PolicyNetwork.forward_original policy_network.py:130-162, MLPBase mlp.py:160-176,
 * Categorical distributions.py:58-72, sampling = torch.multinomial == argmax(probs/q)),
 * envs.step() (see above), add2buffer() :80-152 and ReplayData.insert
 * (openrl/buffers/replay_data.py:245-284).  Envs are independent, so one launch can cover all
 * T steps (t_begin = 0, t_end = T); per-step launches (t_end = t_begin + 1) serve callbacks.
 * Critic values are produced separately by orl_critic_values (they do not influence the
 * trajectory).
 *
 * Sampling: exp_noise != NULL ("parity mode") supplies q ~ Exp(1) of shape (T, B, n) drawn by
 * the host with torch's CPU generator in the reference's order; NULL uses Philox4x32-10 keyed
 * by rng_seed with counter (rng_step_base + *rng_counter + t, row).  deterministic != 0 takes the mode.
 */
typedef struct OrlRolloutArgs {
    int32_t env_kind;       /* ORL_ENV_* */
    int32_t n_envs;         /* N */
    int32_t n_agents;       /* A; rows B = N*A */
    int32_t episode_length; /* T: depth of the (T[+1], B, .) buffers */
    int32_t t_begin, t_end; /* steps to run, 0 <= t_begin < t_end <= T */
    int32_t obs_dim;        /* d, policy observation width: 1..256 with ORL_ENV_NONE (host-stepped envs), 1..64
                               otherwise; ORL_ERR_BAD_ARG outside */
    int32_t critic_obs_dim; /* 0: critic obs == policy obs (critic_obs may be NULL) */
    int32_t n_actions;      /* n: Discrete(n) 1..64 with ORL_ENV_NONE (host-stepped envs), 1..8 otherwise and for
                               DiagGaussian heads; ORL_ERR_BAD_ARG outside */
    int32_t activation_id;  /* cfg.activation_id: 0 tanh, 1 relu, 2 leaky_relu, 3 elu */
    int32_t deterministic;
    int32_t env_table_len;
    const float* policy_params; /* flat net parameters, layout in orl_mlp.cuh / DESIGN.md */
    float* policy_obs;          /* (T+1, B, d)   slot t read at t_begin, slots t+1 written; 16-byte aligned for
                                   CartPole and GridWorld (one float4 per observation), else ORL_ERR_BAD_ARG */
    float* critic_obs;          /* (T+1, B, dc)  or NULL; a separate one is written like policy_obs (and must be aligned
                                   alike), except by orl_rollout on CartPole, which leaves it untouched */
    float* actions;             /* (T, B, 1)  sampled index stored as float32 (replay_data.py:163-166) */
    float* action_log_probs;    /* (T, B, 1) */
    float* rewards;             /* (T, B, 1) */
    float* masks;               /* (T+1, B, 1) */
    float* active_masks;        /* (T+1, B, 1) */
    const float* action_masks;  /* (T+1, B, n) or NULL (all actions available) */
    const float* exp_noise;     /* (T, B, n) or NULL */
    uint64_t rng_seed;
    uint64_t rng_step_base;     /* Philox counter of step t is rng_step_base + *rng_counter + t */
    uint64_t* rng_counter;      /* (1) device counter or NULL; += (t_end - t_begin) after the launch,
                                   so a captured CUDA graph draws fresh noise on every replay */
    double* env_f64;
    uint64_t* env_u64;
    int32_t* env_i32;
    const int32_t* env_table;
    float* ep_return;           /* (N) running episode return  (VecMonitor-style statistics) */
    int32_t* ep_length;         /* (N) running episode length */
    double* episode_stats;      /* (4) += {sum return, sum length, #episodes, 0} of finished episodes */
    int32_t head_kind;          /* ORL_HEAD_CATEGORICAL (Discrete(n)) or ORL_HEAD_GAUSSIAN (Box(n), DiagGaussian,
                                   distributions.py:75-98): then n_actions = action width, actions and
                                   action_log_probs are (T, B, n) (per-dimension log-probs), exp_noise holds
                                   N(0,1) draws (torch.normal == noise*std + mean) and the parameter vector ends
                                   with logstd[n].  Gaussian heads act on host-stepped envs (ORL_ENV_NONE). */
    int32_t rng_row_offset;     /* added to the row index in the Philox counter: rank r of an env-sharded run passes its
                                   first global row (r * B) with the SAME rng_seed on every rank, so that sharded rollouts
                                   draw exactly the noise the unsharded run draws for those rows */
} OrlRolloutArgs;
int orl_rollout(const OrlRolloutArgs* args, void* stream);

/* ---- critic forward over a flat batch of rows ------------------------------------------
 * Replaces the critic half of act() (ValueNetwork.forward, value_network.py:113-136) for all
 * T+1 slots at once and the bootstrap forward of OnPolicyDriver.compute_returns
 * (onpolicy_driver.py:206-215).  obs (rows, d) -> values (rows), d in 1..256 (ORL_ERR_BAD_ARG otherwise). */
int orl_critic_values(const float* critic_params, int obs_dim, int activation_id,
                      const float* obs, float* values, long long rows, void* stream);

/* ---- insert of one HOST env.step into the device rollout buffer ---------------------------
 * Replaces OnPolicyDriver.add2buffer -> ReplayData.insert (onpolicy_driver.py:80-152, replay_data.py:245-284) for
 * host-stepped envs: `staged` is the step's result as ONE uploaded block [obs (B*d) | rewards (B) | dones (B)]
 * (B = n_envs * n_agents rows); writes slot t+1 of policy_obs / masks / active_masks and slot t of rewards with the
 * reference's mask rules (masks = 0 where all agents of the env are done, active_masks = 0 for a done agent of a
 * running env).  Pointers address the given slot / row range (rows of a group are contiguous).
 * action_masks_next (nullable): when the envs reported legal-move masks (`info["action_masks"]`, prepare_action_masks,
 * envs/vec_env/utils/util.py:54-88) for this step, the staged block carries them after the dones, [... | action masks
 * (B*n_actions), n_actions in 1..64], and they are written to slot t+1 of action_masks (replay_data.py:282-283); NULL
 * writes nothing there,
 * so the slot keeps what it held, as in the reference.
 * critic_obs_next (nullable): for an env whose observation space is Dict {"policy", "critic"} (a separate critic
 * observation, as the reference's MAPPO envs give it: get_critic_obs, buffers/utils/util.py:22-55) the block carries the
 * critic observations right after the policy observations, [obs (B*d) | critic obs (B*critic_obs_dim) | rewards | ...],
 * and they are written to slot t+1 of critic_obs at the same first row; critic_obs_dim must be in 1..64
 * (ORL_ERR_BAD_ARG otherwise).  NULL: the block has no critic section. */
int orl_host_insert(const float* staged, int n_envs, int n_agents, int obs_dim, float* policy_obs_next, float* rewards,
                    float* masks_next, float* active_masks_next, float* action_masks_next, int n_actions,
                    float* critic_obs_next, int critic_obs_dim, void* stream);
/* orl_host_insert for critic sections of critic_obs_dim in 1..256, the widths of the feed-forward critic on host-stepped
 * envs; the same kernel, so for 1..64 it writes what orl_host_insert writes. */
int orl_host_insert_wide_obs(const float* staged, int n_envs, int n_agents, int obs_dim, float* policy_obs_next, float* rewards,
                             float* masks_next, float* active_masks_next, float* action_masks_next, int n_actions,
                             float* critic_obs_next, int critic_obs_dim, void* stream);

/* ---- policy evaluation of given actions over a flat batch of rows ------------------------
 * Replaces PolicyNetwork.eval_actions (policy_network.py:164-203) -> ACTLayer.evaluate_actions (act.py:130-172), the
 * policy half of PPOModule.evaluate_actions (ppo_module.py:147-193), outside the fused update: obs (rows, d), actions
 * (rows) [Categorical: index as float32] or (rows, n) [DiagGaussian] -> log_probs and entropy with the shape of
 * `actions` (per row / per dimension; the caller takes the active-mask mean, act.py:160-168).  n_actions: 1..64 for
 * Categorical heads and ORL_HEAD_GAUSSIAN_WIDE, 1..8 for ORL_HEAD_GAUSSIAN; obs_dim: 1..256 (ORL_ERR_BAD_ARG otherwise). */
int orl_policy_eval(const float* policy_params, int obs_dim, int n_actions, int activation_id, int head_kind,
                    const float* obs, const float* actions, const float* action_masks, float* log_probs,
                    float* entropy, long long rows, void* stream);


/* ---- PPO minibatch update ---------------------------------------------------------------
 * Replaces PPOAlgorithm.ppo_update (openrl/algorithms/ppo.py:46-176): prepare_loss :238-361
 * (evaluate_actions -> PolicyNetwork.eval_actions policy_network.py:164-203 / ValueNetwork.forward
 * value_network.py:113-136, ratio + clipped surrogate :300-319, cal_value_loss :178-220 incl.
 * ValueNorm.update/normalize valuenorm.py:59-90, entropy act.py:160-168, construct_loss_list
 * :226-236), loss.backward(), clip_grad_norm_ (:139-150) and Adam.step (rl_module.py:80-87), and
 * the minibatch gather of ReplayData.feed_forward_generator (replay_data.py:553-646).
 *
 * Three launches per update, all asynchronous, no host round trip:
 *   orl_ppo_fwdbwd : fused gather + forward + loss + backward over the minibatch rows; every CTA
 *                    writes its partial FOLDED gradients and loss sums to `partials`.
 *   orl_ppo_reduce : deterministic reduction of the partials over CTAs -> `folded` (2*stride
 *                    floats: policy net then critic net).  With >1 GPU the caller all-reduces
 *                    (SUM) `folded` here — the single NCCL all-reduce per update.
 *   orl_ppo_apply  : unfold to true gradients, per-net global-norm clip, Adam, ValueNorm commit,
 *                    train_info accumulation.
 * flags: */
#define ORL_PPO_HUBER 1               /* cfg.use_huber_loss */
#define ORL_PPO_CLIP_VALUE 2          /* cfg.use_clipped_value_loss */
#define ORL_PPO_VALUE_ACTIVE_MASKS 4  /* cfg.use_value_active_masks */
#define ORL_PPO_POLICY_ACTIVE_MASKS 8 /* cfg.use_policy_active_masks */
#define ORL_PPO_VALUENORM 16          /* cfg.use_valuenorm (normaliser present) */
#define ORL_PPO_ADV_NORMALIZE 32      /* cfg.use_adv_normalize (ppo.py:402-403) */
#define ORL_PPO_MAX_GRAD_NORM 64      /* cfg.use_max_grad_norm */
#define ORL_PPO_A2C 256               /* A2CAlgorithm.prepare_loss (openrl/algorithms/a2c.py:39-140): policy loss
                                         -adv * log-prob instead of the clipped surrogate; ratio reported as 0 */
#define ORL_PPO_DUAL_CLIP 512         /* cfg.dual_clip_ppo: ratio = min(ratio, dual_clip_coeff) (ppo.py:304-305) */
#define ORL_PPO_TENSORCORE 128        /* the 64x64 GEMMs of the trunk (forward, backward-data, weight gradients) on wgmma
                                         tensor cores with split-fp16 operands (x = hi + lo, three MMA passes, FP32
                                         accumulate in registers): fp32-class accuracy, same 1e-4 loss-parity bar as the FFMA
                                         kernel.  Categorical heads, obs widths <= 8, |obs| < 65504.  Minibatch tiles are
                                         staged by TMA when `indices` is NULL, by cp.async gathers otherwise.
                                         Without the flag everything is fp32 FFMA. */
#define ORL_PPO_TF32 ORL_PPO_TENSORCORE /* round-1 name of the flag */
#define ORL_PPO_JOINT_ACTION 1024     /* cfg.use_joint_action_loss (JRPO) on the recurrent update (OrlRnnArgs only, 3 agents):
                                         see orl_rnn_fwdbwd */

typedef struct OrlPpoArgs {
    int32_t obs_dim;         /* d  policy obs width  1..256; 1..64 with ORL_PPO_TENSORCORE (ORL_ERR_BAD_ARG otherwise) */
    int32_t critic_obs_dim;  /* dc critic obs width  1..256; 1..64 with ORL_PPO_TENSORCORE */
    int32_t n_actions;       /* n: 1..64 for Categorical heads, 1..8 for DiagGaussian heads and with ORL_PPO_TENSORCORE
                                (ORL_ERR_BAD_ARG otherwise) */
    int32_t activation_id;
    int32_t flags;           /* ORL_PPO_* */
    int32_t grid_per_net;    /* CTAs per net in orl_ppo_fwdbwd (partials has 2*grid_per_net rows) */
    int64_t batch_rows;      /* rows of this minibatch */
    int64_t row_begin;       /* used when indices == NULL: rows [row_begin, row_begin+batch_rows) */
    int64_t total_rows;      /* T*B, rows of the flattened buffers (bounds) */
    const int64_t* indices;  /* (batch_rows) flat row ids (torch.randperm slice) or NULL */
    /* rollout data flattened to (T*B, .) */
    const float* policy_obs;     /* (T*B, d)  */
    const float* critic_obs;     /* (T*B, dc) */
    const float* actions;        /* (T*B)     */
    const float* old_log_probs;  /* (T*B)     */
    const float* advantages;     /* (T*B) raw, normalised on the fly from gae_stats */
    const float* value_preds;    /* (T*B)     */
    const float* returns;        /* (T*B)     */
    const float* active_masks;   /* (T*B)     */
    const float* action_masks;   /* (T*B, n) or NULL */
    const double* gae_stats;     /* (ORL_GAE_NSTATS) global moments of the raw advantages */
    const double* mb_stats;      /* (3) {sum returns, sum returns^2, sum active} over this minibatch */
    float* vn_state;             /* (3) ValueNorm state BEFORE this update; orl_ppo_apply commits the update */
    float* policy_params;        /* flat, updated in place by orl_ppo_apply */
    float* critic_params;
    float* policy_adam_m; float* policy_adam_v;   /* Adam moments, same layout as params */
    float* critic_adam_m; float* critic_adam_v;
    int32_t* adam_steps;         /* (2) step counters {policy, critic}, incremented by apply */
    const float* lrs;            /* (2) {lr, critic_lr} (device so that CUDA graphs can be replayed) */
    float clip_param, entropy_coef, value_loss_coef, huber_delta, max_grad_norm;
    float adam_beta1, adam_beta2, adam_eps, weight_decay;
    float reserved0;
    double vn_beta;              /* ValueNorm beta (0.99999); double: (1 - beta) is taken in double like the reference */
    float* partials;             /* (2*grid_per_net, stride) scratch */
    float* folded;               /* (2, stride): reduced folded gradients + loss sums */
    float* grads;                /* (2, orl_ppo_grads_stride): true gradients, parameter layout (written by apply) */
    float* train_info;           /* (6) += {value_loss, critic_grad_norm, policy_loss, dist_entropy,
                                             actor_grad_norm, ratio}  (ppo.py:430-451) */
    int32_t head_kind;           /* ORL_HEAD_*: with GAUSSIAN or GAUSSIAN_WIDE actions / old_log_probs are (T*B, n) */
    float dual_clip_coeff;       /* cfg.dual_clip_coeff (used with ORL_PPO_DUAL_CLIP) */
    int64_t norm_rows;           /* rows of the GLOBAL minibatch (all ranks): the 1/rows loss weights, the reported
                                    ratio mean and the ValueNorm batch moments (mb_stats / norm_rows) refer to it, so
                                    that SUM-all-reduced gradients equal the single-process gradients of the global
                                    batch; 0 = batch_rows (single process) */
} OrlPpoArgs;
/* floats per partial row for given shapes (>= folded gradient size + 8 loss slots, multiple of 4) */
int orl_ppo_stride(int obs_dim, int critic_obs_dim, int n_actions);   /* valid for both head kinds */
/* floats per net row of `grads` (>= parameter count of the larger net, multiple of 4) */
int orl_ppo_grads_stride(int obs_dim, int critic_obs_dim, int n_actions);
/* number of parameters of one MLP net with head width n (layout in DESIGN.md) */
int orl_net_param_count(int obs_dim, int n_out);
int orl_ppo_fwdbwd(const OrlPpoArgs* args, void* stream);
int orl_ppo_reduce(const OrlPpoArgs* args, void* stream);
int orl_ppo_apply(const OrlPpoArgs* args, void* stream);

/* Multi-GPU (one process per GPU): the SUM all-reduce of the gradient bucket between orl_ppo_reduce and orl_ppo_apply
 * (the north-star's "single allreduce on the gradient bucket per update"; the reference has no distributed update) fused
 * into the two kernels over NVLink peer memory instead of a separate collective.  Every rank owns one symmetric
 * allocation of orl_ppo_peer_bucket_bytes() bytes, zero-filled before first use, mapped into all peers (CUDA VMM /
 * torch symmetric memory); peer_buffers is a DEVICE array of `world` addresses of these allocations as seen from this
 * rank (entry `rank` = local_buffer).  orl_ppo_reduce_peer PUSHES this rank's bucket into slot [parity of epochs[net]]
 * [rank] of every rank's allocation; orl_ppo_apply_peer signals the peers, waits for their buckets (error_flag := 1 + peer
 * rank if one does not arrive within timeout_ms; the logged losses are then NaN), sums the `world` slots of its own copy
 * in rank order into `summed` and applies the optimiser step exactly as orl_ppo_apply does on the sum; it increments
 * epochs[net].  All ranks must issue the same sequence of reduce_peer / apply_peer pairs. */
#define ORL_PEER_MAX_WORLD 16
#define ORL_PEER_SMALL_MAX 16   /* doubles per orl_peer_sum_f64 call */
typedef struct OrlPeerArgs {
    const uint64_t* peer_buffers; /* device (world): addresses of every rank's symmetric bucket */
    float* local_buffer;          /* this rank's symmetric bucket */
    uint32_t* epochs;             /* device (3): completed exchanges {policy bucket, critic bucket, orl_peer_sum_f64}; start at 0 */
    int32_t* error_flag;          /* device (1): 0, or 1 + rank of a peer that timed out */
    float* summed;                /* device (2, stride): receives the all-rank sum (local scratch) */
    int32_t world, rank;
    int32_t timeout_ms;           /* bound on the wait for a peer's bucket */
    int32_t reserved;
} OrlPeerArgs;
long long orl_ppo_peer_bucket_bytes(int obs_dim, int critic_obs_dim, int n_actions, int world);
int orl_ppo_reduce_peer(const OrlPpoArgs* args, const OrlPeerArgs* peer, void* stream);
int orl_ppo_apply_peer(const OrlPpoArgs* args, const OrlPeerArgs* peer, void* stream);
/* In-place SUM over all ranks of n <= ORL_PEER_SMALL_MAX doubles (the 8 rollout moments of orl_gae, all-reduced once per
 * iteration: parallel.py step 1) through the same symmetric allocation; `stride` = orl_ppo_stride() of the bucket. */
int orl_peer_sum_f64(const OrlPeerArgs* peer, int stride, double* data, int n, void* stream);
/* {sum returns, sum returns^2, sum active} over a minibatch given by `indices` (see mb_stats). */
int orl_minibatch_stats(const int64_t* indices, int64_t batch_rows, const float* returns,
                        const float* active_masks, double* mb_stats_out, void* stream);


/* ---- recurrent (GRU) policy / value networks --------------------------------------------
 * Replace, for cfg.use_recurrent_policy, RNNLayer (openrl/modules/networks/utils/rnn.py:5-99) inside
 * PolicyNetwork / ValueNetwork, the recurrent half of OnPolicyDriver.act / add2buffer
 * (onpolicy_driver.py:80-152,236-279), ReplayData.recurrent_generator (replay_data.py:1062-1258:
 * chunks of L = data_chunk_length over the agent-major / time-minor flattening f = (n*A + a)*T + t,
 * initial hidden state rnn_states[f = c*L], chunks ignore trajectory boundaries) and the BPTT part of
 * PPOAlgorithm.ppo_update.  One warp per env (rollout), row (act, critic) or chunk (update) runs the
 * warp-cooperative step of csrc/orl_rnn_warp.cuh (checked against the sequential core csrc/orl_rnn_core.h,
 * which is pinned to the oracle on the CPU); parameter gradients are reductions of a per-row tape, dW = sum P^T Q.
 * Parameter layout of a recurrent net (reference state_dict order):
 *   W1[64][d] b1 g1 be1 | W3[64][64] b3 g3 be3 | Wih[192][64] Whh[192][64] bih bhh | g_rnn be_rnn | Wh[n][64] bh[n]
 * With ORL_PPO_JOINT_ACTION (JRPO, ppo.py:254-319 + recurrent_generator_v3, replay_data.py:425-551): a chunk c covers the
 * samples f = n*T + t in [c*L, c*L + L), each carrying all A agents; the policy is evaluated on every agent row, the
 * ratio is exp(sum_a logp - sum_a old_logp) per (chunk, step) group with agent 0's advantage, the critic runs on agent
 * 0's rows only.  mb_stats then holds 6 doubles: the {sum ret, sum ret^2, sum active} moments of the agent-0 rows (value
 * loss, ValueNorm, policy-loss weights) and of all agent rows (only the active sum [5] is read: entropy weights).
 * norm_rows counts (chunk, step) groups.
 */
typedef struct OrlRnnArgs {
    int32_t env_kind, n_envs, n_agents, episode_length;   /* N, A, T; rows B = N*A */
    int32_t t_begin, t_end;
    int32_t obs_dim, critic_obs_dim, n_actions, activation_id;   /* n_actions 1..64; 1..8 for orl_rnn_rollout and with
                                                                   ORL_PPO_JOINT_ACTION (ORL_ERR_BAD_ARG otherwise).
                                                                   obs_dim / critic_obs_dim 1..256 for orl_rnn_act_rows,
                                                                   orl_rnn_critic, orl_rnn_fwdbwd and orl_rnn_apply; 1..64 for
                                                                   orl_rnn_rollout and with ORL_PPO_JOINT_ACTION */
    int32_t deterministic, chunk_length;                  /* L = cfg.data_chunk_length (<= 32) */
    int32_t flags;                                        /* ORL_PPO_* */
    int32_t env_table_len;
    int64_t n_chunks;                                     /* chunks in this minibatch */
    const int64_t* chunk_ids;                             /* (n_chunks) chunk indices c (torch.randperm slice) */
    float* policy_params; float* critic_params;
    float* policy_obs; float* critic_obs;                 /* (T+1, B, d) / (T+1, B, dc) */
    float* rnn_states; float* rnn_states_critic;          /* (T+1, B, 64) */
    float* actions; float* action_log_probs; float* rewards;
    float* masks; float* active_masks;
    float* value_preds; const float* returns; const float* advantages;
    const float* exp_noise;                               /* (T, B, n) or NULL */
    uint64_t rng_seed; uint64_t rng_step_base; uint64_t* rng_counter;
    double* env_f64; uint64_t* env_u64; int32_t* env_i32; const int32_t* env_table;
    float* ep_return; int32_t* ep_length; double* episode_stats;
    const double* gae_stats; const double* mb_stats; float* vn_state;
    float* tape;                                          /* workspace: orl_rnn_workspace_floats_wide_obs(n_chunks*L, grads_stride, n_actions, obs_dim,
                                                             critic_obs_dim) floats (the larger net's tape rows, the reduction partials, then with a
                                                             net wider than 64 the dW1 panel buffer); n_chunks*L*A rows with ORL_PPO_JOINT_ACTION */
    float* grads;                                         /* (2, grads_stride) true gradients, policy then critic */
    int32_t grads_stride; int32_t reserved1;
    float* loss_acc;                                      /* (8) zeroed by orl_rnn_fwdbwd: policy_loss, entropy, ratio, value_loss sums */
    float* policy_adam_m; float* policy_adam_v; float* critic_adam_m; float* critic_adam_v;
    int32_t* adam_steps; const float* lrs;
    float clip_param, entropy_coef, value_loss_coef, huber_delta, max_grad_norm;
    float adam_beta1, adam_beta2, adam_eps, weight_decay, dual_clip_coeff;
    double vn_beta;
    float* train_info;
    int64_t norm_rows;                                    /* row-steps of the GLOBAL minibatch (see OrlPpoArgs.norm_rows); 0 = n_chunks*L */
    /* orl_rnn_act_rows only: */
    int32_t rng_row_offset;                               /* added to the buffer row in the action-noise key (first GLOBAL row of this buffer) */
    int32_t row_begin, row_end;                           /* buffer rows [row_begin, row_end) of slot t_begin */
    int32_t reserved2;
    /* (T+1, B, n) legal-move masks (0 = illegal: logit -6e4, no gradient; distributions.py:71) or NULL (every action
     * legal).  Read by orl_rnn_act_rows (slot t_begin) and by the policy pass of orl_rnn_fwdbwd; when the
     * ORL_PPO_JOINT_ACTION flag is set, orl_rnn_fwdbwd rejects it (ORL_ERR_BAD_ARG); orl_rnn_rollout (device envs, which
     * report no masks) ignores it. */
    const float* action_masks;
    /* ORL_HEAD_CATEGORICAL (0, a zeroed struct) or ORL_HEAD_GAUSSIAN: a DiagGaussian policy head of 1..8 dimensions, whose
     * parameters end in logstd[n] (orl_rnn_param_count_head) and whose actions / action_log_probs are (T, B, n); the
     * parity-mode exp_noise of orl_rnn_act_rows is then a (B, n) table of N(0, 1) draws.  Taken by orl_rnn_act_rows,
     * orl_rnn_critic, orl_rnn_fwdbwd and orl_rnn_apply; ORL_ERR_BAD_ARG from orl_rnn_rollout (device envs are Discrete),
     * with ORL_PPO_JOINT_ACTION, with n_actions > 8 and for any other value.  ORL_HEAD_GAUSSIAN_WIDE: the same for a
     * DiagGaussian policy head of 9..64 dimensions (ORL_ERR_BAD_ARG with n_actions <= 8), on the 64-wide head of the GRU
     * kernels. */
    int32_t head_kind;
    int32_t reserved3;
} OrlRnnArgs;
int orl_rnn_param_count(int obs_dim, int n_out);
/* parameters of a GRU policy of head_kind: orl_rnn_param_count plus n for the logstd of ORL_HEAD_GAUSSIAN and
 * ORL_HEAD_GAUSSIAN_WIDE */
int orl_rnn_param_count_head(int obs_dim, int n_out, int head_kind);
int orl_rnn_tape_width(void);
/* floats of OrlRnnArgs.tape for a minibatch of `rows` = n_chunks * chunk_length row-steps (times A with ORL_PPO_JOINT_ACTION)
 * of a policy with at most 8 actions */
long long orl_rnn_workspace_floats(long long rows, int grads_stride);
/* the same for a policy of n_actions actions: a wide head (9..64 actions) tapes dL/dlogits in 64 more floats per row
 * (orl_rnn_tape_width() + 64); equal to orl_rnn_workspace_floats for n_actions <= 8 */
long long orl_rnn_workspace_floats_for(long long rows, int grads_stride, int n_actions);
/* the same for observations of obs_dim / critic_obs_dim 1..256: a net wider than 64 tapes its observation in 256 more
 * floats per row, and its W1 gradient takes a panel buffer of 64 x 256 floats after the partials; equal to
 * orl_rnn_workspace_floats_for when both widths are <= 64 */
long long orl_rnn_workspace_floats_wide_obs(long long rows, int grads_stride, int n_actions, int obs_dim, int critic_obs_dim);
/* the same for a policy head of head_kind: an ORL_HEAD_GAUSSIAN policy tapes dL/dlogstd in 8 more floats per row (before
 * the observation field of a net wider than 64), an ORL_HEAD_GAUSSIAN_WIDE policy (9..64 dimensions) in 64 more floats
 * after the wide head's dL/dmean (rows of 1872, or 2128 with the observation field); equal to
 * orl_rnn_workspace_floats_wide_obs for ORL_HEAD_CATEGORICAL */
long long orl_rnn_workspace_floats_head(long long rows, int grads_stride, int n_actions, int obs_dim, int critic_obs_dim,
                                        int head_kind);
/* policy GRU rollout for steps [t_begin, t_end) fused with the device env (simple_spread, CartPole, GridWorld); device
 * envs only: ORL_ENV_NONE is rejected (the policy step of host-stepped rows is orl_rnn_act_rows).  CartPole and
 * GridWorld need 16-byte aligned policy_obs and critic_obs (ORL_ERR_BAD_ARG otherwise). */
int orl_rnn_rollout(const OrlRnnArgs* args, void* stream);
/* policy GRU act for a HOST-stepped env: one step t = t_begin over buffer rows [row_begin, row_end) (B = n_envs *
 * n_agents rows per slot).  Reads policy_obs[t], rnn_states[t], masks[t]; writes actions[t], action_log_probs[t] and
 * rnn_states[t+1] (orl_host_insert_rnn zeroes the rows of the envs that finish at step t).  The action noise of row r is
 * keyed by (rng_seed, rng_step_base + *rng_counter, r + rng_row_offset) — the slot index is not added — and rng_counter
 * (nullable) advances by one per call; exp_noise (parity mode, nullable) is the (B, n) Exp(1) table of this slot,
 * indexed by buffer row.  With head_kind ORL_HEAD_GAUSSIAN (1..8 dimensions) it writes the (B, n) actions and log-probs
 * of slot t: mean + std * N(0, 1), the normals drawn as the feed-forward act draws them for the same key (Box-Muller of
 * Philox lanes 2..5), or read from exp_noise, then a (B, n) table of N(0, 1) draws; deterministic returns the mean.
 * ORL_HEAD_GAUSSIAN_WIDE (9..64 dimensions) does the same with the feed-forward wide head's noise: dimensions
 * [4k, 4k + 4) are Box-Muller of Philox lanes 2 + 2k and 3 + 2k, so dimensions 0..7 draw what ORL_HEAD_GAUSSIAN draws. */
int orl_rnn_act_rows(const OrlRnnArgs* args, void* stream);
/* orl_host_insert for a recurrent policy: additionally zeroes the 64-float rnn_states_next row of every agent of an env
 * whose agents are all done (rnn_states[dones_env] = 0, onpolicy_driver.py:262-269).  rnn_states_next addresses slot
 * t+1 at the same first row as the other pointers; action_masks_next / n_actions and critic_obs_next / critic_obs_dim
 * as in orl_host_insert, except that masks take n_actions in 1..8 (ORL_ERR_BAD_ARG otherwise). */
int orl_host_insert_rnn(const float* staged, int n_envs, int n_agents, int obs_dim, float* policy_obs_next, float* rewards,
                        float* masks_next, float* active_masks_next, float* rnn_states_next, float* action_masks_next,
                        int n_actions, float* critic_obs_next, int critic_obs_dim, void* stream);
/* orl_host_insert_rnn for masks of n_actions in 1..64, the widths of a GRU policy's wide head (9..64 actions) included;
 * the same kernel, so for 1..8 actions it writes what orl_host_insert_rnn writes. */
int orl_host_insert_rnn_wide(const float* staged, int n_envs, int n_agents, int obs_dim, float* policy_obs_next, float* rewards,
                             float* masks_next, float* active_masks_next, float* rnn_states_next, float* action_masks_next,
                             int n_actions, float* critic_obs_next, int critic_obs_dim, void* stream);
/* orl_host_insert_rnn_wide for critic sections of critic_obs_dim in 1..256 (ORL_ERR_BAD_ARG otherwise), the critic of a
 * GRU MAPPO env wider than 64 included; the same kernel, so for 1..64 it writes what orl_host_insert_rnn_wide writes. */
int orl_host_insert_rnn_wide_obs(const float* staged, int n_envs, int n_agents, int obs_dim, float* policy_obs_next, float* rewards,
                                 float* masks_next, float* active_masks_next, float* rnn_states_next, float* action_masks_next,
                                 int n_actions, float* critic_obs_next, int critic_obs_dim, void* stream);
/* recurrent critic over slots 0..T: value_preds[t] and rnn_states_critic[t+1] */
int orl_rnn_critic(const OrlRnnArgs* args, void* stream);
/* chunked BPTT forward + loss + backward of both nets over the minibatch chunks -> grads, loss_acc */
int orl_rnn_fwdbwd(const OrlRnnArgs* args, void* stream);
/* per-net global-norm clip + Adam on `grads`; ValueNorm commit; train_info accumulation */
int orl_rnn_apply(const OrlRnnArgs* args, void* stream);


/* ---- self-play: two-player GridWorld against an opponent pool in HBM -----------------------
 * Replaces, for BASELINE configs[3], the self-play control flow of the reference around the rollout:
 * OpponentPoolWrapper.reset / get_opponent_action / on_episode_end (openrl/selfplay/wrappers/opponent_pool_wrapper.py:
 * 30-120), RandomOpponent / LastOpponent.sample_opponent (selfplay/sample_strategy/random_opponent.py:25-28,
 * last_opponent.py:24-27); the snapshot cadence of SelfplayCallback._on_step (selfplay/callbacks/selfplay_callback.py:
 * 124-144) is the host's job (it copies the learner's parameters into the pool ring and bumps *pool_count).
 * The env (rules in csrc/orl_selfplay.cu and oracle/selfplay.py; new env, SURVEY.md §8f-2): the learner is player 0 of a
 * 10x10 two-player GridWorld and sees (x0, y0, x1, y1); player 1 is driven by the snapshot pool_params[opponent index]
 * (same policy architecture, d = 4, n = 5) drawn per episode, or acts uniformly at random while the pool is empty.
 * rollout.env_kind = ORL_ENV_GRIDWORLD_2P, rollout.env_i32 = [8][N] (x0, y0, x1, y1, steps, #resets, opponent, -),
 * rollout.env_table = optional [N][len][4] start cells, rollout.deterministic bits: 1 = greedy learner, 2 = learner
 * actions scripted from exp_noise[(t*N+e)*2 + 0], 4 = opponent actions scripted from exp_noise[(t*N+e)*2 + 1]. */
#define ORL_ENV_GRIDWORLD_2P 4
#define ORL_SP_RANDOM 0   /* RandomOpponent: uniform over the snapshots in the ring */
#define ORL_SP_LAST 1     /* LastOpponent: the newest snapshot */
typedef struct OrlSelfPlayArgs {
    OrlRolloutArgs rollout;
    const float* pool_params;    /* (pool_capacity, pool_stride) policy snapshots, flat parameter layout */
    const int32_t* pool_count;   /* (1) device: number of snapshots ever added; ring slot of snapshot k = k % pool_capacity */
    int32_t* pool_stats;         /* (pool_capacity + 1, 3) += wins / losses / draws of the training agent against each ring
                                    slot (last row: the random-action opponent), opponent_pool_wrapper.py:91-120 */
    int32_t pool_capacity, pool_stride, strategy, reserved;
} OrlSelfPlayArgs;
int orl_selfplay_reset(const OrlSelfPlayArgs* args, float* policy_obs_out, void* stream);
int orl_selfplay_rollout(const OrlSelfPlayArgs* args, void* stream);

/* ---- shared policy-value network (cfg.use_share_model) -----------------------------------
 * Replace, for cfg.use_share_model, PolicyValueNetwork (openrl/modules/networks/policy_value_network.py:33-174:
 * obs_prep MLPBase -> common MLPLayer(64, 64, layer_N=0) -> {v_out, act}) in the rollout (get_actions), the value pass
 * (get_values) and PPOAlgorithm.ppo_update with `_use_share_model` (ppo.py:46-176: both losses into one set of
 * gradients, clip_grad_norm_ over all parameters twice, ONE Adam step with lr = cfg.lr).
 * Parameter layout (named_parameters order of the reference):
 *   W1[64][d] b1 g1 be1 | W3[64][64] b3 g3 be3 | W5[64][64] b5 g5 be5 | W7[64][64] b7 g7 be7 | Wv[1][64] bv | Wa[n][64] ba
 *   then, for a DiagGaussian head, logstd[n] (act.action_out.logstd._bias).
 * head_kind ORL_HEAD_CATEGORICAL: Discrete(n) actions, single-agent device envs or ORL_ENV_NONE.  ORL_HEAD_GAUSSIAN:
 * Box(n <= 8) actions, ORL_ENV_NONE only (host-stepped envs); actions / log-probs are (rows, n), no action masks.
 * OrlRolloutArgs.policy_params = the shared model.
 * OrlPpoArgs for the shared model: policy_params / policy_adam_* / lrs[0] / adam_steps[0] = the shared model and its
 * optimiser, partials = workspace of orl_share_workspace_floats() floats, grads = true gradients (>= parameter count),
 * folded = 8 floats of loss sums; critic_* fields are ignored.  With > 1 GPU the caller SUM-all-reduces `grads` and
 * `folded[0..3]` between orl_share_fwdbwd and orl_share_apply.
 * orl_share_param_count / orl_share_tape_width / orl_share_workspace_floats are the Categorical head's; the _head
 * variants take the head kind. */
int orl_share_param_count(int obs_dim, int n_actions);
int orl_share_param_count_head(int obs_dim, int n_actions, int head_kind);
int orl_share_tape_width(void);
long long orl_share_workspace_floats(long long rows, int obs_dim, int n_actions);
long long orl_share_workspace_floats_head(long long rows, int obs_dim, int n_actions, int head_kind);
int orl_share_rollout(const OrlRolloutArgs* args, void* stream);
int orl_share_values(const float* params, int obs_dim, int n_actions, int activation_id, const float* obs, float* values,
                     long long rows, void* stream);
int orl_share_fwdbwd(const OrlPpoArgs* args, void* stream);
int orl_share_apply(const OrlPpoArgs* args, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* OPENRL_B200_H */
