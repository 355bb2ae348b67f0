"""Device-resident vectorised environment with the reference's BaseVecEnv duck type.

Replaces SyncVectorEnv / AsyncVectorEnv + RewardWrapper + VecMonitorWrapper
(openrl/envs/vec_env/{sync_venv,async_venv}.py, wrappers/{reward_wrapper,vec_monitor_wrapper}.py)
for the envs that have a CUDA step function (CartPole-v1, GridWorldEnv).  All env state lives in
CUDA tensors owned by this object; stepping happens inside `orl_rollout` (fused with the policy)
or, for the plain `step()` API, through `orl_env_step`.  Precedent for handing a GPU-resident
vec-env straight to PPONet/PPOAgent: examples/isaac/isaac2openrl.py:28-96.

Interface kept (usage: rl_driver.py:118-131, onpolicy_driver.py:172-203):
  parallel_env_num, agent_num, observation_space, action_space, env_name, use_monitor,
  reset(seed=, options=) -> (obs, infos), step(actions, extra_data) -> (obs, rewards (N,A,1),
  dones (N,A) bool, infos list[dict]), batch_rewards(buffer), statistics(buffer), close(),
  random_action().
"""
import time

import numpy as np
import torch

from .. import _kinds
from ... import lib, spaces


def _pcg64_streams(seed, n, index_offset=0):
    """Host-side seeding only (SeedSequence -> PCG64 initial state, sync_venv.py:137 +
    gymnasium/utils/seeding.py): env i gets np.random.PCG64(SeedSequence(seed + i*10086))."""
    out = np.zeros((4, n), np.uint64)
    mask = (1 << 64) - 1
    for i in range(n):
        s = None if seed is None else seed + (index_offset + i) * 10086
        st = np.random.PCG64(np.random.SeedSequence(s)).state["state"]
        out[0, i], out[1, i] = st["state"] >> 64, st["state"] & mask
        out[2, i], out[3, i] = st["inc"] >> 64, st["inc"] & mask
    return out


class DeviceVecEnv:
    def __init__(self, env_id, env_num, device="cuda:0", seed=None, reset_table=None, env_index_offset=0, opponent_pool_size=8,
                 opponent_strategy="RandomOpponent"):
        spec = _kinds.ENV_SPECS[env_id]
        self.env_name = env_id
        # global index of env 0 when a larger vec-env is sharded over ranks (multi-GPU): env i is seeded
        # seed + (offset + i)*10086, i.e. exactly the stream it would own in the unsharded vec-env
        self.env_index_offset = int(env_index_offset)
        self.kind = spec["kind"]
        self.parallel_env_num = int(env_num)
        self.agent_num = spec["agents"]
        self.obs_dim = spec["obs_dim"]
        self.critic_obs_dim = spec.get("critic_obs_dim", 0)  # 0: critic observes the policy observation
        self.n_actions = spec["n_actions"]
        self.observation_space = spec["observation_space"]()
        self.action_space = spaces.Discrete(self.n_actions)
        self.device = torch.device(device)
        self.use_monitor = True
        self._lib = lib.load()
        N = self.parallel_env_num
        dev = self.device
        self.env_f64 = torch.zeros(spec.get("f64_rows", 4), N, dtype=torch.float64, device=dev)
        self.env_u64 = torch.zeros(4, N, dtype=torch.int64, device=dev)  # bit pattern of uint64
        self.env_i32 = torch.zeros(spec.get("i32_rows", 4), N, dtype=torch.int32, device=dev)
        self.ep_return = torch.zeros(N, dtype=torch.float32, device=dev)
        self.ep_length = torch.zeros(N, dtype=torch.int32, device=dev)
        self.episode_stats = torch.zeros(4, dtype=torch.float64, device=dev)
        self.rng_seed = 0
        self.env_table = None
        self.env_table_len = 0
        self.opponent_pool = None
        if self.kind == lib.ENV_GRIDWORLD_2P:
            from ...selfplay import OpponentPool

            n_params = int(self._lib.orl_net_param_count(self.obs_dim, self.n_actions))
            self.opponent_pool = OpponentPool(opponent_pool_size, n_params, opponent_strategy, device=dev)
        if reset_table is not None:  # (N, K, 2) int start cells for GridWorld parity runs ((N, K, 4) for the 2-player grid)
            t = torch.as_tensor(np.asarray(reset_table), dtype=torch.int32).contiguous()
            self.env_table = t.to(dev)
            self.env_table_len = int(t.shape[1])
        self._obs = torch.zeros(N * self.agent_num, self.obs_dim, dtype=torch.float32, device=dev)
        self._critic_obs = (torch.zeros(N * self.agent_num, self.critic_obs_dim, dtype=torch.float32, device=dev)
                            if self.critic_obs_dim else None)
        self._start_time = time.time()
        self._total_step = 0
        self._seed_streams(seed)

    # -- seeding / reset -------------------------------------------------------------------
    def _seed_streams(self, seed):
        if self.kind in (lib.ENV_CARTPOLE, lib.ENV_MPE_SPREAD):
            st = _pcg64_streams(seed, self.parallel_env_num, self.env_index_offset)
            self.env_u64.copy_(torch.from_numpy(st.view(np.int64)))
        self.rng_seed = int(seed if seed is not None else np.random.SeedSequence().entropy % (1 << 63))

    def reset(self, seed=None, options=None):
        if seed is not None:
            self._seed_streams(int(seed))
        self.reset_into(self._obs, self._critic_obs)
        return self._host_obs(), [{} for _ in range(self.parallel_env_num)]

    def _host_obs(self):
        N, A = self.parallel_env_num, self.agent_num
        pol = self._obs.view(N, A, self.obs_dim).cpu().numpy()
        if self._critic_obs is None:
            return pol
        return {"policy": pol, "critic": self._critic_obs.view(N, A, self.critic_obs_dim).cpu().numpy()}

    def reset_into(self, obs_out, critic_obs_out=None):
        """Device-side reset writing the (B, d) observations (and (B, d_c) critic observations) into
        the given tensors (no host copy)."""
        L = self._lib
        if self._critic_obs is not None and critic_obs_out is None:
            critic_obs_out = self._critic_obs
        if self.kind == lib.ENV_GRIDWORLD_2P:
            lib.check(L.orl_selfplay_reset(self.selfplay_args(), lib.ptr(obs_out), lib.current_stream()), "orl_selfplay_reset")
            self.ep_return.zero_()
            self.ep_length.zero_()
            if obs_out.data_ptr() != self._obs.data_ptr():
                self._obs.copy_(obs_out.view_as(self._obs))
            return
        lib.check(L.orl_env_reset(self.kind, self.parallel_env_num, self.agent_num, lib.ptr(self.env_f64),
                                  lib.ptr(self.env_u64), lib.ptr(self.env_i32), lib.ptr(self.env_table),
                                  self.env_table_len, self.rng_seed, lib.ptr(obs_out), lib.ptr(critic_obs_out),
                                  lib.current_stream()), "orl_env_reset")
        self.ep_return.zero_()
        self.ep_length.zero_()
        if obs_out.data_ptr() != self._obs.data_ptr():
            self._obs.copy_(obs_out.view_as(self._obs))
        if critic_obs_out is not None and critic_obs_out.data_ptr() != self._critic_obs.data_ptr():
            self._critic_obs.copy_(critic_obs_out.view_as(self._critic_obs))

    # -- self-play (ENV_GRIDWORLD_2P) ----------------------------------------------------------
    def selfplay_args(self, rollout=None):
        """OrlSelfPlayArgs around `rollout` (an OrlRolloutArgs; a minimal one for reset when None)."""
        s = lib.OrlSelfPlayArgs()
        a = rollout if rollout is not None else lib.OrlRolloutArgs()
        if rollout is None:
            a.env_kind, a.n_envs, a.n_agents = self.kind, self.parallel_env_num, 1
            a.obs_dim, a.n_actions = self.obs_dim, self.n_actions
            a.env_i32, a.env_table, a.env_table_len = lib.ptr(self.env_i32), lib.ptr(self.env_table), self.env_table_len
            a.rng_seed, a.rng_row_offset = self.rng_seed, self.env_index_offset
        s.rollout = a
        p = self.opponent_pool
        s.pool_params, s.pool_count, s.pool_stats = lib.ptr(p.params), lib.ptr(p.count_dev), lib.ptr(p.stats)
        s.pool_capacity, s.pool_stride, s.strategy = p.capacity, p.stride, p.strategy
        return s

    def _selfplay_step(self, actions):
        """vec-env step API for the 2-player grid: the learner's actions are given, the opponent acts from the pool with the
        snapshots' activation.  Runs the rollout kernel for one step on a two-slot scratch buffer (policy parameters are not
        needed: actions are scripted)."""
        N = self.parallel_env_num
        dev = self.device
        if getattr(self, "_sp_scratch", None) is None:
            z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)   # noqa: E731
            n_params = int(self._lib.orl_net_param_count(self.obs_dim, self.n_actions))
            self._sp_scratch = dict(obs=z(2, N, 4), act=z(1, N), logp=z(1, N), rew=z(1, N), masks=z(2, N), active=z(2, N), scripted=z(1, N, 2),
                                    params=z(n_params))
        sc = self._sp_scratch
        sc["obs"][0].copy_(self._obs.view(N, 4))
        sc["scripted"][0, :, 0].copy_(torch.as_tensor(np.asarray(actions, dtype=np.float32).reshape(N)).to(dev))
        a = lib.OrlRolloutArgs()
        a.env_kind, a.n_envs, a.n_agents, a.episode_length = self.kind, N, 1, 1
        a.t_begin, a.t_end, a.obs_dim, a.n_actions, a.deterministic = 0, 1, 4, self.n_actions, 2
        a.activation_id = self.opponent_pool.activation_id   # the kernel evaluates the pool's snapshots with this activation
        a.policy_params, a.policy_obs = lib.ptr(sc["params"]), lib.ptr(sc["obs"])
        a.actions, a.action_log_probs, a.rewards = lib.ptr(sc["act"]), lib.ptr(sc["logp"]), lib.ptr(sc["rew"])
        a.masks, a.active_masks, a.exp_noise = lib.ptr(sc["masks"]), lib.ptr(sc["active"]), lib.ptr(sc["scripted"])
        self._sp_steps = getattr(self, "_sp_steps", 0) + 1
        a.rng_seed, a.rng_step_base, a.rng_row_offset = self.rng_seed, (1 << 40) + self._sp_steps, self.env_index_offset
        a.env_i32, a.env_table, a.env_table_len = lib.ptr(self.env_i32), lib.ptr(self.env_table), self.env_table_len
        a.ep_return, a.ep_length, a.episode_stats = lib.ptr(self.ep_return), lib.ptr(self.ep_length), lib.ptr(self.episode_stats)
        lib.check(self._lib.orl_selfplay_rollout(self.selfplay_args(a), lib.current_stream()), "orl_selfplay_rollout(step)")
        self._obs.view(N, 4).copy_(sc["obs"][1])
        obs = self._host_obs()
        dones = (sc["masks"][1].cpu().numpy() == 0).reshape(N, 1)
        rewards = sc["rew"][0].cpu().numpy().astype(np.float64).reshape(N, 1, 1)
        return obs, rewards, dones, [{} for _ in range(N)]

    # -- plain step API (evaluation loops; the training loop uses the fused rollout) ---------
    def step(self, actions, extra_data=None):
        if self.kind == lib.ENV_GRIDWORLD_2P:
            return self._selfplay_step(actions)
        N, A = self.parallel_env_num, self.agent_num
        act = torch.as_tensor(np.asarray(actions, dtype=np.float32).reshape(N * A)).to(self.device)
        rew = torch.empty(N * A, dtype=torch.float32, device=self.device)
        done = torch.empty(N * A, dtype=torch.float32, device=self.device)
        # last output: terminal observation (single-agent envs) or the critic observation (simple_spread)
        fin = self._critic_obs if self._critic_obs is not None else torch.empty(N * A, self.obs_dim, dtype=torch.float32, device=self.device)
        lib.check(self._lib.orl_env_step(self.kind, N, A, lib.ptr(self.env_f64), lib.ptr(self.env_u64),
                                         lib.ptr(self.env_i32), lib.ptr(self.env_table), self.env_table_len,
                                         self.rng_seed, lib.ptr(self.ep_return), lib.ptr(self.ep_length),
                                         lib.ptr(self.episode_stats), lib.ptr(act), lib.ptr(self._obs), lib.ptr(rew),
                                         lib.ptr(done), lib.ptr(fin), lib.current_stream()), "orl_env_step")
        obs = self._host_obs()
        dones = done.view(N, A).cpu().numpy() != 0
        rewards = rew.view(N, A, 1).cpu().numpy().astype(np.float64)
        infos = []
        if self._critic_obs is None:
            fin_h = fin.view(N, A, self.obs_dim).cpu().numpy()
            for i in range(N):
                info = {}
                if dones[i].all():
                    info["final_observation"] = fin_h[i]
                    info["final_info"] = {}
                infos.append(info)
        else:  # MPE: a list of per-agent dicts (multiagent_env.py:184-188)
            infos = [[{"individual_reward": float(rewards[i, a, 0]) / A} for a in range(A)] for i in range(N)]
        return obs, rewards, dones, infos

    def random_action(self, infos=None):
        return np.array([[[self.action_space.sample()] for _ in range(self.agent_num)]
                         for _ in range(self.parallel_env_num)])

    # -- statistics (SimpleVecInfo.statistics, vec_info/simple_vec_info.py:18-32) ------------
    def batch_rewards(self, buffer):
        return {}

    def statistics_device(self, buffer, out):
        """Device half of `statistics` (graph-capturable): out[:A] = per-agent rollout reward, out[A:A+4] = episode_stats
        (then zeroed).  `statistics_host` turns the copied-back vector into the reference's info dict."""
        rewards = buffer.data.rewards
        A = self.agent_num
        out[:A].copy_(rewards.mean(dim=1).sum(dim=0).reshape(-1).to(out.dtype))
        out[A:A + 4].copy_(self.episode_stats)
        self.episode_stats.zero_()

    def statistics_host(self, vals, steps):
        A = self.agent_num
        self._total_step += steps
        info = {f"agent_{i}/rollout_episode_reward": float(v) for i, v in enumerate(vals[:A])}
        info["FPS"] = int(self._total_step / max(time.time() - self._start_time, 1e-9))
        info["rollout_episode_reward"] = float(np.mean(vals[:A]))
        st = vals[A:A + 4]
        if st[2] > 0:
            info["episode_return_mean"] = float(st[0] / st[2])
            info["episode_length_mean"] = float(st[1] / st[2])
        return info

    def statistics(self, buffer):
        rewards = buffer.data.rewards  # (T, N, A, 1) device
        T, N = rewards.shape[0], rewards.shape[1]
        self._total_step += T * N
        per_agent = rewards.mean(dim=1).sum(dim=0).reshape(-1)  # (A,)
        vals = per_agent.cpu().numpy()
        self.d2h_bytes = getattr(self, "d2h_bytes", 0) + vals.nbytes + 32
        info = {f"agent_{i}/rollout_episode_reward": float(v) for i, v in enumerate(vals)}
        info["FPS"] = int(self._total_step / max(time.time() - self._start_time, 1e-9))
        info["rollout_episode_reward"] = float(np.mean(vals))
        st = self.episode_stats.cpu().numpy()
        if st[2] > 0:
            info["episode_return_mean"] = float(st[0] / st[2])
            info["episode_length_mean"] = float(st[1] / st[2])
        self.episode_stats.zero_()
        return info

    # call / get_attr / set_attr / exec_func (base_venv.py:231-302).  There are no per-env Python objects on the device:
    # a property of the vec-env is reported once per env, setting broadcasts, exec_func sees lightweight per-env views.
    def call(self, name, *args, **kwargs):
        f = getattr(self, name)
        v = f(*args, **kwargs) if callable(f) else f
        return [v for _ in range(self.parallel_env_num)]

    def get_attr(self, name):
        return self.call(name)

    def set_attr(self, name, values):
        if isinstance(values, (list, tuple)):
            if len(values) != self.parallel_env_num:
                raise ValueError(f"Values must be a list or tuple with length equal to the number of environments. "
                                 f"Got `{len(values)}` values for {self.parallel_env_num} environments.")
            if any(v != values[0] for v in values[1:]):
                raise NotImplementedError("per-env attribute values are not supported by the device vec-env (one batched state)")
            values = values[0]
        setattr(self, name, values)

    def exec_func(self, func, indices=None, *args, **kwargs):
        import types

        idx = range(self.parallel_env_num) if indices is None else indices
        return [func(types.SimpleNamespace(index=i, vec_env=self, observation_space=self.observation_space,
                                           action_space=self.action_space, env_name=self.env_name), *args, **kwargs) for i in idx]

    def close(self):
        pass
