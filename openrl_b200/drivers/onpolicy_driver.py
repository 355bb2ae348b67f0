"""OnPolicyDriver: rollout -> returns -> update loop on the device
(reference: openrl/drivers/rl_driver.py:27-180, onpolicy_driver.py:32-279).

Per iteration (`_inner_loop`):
  actor_rollout   ONE orl_rollout launch for all T steps when no callback needs per-step locals
                  (envs are independent; SURVEY.md §5.5), else T one-step launches with the
                  reference's `update_locals(locals()) / on_step()` contract;
  compute_returns one orl_critic_values launch over the (T+1)*B observations (values of every
                  slot + bootstrap), then the orl_gae scan (returns + raw advantages + moments);
  trainer.train   ppo_epoch x num_mini_batch fused updates;
  after_update    slot T -> slot 0.
Sampling noise: cfg.parity_mode draws `exponential_` per step from torch's global CPU generator in
the reference's order (act.py:79-81 -> torch.multinomial) and uploads it; otherwise Philox on device.
"""
import numpy as np
import torch

from .. import lib


class OnPolicyDriver:
    def __init__(self, config, trainer, buffer, agent, rank=0, world_size=1, client=None, logger=None, callback=None):
        cfg = config["cfg"]
        self.cfg = cfg
        self.trainer, self.buffer, self.agent = trainer, buffer, agent
        self.envs = config["envs"]
        self.device = config["device"]
        self.num_agents = config["num_agents"]
        self.rank, self.world_size = rank, world_size
        self.logger, self.callback = logger, callback
        self.num_env_steps = cfg.num_env_steps
        self.episode_length = cfg.episode_length
        self.n_rollout_threads = cfg.n_rollout_threads
        self.learner_n_rollout_threads = cfg.learner_n_rollout_threads
        self.use_linear_lr_decay = cfg.use_linear_lr_decay
        self.log_interval = cfg.log_interval
        self.episode = 0
        self.total_num_steps = 0
        self._lib = lib.load()
        self._global_step = 0
        self.rng_counter = torch.zeros(1, dtype=torch.int64, device=self.device)
        self.host_act_steps = 0     # slots acted on by host-stepped rollouts: the Philox step of slot t is this + t
        self.gpu_launches = 0
        self.h2d_bytes = 0
        self.d2h_bytes = 0
        self.phase_events = None  # set to a list by bench.py to collect (name, start, end) CUDA events
        self.recurrent = bool(cfg.use_recurrent_policy or getattr(cfg, "use_naive_recurrent_policy", False))
        if self.recurrent and self.envs.kind == lib.ENV_NONE and getattr(cfg, "use_joint_action_loss", False):
            raise NotImplementedError("use_joint_action_loss (JRPO) is built for simple_spread on the device (3 agents, agent-0 "
                                      "critic); host-stepped envs take the per-agent recurrent update")
        if self.envs.kind == lib.ENV_NONE and getattr(trainer, "share", False) and getattr(self.envs, "dict_obs", False):
            # the shared net's update computes the value from policy_obs (critic_obs_prep is obs_prep, policy_value_network.py:75)
            raise NotImplementedError("use_share_model computes the value from the policy observation; a host env with a "
                                      "Dict {'policy', 'critic'} observation space needs the two-net policy and critic")

    # -- reference surface -------------------------------------------------------------------
    def run(self):
        episodes = int(self.num_env_steps) // self.episode_length // self.learner_n_rollout_threads
        self.episodes = episodes
        self.reset_and_buffer_init()
        for episode in range(episodes):
            if self.cfg.log_each_episode and self.logger is not None:
                self.logger.info("Episode: {}/{}".format(episode, episodes))
            self.episode = episode
            if not self._inner_loop():
                break

    def reset_and_buffer_init(self):
        d = self.buffer.data
        cri = None if d.critic_obs is d.policy_obs else d.critic_obs[0].view(-1, d.critic_obs_dim)
        if self.envs.kind == lib.ENV_NONE and not d.continuous:
            # rl_driver.py:118-131: the reset infos' action masks go to slot 0 (init_buffer, replay_data.py:286-298)
            if self.envs.reset_into(d.policy_obs[0].view(-1, d.obs_dim), cri, d.action_masks[0].view(-1, d.n_actions)):
                d.action_masks_trivial = False
        else:
            self.envs.reset_into(d.policy_obs[0].view(-1, d.obs_dim), cri)  # rl_driver.py:118-131, no host copy
        d.masks[0].fill_(1.0)
        d.active_masks[0].fill_(1.0)

    def _selfplay_snapshot(self):
        """SelfplayCallback._on_step cadence (selfplay_callback.py:124-144): every `selfplay_save_freq` iterations the learner's
        current policy becomes the newest opponent of the pool (device copy; a captured graph sees it on its next replay)."""
        pool = getattr(self.envs, "opponent_pool", None)
        freq = int(getattr(self.cfg, "selfplay_save_freq", 5))
        if pool is not None and freq > 0 and (self.episode + 1) % freq == 0:
            pol = self.trainer.algo_module.models["policy"]
            pool.add(pol.flat_params, self.agent.num_time_steps, activation_id=pol.activation_id)

    # -- one captured CUDA graph per iteration -------------------------------------------------
    def _graph_ok(self):
        import os

        return (bool(getattr(self.cfg, "use_cuda_graph", True)) and not os.environ.get("ORL_NO_GRAPH") and not self.cfg.parity_mode
                and self.callback is None
                and self.envs.kind != lib.ENV_NONE and self.phase_events is None and hasattr(self.envs, "statistics_device"))

    def _iteration_body(self):
        """Everything an iteration launches, in order, with no host read-back (capturable)."""
        self._launch_steps(0, self.episode_length, None)
        self.compute_returns()
        self.trainer.train_async(self.buffer.data)
        A = self.envs.agent_num
        self._stats_dev[:6].copy_(self.trainer.train_info.double() / float(self.trainer.ppo_epoch * self.trainer.num_mini_batch))
        self.envs.statistics_device(self.buffer, self._stats_dev[6:6 + A + 4])
        self.buffer.after_update()

    def graph_iteration(self):
        """Replay (or, the first times, warm up / capture) the iteration graph.  The first two iterations run eagerly on a
        side stream (they are real training iterations), the third is captured and every iteration from then on is one
        graph launch.  The captured graph lives on the trainer (which, like the buffer, survives across
        `PPOAgent.train` calls), so a later call with the same trainer / buffer / env replays it without re-capturing."""
        st = getattr(self.trainer, "_iter_graph", None)
        if st is None or st["buffer"] is not self.buffer.data or st["envs"] is not self.envs:
            A = self.envs.agent_num
            st = dict(buffer=self.buffer.data, envs=self.envs, graph=None, warm=0, launches=0, rng_counter=self.rng_counter,
                      stats_dev=torch.zeros(6 + A + 4, dtype=torch.float64, device=self.device),
                      stats_host=torch.zeros(6 + A + 4, dtype=torch.float64, pin_memory=True))
            self.trainer._iter_graph = st
        self._stats_dev, self._stats_host = st["stats_dev"], st["stats_host"]
        self.rng_counter = st["rng_counter"]      # the captured launches read this device counter
        self.trainer.sync_lrs()
        if st["graph"] is None:
            if st["warm"] < 2:
                s = torch.cuda.Stream(device=self.device)
                s.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(s):
                    self._iteration_body()
                torch.cuda.current_stream().wait_stream(s)
                st["warm"] += 1
                return
            l0 = self.gpu_launches + self.trainer.gpu_launches
            g = torch.cuda.CUDAGraph()
            try:
                with torch.cuda.graph(g):
                    self._iteration_body()
            except Exception as e:  # noqa: BLE001  (e.g. a collective that cannot be captured): stay eager for good
                import warnings

                warnings.warn(f"openrl_b200: CUDA-graph capture of the iteration failed ({type(e).__name__}: {e}); running eagerly")
                self.cfg.use_cuda_graph = False
                self.trainer._iter_graph = None
                torch.cuda.synchronize()
                self._iteration_body()
                return
            st["launches"] = self.gpu_launches + self.trainer.gpu_launches - l0
            self.gpu_launches -= st["launches"]     # capture launched nothing
            st["graph"] = g
        self._graph = st["graph"]
        st["graph"].replay()
        self.gpu_launches += st["launches"]

    def _read_graph_stats(self):
        self._stats_host.copy_(self._stats_dev, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        self.d2h_bytes += self._stats_host.numel() * 8
        return self._stats_host.numpy().copy()

    def _inner_loop_graph(self):
        if self.use_linear_lr_decay:
            self.trainer.algo_module.lr_decay(self.episode, self.episodes)
        self.graph_iteration()
        T, N = self.episode_length, self.envs.parallel_env_num
        self.agent.num_time_steps += N * T
        self._selfplay_snapshot()
        self.total_num_steps = (self.episode + 1) * T * self.n_rollout_threads
        if self.episode % self.log_interval == 0 and self.logger is not None:
            vals = self._read_graph_stats()        # the only device -> host read of the iteration
            keys = ["value_loss", "critic_grad_norm", "policy_loss", "dist_entropy", "actor_grad_norm", "ratio"]
            train_infos = {k: float(v) for k, v in zip(keys, vals[:6])}
            if getattr(self.trainer, "peer", None) is not None and not (vals[:6] == vals[:6]).all():
                self.trainer.peer.check()
            if type(self.trainer).__name__ == "A2CAlgorithm":
                train_infos.pop("ratio", None)
            rollout_infos = self.envs.statistics_host(vals[6:], T * N) if self.envs.use_monitor else {}
            self.logger.log_info(rollout_infos, step=self.total_num_steps)
            self.logger.log_info(train_infos, step=self.total_num_steps)
        elif self.envs.use_monitor:
            self.envs._total_step += T * N
        return True

    def _inner_loop(self):
        if self._graph_ok():
            return self._inner_loop_graph()
        rollout_infos, cont = self.actor_rollout()
        if not cont:
            return False
        train_infos = self.learner_update()
        self.buffer.after_update()
        self._selfplay_snapshot()
        self.total_num_steps = (self.episode + 1) * self.episode_length * self.n_rollout_threads
        if self.episode % self.log_interval == 0 and self.logger is not None:
            self.logger.log_info(rollout_infos, step=self.total_num_steps)
            self.logger.log_info(train_infos, step=self.total_num_steps)
        return True

    def learner_update(self):
        if self.use_linear_lr_decay:
            self.trainer.algo_module.lr_decay(self.episode, self.episodes)
        self.compute_returns()
        self.trainer.prep_training()
        with self._phase("update"):
            return self.trainer.train(self.buffer.data)

    def device_iteration(self):
        """One collect + update iteration as pure device work (no host read-back, no logging):
        what bench.py times as `value`."""
        if self._graph_ok():
            self.graph_iteration()
            self.agent.num_time_steps += self.envs.parallel_env_num * self.episode_length
        else:
            self._rollout_launch()
            self.compute_returns()
            with self._phase("update"):
                self.trainer.train_async(self.buffer.data)
            with self._phase("after_update"):
                self.buffer.after_update()
        self._selfplay_snapshot()
        self.episode += 1

    class _Phase:
        def __init__(self, drv, name):
            self.drv, self.name = drv, name

        def __enter__(self):
            if self.drv.phase_events is not None:
                self.e0 = torch.cuda.Event(enable_timing=True)
                self.e0.record()

        def __exit__(self, *a):
            if self.drv.phase_events is not None:
                e1 = torch.cuda.Event(enable_timing=True)
                e1.record()
                self.drv.phase_events.append((self.name, self.e0, e1))

    def _phase(self, name):
        return OnPolicyDriver._Phase(self, name)

    # -- rollout -----------------------------------------------------------------------------
    def _rollout_args(self, t_begin, t_end, noise):
        d, env = self.buffer.data, self.envs
        pol = self.trainer.algo_module.models["policy"]
        a = lib.OrlRolloutArgs()
        a.env_kind, a.n_envs, a.n_agents = env.kind, env.parallel_env_num, env.agent_num
        a.episode_length, a.t_begin, a.t_end = self.episode_length, t_begin, t_end
        separate_critic = d.critic_obs is not d.policy_obs
        a.obs_dim, a.critic_obs_dim, a.n_actions = d.obs_dim, (d.critic_obs_dim if separate_critic else 0), d.n_actions
        a.activation_id, a.deterministic = pol.activation_id, 0
        a.head_kind = pol.head_kind
        a.env_table_len = env.env_table_len
        a.policy_params = lib.ptr(pol.flat_params)
        a.policy_obs, a.critic_obs = lib.ptr(d.policy_obs), (lib.ptr(d.critic_obs) if separate_critic else None)
        a.actions, a.action_log_probs, a.rewards = lib.ptr(d.actions), lib.ptr(d.action_log_probs), lib.ptr(d.rewards)
        a.masks, a.active_masks = lib.ptr(d.masks), lib.ptr(d.active_masks)
        a.action_masks = None if d.action_masks_trivial else lib.ptr(d.action_masks)
        a.exp_noise = lib.ptr(noise)
        # one noise key for all ranks; a rank's rows are offset by its first GLOBAL row, so an env-sharded rollout draws
        # exactly the noise the unsharded rollout draws for the same envs
        # the env's own seed (what reset()/step() of the vec-env API use), so fused and per-call stepping agree
        a.rng_seed, a.rng_step_base, a.rng_counter = int(getattr(env, "rng_seed", self.cfg.seed)), 0, lib.ptr(self.rng_counter)
        a.rng_row_offset = int(getattr(env, "env_index_offset", 0)) * env.agent_num
        a.env_f64, a.env_u64, a.env_i32 = lib.ptr(env.env_f64), lib.ptr(env.env_u64), lib.ptr(env.env_i32)
        a.env_table = lib.ptr(env.env_table)
        a.ep_return, a.ep_length, a.episode_stats = lib.ptr(env.ep_return), lib.ptr(env.ep_length), lib.ptr(env.episode_stats)
        return a

    def _rnn_args(self, t_begin, t_end, noise):
        """OrlRnnArgs for the recurrent rollout / critic launches (update fields are filled by PPOAlgorithm)."""
        d, env = self.buffer.data, self.envs
        pol, cri = self.trainer.algo_module.models["policy"], self.trainer.algo_module.models["critic"]
        a = lib.OrlRnnArgs()
        a.env_kind, a.n_envs, a.n_agents = env.kind, env.parallel_env_num, env.agent_num
        a.episode_length, a.t_begin, a.t_end = self.episode_length, t_begin, t_end
        a.obs_dim, a.critic_obs_dim, a.n_actions = d.obs_dim, d.critic_obs_dim, d.n_actions
        a.activation_id, a.deterministic = pol.activation_id, 0
        a.env_table_len = env.env_table_len
        a.policy_params, a.critic_params = lib.ptr(pol.flat_params), lib.ptr(cri.flat_params)
        a.policy_obs, a.critic_obs = lib.ptr(d.policy_obs), lib.ptr(d.critic_obs)
        a.rnn_states, a.rnn_states_critic = lib.ptr(d.rnn_states), lib.ptr(d.rnn_states_critic)
        a.actions, a.action_log_probs, a.rewards = lib.ptr(d.actions), lib.ptr(d.action_log_probs), lib.ptr(d.rewards)
        a.masks, a.active_masks, a.value_preds = lib.ptr(d.masks), lib.ptr(d.active_masks), lib.ptr(d.value_preds)
        a.exp_noise = lib.ptr(noise)
        a.action_masks = None if d.action_masks_trivial else lib.ptr(d.action_masks)
        a.rng_seed, a.rng_step_base, a.rng_counter = int(self.cfg.seed) + 0x9E3779B9 * (self.rank + 1), 0, lib.ptr(self.rng_counter)
        state = lambda name: lib.ptr(getattr(env, name, None))   # a host-stepped env has no device state
        a.env_f64, a.env_u64, a.env_i32, a.env_table = state("env_f64"), state("env_u64"), state("env_i32"), state("env_table")
        a.ep_return, a.ep_length, a.episode_stats = state("ep_return"), state("ep_length"), state("episode_stats")
        return a

    def _host_insert(self, staged, step, lo, hi, has_masks=False):
        """One host env.step of envs [lo, hi) into slot step + 1 (rewards: slot step): orl_host_insert_wide_obs, or for a GRU
        policy orl_host_insert_rnn_wide_obs, which also zeroes rnn_states[step + 1] of the envs that finished (the inserts
        that take every width the nets take: masks of 1..64 actions, critic sections of 1..256 features).  With `has_masks`
        the staged block carries the envs' action masks, written to action_masks[step + 1] (replay_data.py:282-283); the
        buffer's masks stop being trivial for good.  A buffer with its own critic_obs (Dict observations) takes the
        block's critic section into critic_obs[step + 1]."""
        d, A = self.buffer.data, self.envs.agent_num
        r0, r1 = lo * A, hi * A
        cri = None if d.critic_obs is d.policy_obs else d.critic_obs[step + 1].view(-1, d.critic_obs_dim)[r0:r1]
        args = (lib.ptr(staged), hi - lo, A, d.obs_dim, lib.ptr(d.policy_obs[step + 1].view(-1, d.obs_dim)[r0:r1]),
                lib.ptr(d.rewards[step].view(-1)[r0:r1]), lib.ptr(d.masks[step + 1].view(-1)[r0:r1]),
                lib.ptr(d.active_masks[step + 1].view(-1)[r0:r1]))
        am = None
        if has_masks:
            d.action_masks_trivial = False
            am = d.action_masks[step + 1].view(-1, d.n_actions)[r0:r1]
        tail = (lib.ptr(am), d.n_actions, lib.ptr(cri), d.critic_obs_dim, lib.current_stream())
        if self.recurrent:
            states = d.rnn_states[step + 1].view(d.n_rollout_threads * A, -1)[r0:r1]
            lib.check(self._lib.orl_host_insert_rnn_wide_obs(*args, lib.ptr(states), *tail), "orl_host_insert_rnn_wide_obs")
        else:
            lib.check(self._lib.orl_host_insert_wide_obs(*args, *tail), "orl_host_insert_wide_obs")
        self.gpu_launches += 1

    def _launch_steps(self, t_begin, t_end, noise):
        """Policy + env for steps [t_begin, t_end): feed-forward (orl_rollout) or recurrent (orl_rnn_rollout)."""
        s = lib.current_stream()
        if self.recurrent:
            lib.check(self._lib.orl_rnn_rollout(self._rnn_args(t_begin, t_end, noise), s), "orl_rnn_rollout")
            self.gpu_launches += 2
        elif self.envs.kind == lib.ENV_GRIDWORLD_2P:
            if getattr(self.trainer, "share", False) or noise is not None:
                raise NotImplementedError("the self-play rollout is built for the two-net MLP policy with device sampling")
            sp = self.envs.selfplay_args(self._rollout_args(t_begin, t_end, None))
            lib.check(self._lib.orl_selfplay_rollout(sp, s), "orl_selfplay_rollout")
            self.gpu_launches += 2
        elif getattr(self.trainer, "share", False):
            lib.check(self._lib.orl_share_rollout(self._rollout_args(t_begin, t_end, noise), s), "orl_share_rollout")
            self.gpu_launches += 2
        else:
            lib.check(self._lib.orl_rollout(self._rollout_args(t_begin, t_end, noise), s), "orl_rollout")
            self.gpu_launches += 2

    def _draw_noise(self):
        """(T, B, n) Exp(1) noise from the global CPU generator, one draw per step like the
        reference's `torch.multinomial` inside Categorical.sample()."""
        d = self.buffer.data
        B, n = d.n_rollout_threads * d.num_agents, d.n_actions
        host = torch.empty(self.episode_length, B, n, dtype=torch.float32, pin_memory=True)
        gaussian = lib.is_gaussian(self.trainer.algo_module.models["policy"].head_kind)
        for t in range(self.episode_length):
            if gaussian:
                host[t].normal_()       # Normal.sample() == torch.normal(mean, std) == N(0,1)*std + mean
            else:
                host[t].exponential_(1)
        self.h2d_bytes += host.numel() * 4
        return host.to(self.device, non_blocking=True)

    def _rollout_launch(self):
        noise = self._draw_noise() if self.cfg.parity_mode else None
        with self._phase("rollout"):
            self._launch_steps(0, self.episode_length, noise)
        self.agent.num_time_steps += self.envs.parallel_env_num * self.episode_length

    def actor_rollout(self):
        cb = self.callback
        if cb is not None:
            cb.on_rollout_start()
        self.trainer.prep_rollout()
        T, N = self.episode_length, self.envs.parallel_env_num
        per_step = cb is not None and getattr(cb, "needs_per_step", True)
        s = lib.current_stream()
        if self.envs.kind == lib.ENV_NONE:
            if not self._host_rollout(cb):
                return {}, False
        elif not per_step:
            self._rollout_launch()
        else:
            noise = self._draw_noise() if self.cfg.parity_mode else None
            d = self.buffer.data
            for step in range(T):
                self._launch_steps(step, step + 1, noise)
                self.agent.num_time_steps += N
                # materialise the reference's per-step locals for the callbacks (SURVEY.md §5.5)
                actions = d.actions[step].cpu().numpy()  # noqa: F841
                action_log_probs = d.action_log_probs[step].cpu().numpy()  # noqa: F841
                obs = d.policy_obs[step + 1].cpu().numpy()  # noqa: F841
                rewards = d.rewards[step].cpu().numpy()  # noqa: F841
                dones = d.masks[step + 1].cpu().numpy()[..., 0] == 0.0  # noqa: F841
                infos = [{} for _ in range(N)]  # noqa: F841
                cb.update_locals(locals())
                if cb.on_step() is False:
                    return {}, False
        batch_rew_infos = self.envs.batch_rewards(self.buffer)
        cont = True
        if cb is not None:
            cont = cb.on_rollout_end() is not False   # callbacks without per-step hooks stop training here
        if self.envs.use_monitor:
            info = self.envs.statistics(self.buffer)
            info.update(batch_rew_infos)
            return info, cont
        return batch_rew_infos, cont

    def _host_rollout(self, cb):
        """Per-step loop for host-stepped envs (onpolicy_driver.py:154-203): device act -> D2H actions -> host env.step
        -> one pinned H2D copy -> in-place insert with the reference's mask rules (add2buffer, onpolicy_driver.py:80-152).
        With `host_env_groups` (and no callback or parity noise) the envs run as two groups in ping-pong: while the host
        steps one group, the device inserts the other group's results and acts on them for the next step; a group's
        actions travel D2H asynchronously and are awaited (CUDA event) only when the host is ready to step that group."""
        d, env = self.buffer.data, self.envs
        T, N = self.episode_length, env.parallel_env_num
        grouped = getattr(env, "supports_groups", False) and cb is None and not self.cfg.parity_mode and bool(getattr(self.cfg, "host_env_groups", True))
        groups = env.group_bounds(2) if grouped else [(0, N)]
        with self._phase("rollout"):
            noise = self._host_noise()
            for lo, hi in groups:                       # prime: actions of step 0 for every group
                env.fetch_actions(lo, hi, self._act(0, lo, hi, noise))
            for step in range(T):
                for g, (lo, hi) in enumerate(groups):
                    staged, obs, rewards, dones, infos, has_masks = env.step_staged(lo, hi)
                    self._host_insert(staged, step, lo, hi, has_masks)
                    self.agent.num_time_steps += hi - lo
                    if cb is not None:
                        actions = d.actions[step].cpu().numpy()  # noqa: F841
                        cb.update_locals(locals())
                        if cb.on_step() is False:
                            self.host_act_steps += step + 1
                            return False
                    if step + 1 < T:
                        if g == 0:
                            noise = self._host_noise()
                        env.fetch_actions(lo, hi, self._act(step + 1, lo, hi, noise))
        self.host_act_steps += T
        return True

    def _host_noise(self):
        """cfg.parity_mode: one step's (B, n) noise from the global CPU generator, drawn as `_draw_noise` draws each step;
        else None (Philox on the device)."""
        if not self.cfg.parity_mode:
            return None
        d = self.buffer.data
        noise = torch.empty(d.n_rollout_threads * d.num_agents, d.n_actions, dtype=torch.float32)
        noise.normal_() if lib.is_gaussian(self.trainer.algo_module.models["policy"].head_kind) else noise.exponential_(1)
        self.h2d_bytes += noise.numel() * 4
        return noise.to(self.device)

    def _act(self, step, lo, hi, noise):
        """The policy act for envs [lo, hi) of slot `step` of a host-stepped rollout (PPOModule.act_rows): actions and
        log-probs of their rows and, for a GRU policy, their rnn_states[step + 1].  The noise of a row is keyed by
        (per-rank seed, host_act_steps + step, buffer row + env_index_offset * A).  Returns the actions of the rows."""
        d, A = self.buffer.data, self.envs.agent_num
        B, w = d.n_rollout_threads * A, d.actions.shape[-1]
        acts = d.actions[step].view(B, w)
        self.trainer.algo_module.act_rows(
            d.policy_obs[step].view(B, d.obs_dim), acts, d.action_log_probs[step].view(B, w), lo * A, hi * A,
            int(self.cfg.seed) + 0x9E3779B9 * (self.rank + 1), self.host_act_steps + step,
            rng_row_offset=int(getattr(self.envs, "env_index_offset", 0)) * A,
            action_masks=None if d.action_masks_trivial else d.action_masks[step].view(B, d.n_actions), noise=noise,
            masks=d.masks[step], rnn_states=d.rnn_states[step:step + 2] if self.recurrent else None)
        self.gpu_launches += 1
        return acts[lo * A:hi * A]

    @torch.no_grad()
    def compute_returns(self):
        """onpolicy_driver.py:206-233: critic values of every slot (incl. the bootstrap slot T) in
        one launch, then the GAE scan."""
        d = self.buffer.data
        cri = self.trainer.algo_module.models["critic"]
        rows = (self.episode_length + 1) * d.n_rollout_threads * d.num_agents
        if self.recurrent:
            # the recurrent critic replays slots 0..T in order (its hidden state is part of the path)
            with self._phase("critic"):
                lib.check(self._lib.orl_rnn_critic(self._rnn_args(0, self.episode_length, None), lib.current_stream()),
                          "orl_rnn_critic")
            with self._phase("gae"):
                self.buffer.compute_returns(None, self.trainer.algo_module.get_critic_value_normalizer())
            self.gpu_launches += 2
            return
        with self._phase("critic"):
            if getattr(self.trainer, "share", False):
                lib.check(self._lib.orl_share_values(lib.ptr(cri.flat_params), cri.obs_dim, cri.n_actions, cri.activation_id,
                                                     lib.ptr(d.critic_obs), lib.ptr(d.value_preds), rows, lib.current_stream()),
                          "orl_share_values")
            else:
                lib.check(self._lib.orl_critic_values(lib.ptr(cri.flat_params), cri.obs_dim, cri.activation_id,
                                                      lib.ptr(d.critic_obs), lib.ptr(d.value_preds), rows,
                                                      lib.current_stream()), "orl_critic_values")
        with self._phase("gae"):
            self.buffer.compute_returns(None, self.trainer.algo_module.get_critic_value_normalizer())
        self.gpu_launches += 2
