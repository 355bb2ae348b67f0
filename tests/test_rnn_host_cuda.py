"""Recurrent (GRU) PPO / MAPPO on host-stepped envs (`HostVecEnv`, ORL_ENV_NONE): per step one `orl_rnn_act_rows` launch
between two host env.step calls, and `orl_host_insert_rnn`, which zeroes the hidden state of the envs that finished.

Bars: the reference's CartPole-GRU trace (tests/golden/trace_cartpole_gru.npz) reproduced with the numpy CartPole stepped
on the host, with the bars of `check_recurrent_trace`; the host-stepped rollout bit-identical to the device-env rollout of
the same seed, in both host loops, and parameters within 1e-6 after one update; on a multi-agent host env every recorded
hidden state within 2e-6 of the sequential core (orl_rnn_core.h compiled by g++) and exactly zero where the env finished."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from helpers import KEYS, gxx_shim, make_agent, ptr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return gxx_shim(tmp_path_factory, "rnn", "rnn_core_shim.cpp")


class _OracleHost:
    """Host vec-env with the reference's duck type over an oracle numpy vec-env.  `step_range` steps envs [lo, hi) only
    (what the two-group ping-pong loop asks for) through a shallow copy whose per-env state arrays are views."""

    def __init__(self, inner, n_actions, per_env_fields):
        from openrl_b200 import spaces

        self.inner, self.fields = inner, per_env_fields
        self.parallel_env_num, self.agent_num = inner.N, 1
        self.observation_space = spaces.Box(-np.inf, np.inf, (inner.obs_dim,), np.float32)
        self.action_space = spaces.Discrete(n_actions)

    def reset(self, seed=None):
        return self.inner.reset(seed=seed)

    def step(self, actions):
        return self.step_range(0, self.parallel_env_num, actions)

    def step_range(self, lo, hi, actions):
        import copy

        sub = copy.copy(self.inner)
        sub.N = hi - lo
        for f in self.fields:
            setattr(sub, f, getattr(self.inner, f)[lo:hi])
        o, r, d, _ = sub.step(actions)
        return o, r, d, [{} for _ in range(hi - lo)]


def _cartpole_host(n):
    from oracle.envs import CartPoleVec

    return _OracleHost(CartPoleVec(n), 2, ("rng", "state", "elapsed"))


def _gridworld_table(n, k=64, seed=1):
    """Start cells near the goal (1, 1), so that random walks finish episodes inside the rollout."""
    rng = np.random.default_rng(seed)
    table = np.zeros((n, k, 2), np.int64)
    for i in range(n):
        for j in range(k):
            while True:
                p = rng.integers(0, 4, size=2)
                if not (p == 1).all():
                    table[i, j] = p
                    break
    return table


def _gridworld_host(n, table):
    """GridWorldVec with env i's k-th reset at table[i, k] (the device env's reset_table semantics)."""
    from oracle.envs import GridWorldVec

    class PerEnvTable(GridWorldVec):
        def __init__(self, n, table):
            super().__init__(n)
            self.table, self.count = table, np.zeros(n, np.int64)

        def _reset_one(self, i):
            self.steps[i] = 0
            self.pos[i] = self.table[i, self.count[i]]
            self.count[i] += 1

    return _OracleHost(PerEnvTable(n, table), 5, ("pos", "steps", "table", "count"))


class _SyntheticMultiAgent:
    """A agents per env, obs (N, A, d) ~ N(0, 1), Discrete(4); an env finishes (all agents done) with probability 0.15
    per step, and a single agent of a running env is done with probability 0.05 (active_masks)."""

    def __init__(self, n, agents, obs_dim=6, seed=0):
        from openrl_b200 import spaces

        self.parallel_env_num, self.agent_num, self.obs_dim = n, agents, obs_dim
        self.observation_space = spaces.Box(-np.inf, np.inf, (obs_dim,), np.float32)
        self.action_space = spaces.Discrete(4)
        self.rng = np.random.default_rng(seed)
        self.finished = [[] for _ in range(n)]   # per env, per step: every agent of the env done

    def reset(self, seed=None):
        if seed is not None:
            self.rng = np.random.default_rng(seed)
        return self.rng.standard_normal((self.parallel_env_num, self.agent_num, self.obs_dim)).astype(np.float32)

    def step(self, actions):
        return self._step(0, self.parallel_env_num, actions)

    def _step(self, lo, hi, actions):
        n, A = hi - lo, self.agent_num
        assert actions.shape == (n, A, 1) and set(np.unique(actions)) <= {0, 1, 2, 3}
        env_done = self.rng.random(n) < 0.15
        dones = np.repeat(env_done[:, None], A, axis=1) | (self.rng.random((n, A)) < 0.05)
        for i in range(n):
            self.finished[lo + i].append(bool(dones[i].all()))
        obs = self.rng.standard_normal((n, A, self.obs_dim)).astype(np.float32)
        return obs, self.rng.standard_normal((n, A, 1)), dones, [{} for _ in range(n)]

    def finished_table(self):
        """(steps, N) bool of the steps since the last call."""
        t = np.array(self.finished, dtype=bool).T
        self.finished = [[] for _ in range(self.parallel_env_num)]
        return t


class _SyntheticMultiAgentRanges(_SyntheticMultiAgent):
    """The same env, steppable by env range (the two-group ping-pong loop)."""

    def step_range(self, lo, hi, actions):
        return self._step(lo, hi, actions)


def test_host_recurrent_cartpole_matches_reference_trace(cuda):
    """The executed reference's CartPole GRU run (8 envs, T = 32, episodes ending inside chunks, L = 4, two minibatches)
    with the numpy CartPole stepped on the host in parity mode."""
    from openrl_b200.envs.vec_env import HostVecEnv

    d = np.load(os.path.join(GOLDEN, "trace_cartpole_gru.npz"), allow_pickle=True)
    iters, N = int(d["meta/iters"]), int(d["meta/env_num"])
    flags = str(d["meta/flags"]).split() + ["--parity_mode", "true", "--log_interval", "1"]
    env = HostVecEnv(_cartpole_host(N))
    cfg, net, agent = make_agent(env, flags, golden=d)
    drv = agent.driver
    assert drv.recurrent and env.kind == 0
    b = drv.buffer.data
    for it in range(iters):
        tag = f"it{it}"
        drv.episode = it
        drv.actor_rollout()
        assert np.array_equal(b.actions.cpu().numpy(), d[f"{tag}/actions"]), tag
        assert np.array_equal(b.masks.cpu().numpy(), d[f"{tag}/masks"]), tag
        np.testing.assert_allclose(b.action_log_probs.cpu().numpy(), d[f"{tag}/action_log_probs"], rtol=0, atol=2e-5)
        np.testing.assert_allclose(b.rnn_states.cpu().numpy(), d[f"{tag}/rnn_states"], rtol=0, atol=2e-5)
        np.testing.assert_allclose(b.policy_obs.cpu().numpy(), d[f"{tag}/policy_obs"], rtol=0, atol=2e-6)
        np.testing.assert_allclose(b.rewards.cpu().numpy(), d[f"{tag}/rewards"], rtol=1e-6, atol=1e-5)
        drv.compute_returns()   # the recurrent critic over slots 0..T reads the policy observation (critic_obs is policy_obs)
        assert b.critic_obs is b.policy_obs
        np.testing.assert_allclose(b.rnn_states_critic.cpu().numpy(), d[f"{tag}/rnn_states_critic"], rtol=0, atol=2e-5)
        np.testing.assert_allclose(b.value_preds.cpu().numpy()[:-1], d[f"{tag}/value_preds"][:-1], rtol=0, atol=2e-5)
        np.testing.assert_allclose(b.returns.cpu().numpy()[:-1], d[f"{tag}/returns"][:-1], rtol=1e-4, atol=2e-4)
        info = drv.trainer.train(b)
        want = d[f"{tag}/updates"].mean(axis=0)
        for col, name in enumerate(KEYS):
            np.testing.assert_allclose(info[name], want[col], rtol=2e-4, atol=1e-5, err_msg=f"{tag} {name}")
        for mk in ("policy", "critic"):
            for k, v in net.module.models[mk].state_dict().items():
                gk = f"{tag}/params/{mk}.{k}"
                if gk in d and "value_normalizer" not in k:
                    np.testing.assert_allclose(v.cpu().numpy(), d[gk], rtol=2e-3, atol=2e-5, err_msg=gk)
        b.after_update()
    assert (b.masks.cpu().numpy()[1:] == 0).any()    # episodes did end inside the rollout


@pytest.mark.parametrize("grouped", [False, True])
@pytest.mark.parametrize("env_id", ["CartPole-v1", "GridWorldEnv"])
def test_host_recurrent_rollout_is_bit_identical_to_device_rollout(cuda, env_id, grouped):
    """Philox sampling, 37 envs (two ragged groups), T = 25: the host-stepped recurrent rollout (the numpy env on the host,
    orl_rnn_act_rows + orl_host_insert_rnn) and the device-env recurrent rollout (orl_rnn_rollout) of the same seed write
    the same bits; one update from the two buffers gives the same parameters."""
    import torch

    from openrl_b200.envs.common import make
    from openrl_b200.envs.vec_env import HostVecEnv

    N, T = 37, 25
    flags = ["--seed", "5", "--use_recurrent_policy", "true", "--episode_length", str(T), "--data_chunk_length", "5",
             "--num_mini_batch", "2", "--ppo_epoch", "1", "--host_env_groups", "true" if grouped else "false", "--log_interval", "1"]
    if env_id == "GridWorldEnv":
        table = _gridworld_table(N)
        dev_env, host = make(env_id, env_num=N, reset_table=table), _gridworld_host(N, table)
    else:
        dev_env, host = make(env_id, env_num=N), _cartpole_host(N)
    host_env = HostVecEnv(host)
    assert host_env.supports_groups
    runs, init = [], None
    for env in (dev_env, host_env):
        cfg, net, agent = make_agent(env, flags, like=init)   # the host run starts from the device run's initial weights
        if init is None:
            init = {mk: {k: v.clone() for k, v in net.module.models[mk].state_dict().items()} for mk in ("policy", "critic")}
        drv = agent.driver
        drv.actor_rollout()
        torch.cuda.synchronize()
        b = drv.buffer.data
        bufs = {k: getattr(b, k).cpu().numpy().copy()
                for k in ("actions", "action_log_probs", "rnn_states", "policy_obs", "masks", "rewards")}
        drv.compute_returns()
        torch.manual_seed(7)   # the minibatch permutation
        drv.trainer.train(b)
        params = {mk: {k: v.cpu().numpy().copy() for k, v in net.module.models[mk].state_dict().items()} for mk in ("policy", "critic")}
        runs.append((bufs, params))
    (dev, p_dev), (hst, p_host) = runs
    for k in dev:
        assert np.array_equal(dev[k], hst[k]), k
    assert (dev["masks"][1:] == 0).any() and (dev["masks"][1:] == 1).any()   # episodes ended inside the rollout
    done = dev["masks"][1:, ..., 0] == 0
    assert (dev["rnn_states"][1:][done] == 0).all() and np.abs(dev["rnn_states"][1:][~done]).max() > 0
    for mk in p_dev:
        for k in p_dev[mk]:
            np.testing.assert_allclose(p_host[mk][k], p_dev[mk][k], rtol=0, atol=1e-6, err_msg=f"{mk}.{k}")
    assert any(not np.array_equal(p_dev["policy"][k], init["policy"][k].cpu().numpy()) for k in p_dev["policy"])


@pytest.mark.parametrize("grouped", [False, True])
@pytest.mark.parametrize("mode", ["use_recurrent_policy", "use_naive_recurrent_policy"])
def test_host_recurrent_multi_agent_states_match_sequential_core(cuda, shim, mode, grouped):  # noqa: F811
    """3 agents per env, ragged minibatches (chunked: 11*3*20/3 = 220 chunks in 3 minibatches; naive: 33 rows in 2), three
    iterations: every recorded rnn_states[t+1] is the sequential core's step from (obs[t], rnn_states[t], masks[t]),
    zero exactly where the env finished, and the metrics are finite."""
    import torch

    from openrl_b200.envs.vec_env import HostVecEnv

    N, A, T = 11, 3, 20
    chunk = ["--data_chunk_length", "3", "--num_mini_batch", "3"] if mode == "use_recurrent_policy" else ["--num_mini_batch", "2"]
    flags = ["--seed", "2", f"--{mode}", "true", "--episode_length", str(T), "--ppo_epoch", "2", "--use_valuenorm", "true",
             "--host_env_groups", "true" if grouped else "false"] + chunk
    host = (_SyntheticMultiAgentRanges if grouped else _SyntheticMultiAgent)(N, A)
    env = HostVecEnv(host)
    assert env.supports_groups == grouped
    cfg, net, agent = make_agent(env, flags)
    drv = agent.driver
    b = drv.buffer.data
    rows = N * A
    pol = net.module.models["policy"]
    for it in range(3):
        drv.episode = it
        host.finished_table()
        drv.actor_rollout()
        torch.cuda.synchronize()
        obs, hs, mk = b.policy_obs.view(T + 1, rows, -1), b.rnn_states.view(T + 1, rows, 1, 64), b.masks.view(T + 1, rows, 1)
        fin = np.repeat(host.finished_table(), A, axis=1)              # (T, rows)
        assert fin.shape == (T, rows) and fin.any()
        assert np.array_equal(mk[1:, :, 0].cpu().numpy() == 0, fin)
        P = pol.flat_params.cpu().numpy()
        for t in range(T):
            X, H0, m = (np.ascontiguousarray(v.cpu().numpy().reshape(rows, -1)) for v in (obs[t], hs[t], mk[t]))
            want, out = np.zeros((rows, 64), np.float32), np.zeros((rows, pol.n_actions), np.float32)
            shim.shim_forward_rows(ptr(P), pol.obs_dim, pol.n_actions, pol.activation_id, rows, ptr(X), ptr(H0), ptr(m),
                                   ptr(want), ptr(out))
            got = hs[t + 1].cpu().numpy().reshape(rows, 64)
            assert (got[fin[t]] == 0).all(), t
            np.testing.assert_allclose(got[~fin[t]], want[~fin[t]], rtol=0, atol=2e-6, err_msg=f"it{it} t{t}")
        drv.compute_returns()
        info = drv.trainer.train(b)
        assert np.isfinite([info[k] for k in KEYS if k in info]).all(), info
        b.after_update()


def test_make_custom_envs_trains_a_recurrent_policy(cuda):
    """make(id, make_custom_envs=...) -> SyncHostVecEnv behind HostVecEnv: PPOAgent.train runs with use_recurrent_policy."""
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.common import make
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.logger import Logger
    from helpers import CountEnv

    T, N = 16, 6
    for grouped in ("false", "true"):
        cfg = create_config_parser().parse_args(["--use_recurrent_policy", "true", "--episode_length", str(T), "--data_chunk_length", "4",
                                                 "--host_env_groups", grouped, "--log_interval", "1"])
        cfg.quiet = True
        env = make("CartPole-v1", env_num=N,
                   make_custom_envs=lambda id, env_num, render_mode=None, **kw: [(lambda i=i: CountEnv(i, horizon=5)) for i in range(env_num)])
        agent = PPOAgent(PPONet(env, cfg=cfg, device="cuda:0"))
        logger = Logger(quiet=True)
        agent.train(total_time_steps=T * N * 2, logger=logger)
        logs = [h[1] for h in logger.history if "value_loss" in h[1]]
        assert len(logs) == 2 and all(np.isfinite(list(l.values())).all() for l in logs), logs
        hs, mk = agent.driver.buffer.data.rnn_states.cpu().numpy(), agent.driver.buffer.data.masks.cpu().numpy()
        assert (hs[1:][mk[1:, ..., 0] == 0] == 0).all() and (mk[1:] == 0).any()


def test_host_recurrent_limits_are_loud(cuda):
    from openrl_b200 import lib, spaces
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.vec_env import HostVecEnv
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent

    for name in ("orl_rnn_act_rows", "orl_host_insert_rnn"):
        assert name in lib.declared_symbols() and hasattr(lib.load(), name)
    # JRPO: its kernels are built for simple_spread on the device (3 agents, agent-0 critic)
    cfg = create_config_parser().parse_args(["--use_recurrent_policy", "true", "--use_joint_action_loss", "true", "--episode_length", "8"])
    cfg.quiet = True
    with pytest.raises(NotImplementedError, match="JRPO"):
        PPOAgent(PPONet(HostVecEnv(_SyntheticMultiAgent(4, 3)), cfg=cfg, device="cuda:0")).train(total_time_steps=8 * 4)

    class BoxActions(_SyntheticMultiAgent):
        def __init__(self, n, agents, obs_dim=6):
            super().__init__(n, agents, obs_dim)
            self.action_space = spaces.Box(-1, 1, (2,), np.float32)

    cfg2 = create_config_parser().parse_args(["--use_recurrent_policy", "true", "--episode_length", "8"])
    cfg2.quiet = True
    with pytest.raises(NotImplementedError, match="Discrete"):
        PPOAgent(PPONet(HostVecEnv(BoxActions(4, 1)), cfg=cfg2, device="cuda:0")).train(total_time_steps=8 * 4)
    with pytest.raises(NotImplementedError, match="64"):
        PPOAgent(PPONet(HostVecEnv(_SyntheticMultiAgent(4, 1, obs_dim=65)), cfg=cfg2, device="cuda:0")).train(total_time_steps=8 * 4)
