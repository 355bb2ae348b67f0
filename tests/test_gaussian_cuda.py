"""DiagGaussian head + host-stepped env path (BASELINE config 5 class: continuous actions, env.step on
the host) against the reference trace of IdentityEnvcontinuous (tests/golden/
trace_identity_continuous.npz) and at the HalfCheetah shape (obs 17, act 6, 1024 envs) on synthetic
host dynamics."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from helpers import SyntheticHost, make_agent
from openrl_b200.envs.vec_env import HostVecEnv

pytestmark = pytest.mark.gpu


class _IdentityHost:
    """Host vec-env with the reference's duck type, backed by the oracle's env restatement."""

    def __init__(self, n):
        from openrl_b200 import spaces
        from oracle.envs import IdentityContinuousVec

        self.inner = IdentityContinuousVec(n)
        self.parallel_env_num, self.agent_num = n, 1
        self.observation_space = spaces.Box(0, 2, (1,), np.float32)
        self.action_space = spaces.Box(0, 1, (1,), np.float32)

    def reset(self, seed=None):
        return self.inner.reset(seed=seed)

    def step(self, actions):
        o, r, d, _ = self.inner.step(actions)
        return o, r, d, [{} for _ in range(self.parallel_env_num)]


def test_gaussian_head_host_env_matches_reference_trace(cuda):
    from openrl_b200.utils.logger import Logger

    d = np.load(os.path.join(GOLDEN, "trace_identity_continuous.npz"), allow_pickle=True)
    iters, N = int(d["meta/iters"]), int(d["meta/env_num"])
    flags = str(d["meta/flags"]).split() + ["--parity_mode", "true", "--log_interval", "1"]
    env = HostVecEnv(_IdentityHost(N))
    cfg, net, agent = make_agent(env, flags, golden=d, start=False)
    # same parameter tree as the reference (incl. act.action_out.logstd._bias)
    keys = [k for k, _ in net.module.models["policy"].named_parameters()]
    assert keys[-3:] == ["act.action_out.fc_mean.weight", "act.action_out.fc_mean.bias", "act.action_out.logstd._bias"]
    logger = Logger(quiet=True)
    agent.train(total_time_steps=cfg.episode_length * N * iters, logger=logger)
    logs = [h[1] for h in logger.history if "value_loss" in h[1]]
    assert len(logs) == iters
    for it in range(iters):
        want = d[f"it{it}/updates"].mean(axis=0)
        for col, name in enumerate(["value_loss", "critic_grad_norm", "policy_loss", "dist_entropy", "actor_grad_norm", "ratio"]):
            np.testing.assert_allclose(logs[it][name], want[col], rtol=2e-4, atol=5e-6, err_msg=f"it{it} {name}")
    b = agent.driver.buffer.data
    last = iters - 1
    np.testing.assert_allclose(b.actions.cpu().numpy(), d[f"it{last}/actions"], rtol=1e-5, atol=1e-6)
    np.testing.assert_array_equal(b.policy_obs.cpu().numpy()[1:], d[f"it{last}/policy_obs"][1:])
    np.testing.assert_allclose(b.rewards.cpu().numpy(), d[f"it{last}/rewards"], rtol=1e-5, atol=1e-6)
    np.testing.assert_array_equal(b.masks.cpu().numpy(), d[f"it{last}/masks"])
    for k, v in net.module.models["policy"].state_dict().items():
        gk = f"it{last}/params/policy.{k}"
        np.testing.assert_allclose(v.cpu().numpy(), d[gk], rtol=2e-3, atol=5e-6, err_msg=gk)


def test_config5_shape_runs(cuda):
    """HalfCheetah-shaped workload: obs 17, Box(6), 1024 envs, host env.step, device act/GAE/update."""
    from openrl_b200.utils.logger import Logger

    flags = ["--seed", "1", "--episode_length", "16", "--ppo_epoch", "2", "--log_interval", "1"]
    env = HostVecEnv(SyntheticHost(1024))
    cfg, net, agent = make_agent(env, flags, start=False)
    logger = Logger(quiet=True)
    agent.train(total_time_steps=16 * 1024 * 2, logger=logger)
    logs = [h[1] for h in logger.history if "value_loss" in h[1]]
    assert len(logs) == 2 and all(np.isfinite(list(l.values())).all() for l in logs)
    assert 8.0 < logs[0]["dist_entropy"] < 9.0   # 6 * (0.5 + 0.5 log(2 pi)) = 8.51 at logstd = 0
    assert abs(logs[0]["ratio"] - 1.0) < 1e-3
    assert env.h2d_bytes > 0 and env.d2h_bytes > 0


@pytest.mark.parametrize("grouped", ["true", "false"])
def test_host_rollout_grouped_and_synchronous_fill_the_buffer_identically(cuda, grouped):
    """Host-stepped rollout through make(make_custom_envs=...): the two-group ping-pong ingest (double-buffered pinned
    staging, device work of one group overlapping host stepping of the other) and the synchronous loop must insert the
    same things: next observations, rewards (= the action taken), masks 0 exactly at episode ends, for EVERY env."""
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.common import make
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.logger import Logger
    from helpers import CountEnv

    T, N, H = 12, 10, 5
    cfg = create_config_parser().parse_args(["--seed", "0", "--episode_length", str(T), "--ppo_epoch", "1", "--host_env_groups", grouped,
                                             "--log_interval", "1"])
    cfg.quiet = True
    env = make("Count-v0", env_num=N, make_custom_envs=lambda id, env_num, render_mode=None, **kw: [(lambda i=i: CountEnv(i, horizon=H)) for i in range(env_num)])
    agent = PPOAgent(PPONet(env, cfg=cfg, device="cuda:0"))
    logger = Logger(quiet=True)
    agent.train(total_time_steps=T * N, logger=logger)
    b = agent.driver.buffer.data
    # after_update moved slot T to slot 0; slots 1..T still hold the rollout
    obs = b.policy_obs.cpu().numpy()[:, :, 0, :]          # (T+1, N, 2) = [t, id]
    acts = b.actions.cpu().numpy()[:, :, 0, 0]
    rew = b.rewards.cpu().numpy()[:, :, 0, 0]
    masks = b.masks.cpu().numpy()[:, :, 0, 0]
    for t in range(T):
        step_in_ep = (t + 1) % H
        assert (obs[t + 1, :, 1] == np.arange(N)).all()                          # every env (both groups) was inserted
        assert (obs[t + 1, :, 0] == (0 if step_in_ep == 0 else step_in_ep)).all()  # auto-reset observation at episode ends
        assert (masks[t + 1] == (0.0 if step_in_ep == 0 else 1.0)).all()
        assert (rew[t] == acts[t]).all()                                         # CountEnv rewards the action index
    assert set(np.unique(acts)) <= {0.0, 1.0, 2.0} and len(np.unique(acts)) > 1   # sampled integer actions reached the host envs
    for e in env.env.envs:
        assert len(e.actions) == T
    logs = [h[1] for h in logger.history if "value_loss" in h[1]]
    assert len(logs) == 1 and np.isfinite(list(logs[0].values())).all()
