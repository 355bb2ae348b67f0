"""Fused rollout kernel (orl_rollout) + critic pass (orl_critic_values) + env kernels through the
product API, against the oracle (oracle/loop.py) and the reference's golden traces.

Bars: bit-exact sampled actions, observations (CartPole float64 dynamics + numpy-compatible PCG64
resets), rewards and masks; log-probs / values within 1e-5 absolute (fp32 reassociation)."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from helpers import product

pytestmark = pytest.mark.gpu


def test_seeded_init_matches_reference(cuda):
    d = np.load(os.path.join(GOLDEN, "trace_cartpole.npz"), allow_pickle=True)
    cfg, env, net, agent = product("CartPole-v1", 8, str(d["meta/flags"]).split())
    for mk in ("policy", "critic"):
        for k, v in net.module.models[mk].state_dict().items():
            gk = f"init/{mk}.{k}"
            if gk in d:
                np.testing.assert_allclose(v.cpu().numpy(), d[gk], rtol=0, atol=2e-7, err_msg=gk)


@pytest.mark.parametrize("tag", ["cartpole", "cartpole_c1"])
def test_cartpole_rollout_matches_reference_trace(cuda, tag):
    """First rollout of the reference run: same seeds -> same trajectories."""
    import torch

    d = np.load(os.path.join(GOLDEN, f"trace_{tag}.npz"), allow_pickle=True)
    flags = str(d["meta/flags"]).split()
    cfg, env, net, agent = product("CartPole-v1", int(d["meta/env_num"]), flags, golden=d)
    from openrl_b200.algorithms.ppo import PPOAlgorithm
    from openrl_b200.buffers import NormalReplayBuffer
    from openrl_b200.drivers.onpolicy_driver import OnPolicyDriver

    trainer = PPOAlgorithm(cfg, net.module, agent_num=1, device=net.device)
    buf = NormalReplayBuffer(cfg, 1, env.observation_space, env.action_space, device=net.device)
    drv = OnPolicyDriver({"cfg": cfg, "num_agents": 1, "run_dir": None, "envs": env, "device": net.device}, trainer, buf,
                         agent, logger=None, callback=None)
    drv.reset_and_buffer_init()
    drv.actor_rollout()
    drv.compute_returns()
    torch.cuda.synchronize()
    b = buf.data
    g = lambda k: d[f"it0/{k}"]
    assert np.array_equal(b.actions.cpu().numpy(), g("actions"))
    assert np.array_equal(b.policy_obs.cpu().numpy(), g("policy_obs"))
    assert np.array_equal(b.rewards.cpu().numpy(), g("rewards"))
    assert np.array_equal(b.masks.cpu().numpy(), g("masks"))
    assert np.array_equal(b.active_masks.cpu().numpy(), g("active_masks"))
    np.testing.assert_allclose(b.action_log_probs.cpu().numpy(), g("action_log_probs"), rtol=0, atol=1e-5)
    np.testing.assert_allclose(b.value_preds.cpu().numpy(), g("value_preds"), rtol=0, atol=1e-5)
    np.testing.assert_allclose(b.returns.cpu().numpy()[:-1], g("returns")[:-1], rtol=1e-5, atol=1e-5)


def test_rollout_single_launch_equals_per_step_launches(cuda):
    """t-range semantics: one launch over [0,T) == T launches of one step (callback mode)."""
    import torch

    from openrl_b200 import lib

    outs = []
    for per_step in (False, True):
        cfg, env, net, agent = product("CartPole-v1", 64, ["--seed", "3", "--episode_length", "40"])
        from openrl_b200.algorithms.ppo import PPOAlgorithm
        from openrl_b200.buffers import NormalReplayBuffer
        from openrl_b200.drivers.onpolicy_driver import OnPolicyDriver

        trainer = PPOAlgorithm(cfg, net.module, agent_num=1, device=net.device)
        buf = NormalReplayBuffer(cfg, 1, env.observation_space, env.action_space, device=net.device)
        drv = OnPolicyDriver({"cfg": cfg, "num_agents": 1, "run_dir": None, "envs": env, "device": net.device}, trainer,
                             buf, agent)
        drv.reset_and_buffer_init()
        noise = drv._draw_noise()
        if per_step:
            for t in range(40):
                lib.check(drv._lib.orl_rollout(drv._rollout_args(t, t + 1, noise), lib.current_stream()), "rollout")
        else:
            lib.check(drv._lib.orl_rollout(drv._rollout_args(0, 40, noise), lib.current_stream()), "rollout")
        torch.cuda.synchronize()
        b = buf.data
        outs.append([x.cpu().numpy().copy() for x in (b.actions, b.policy_obs, b.rewards, b.masks, b.action_log_probs)])
    for x, y in zip(*outs):
        assert np.array_equal(x, y)


def test_cartpole_env_step_matches_oracle_env(cuda):
    """Env kernel alone (orl_env_step via DeviceVecEnv.step) vs the numpy restatement, random actions,
    long enough to see terminations, TimeLimit truncation never (500) but many auto-resets."""
    from openrl_b200.envs.common import make
    from oracle.envs import CartPoleVec

    N = 16
    env = make("CartPole-v1", env_num=N)
    ref = CartPoleVec(N)
    o1, _ = env.reset(seed=5)
    o2 = ref.reset(seed=5)
    assert np.array_equal(o1, o2)
    rng = np.random.default_rng(0)
    n_done = 0
    for t in range(300):
        a = rng.integers(0, 2, size=(N, 1, 1))
        o1, r1, d1, infos = env.step(a)
        o2, r2, d2, fin = ref.step(a)
        assert np.array_equal(o1, o2), t
        assert np.array_equal(d1, d2)
        assert np.array_equal(r1, r2)
        for i in range(N):
            if d2[i, 0]:
                n_done += 1
                assert np.array_equal(infos[i]["final_observation"][0], fin[i])
    assert n_done > 50


def test_cartpole_time_limit_truncation(cuda):
    """A policy that balances never exists here, so force it: alternate actions keep the pole up long
    enough on some envs?  Instead check the counter directly: elapsed resets on done and done fires at 500."""
    import torch

    from openrl_b200.envs.common import make

    env = make("CartPole-v1", env_num=4)
    env.reset(seed=0)
    env.env_i32[0].fill_(498)  # two steps before the limit
    a = np.zeros((4, 1, 1))
    _, _, d1, _ = env.step(a)
    assert not d1.any()
    _, _, d2, _ = env.step(1 - a)
    assert d2.all()  # truncated at 500 -> done (RemoveTruncated: done = terminated or truncated)
    assert (env.env_i32[0].cpu().numpy() == 0).all()


def test_gridworld_env_matches_oracle_with_reset_table(cuda):
    from openrl_b200.envs.common import make
    from oracle.envs import GridWorldVec

    N, K = 8, 64
    rng = np.random.default_rng(1)
    table = np.zeros((N, K, 2), np.int64)
    for i in range(N):
        for k in range(K):
            while True:
                p = rng.integers(0, 10, size=2)
                if not (p == 1).all():
                    table[i, k] = p
                    break

    class PerEnvTable(GridWorldVec):
        def __init__(self, n, table):
            super().__init__(n)
            self.table, self.count = table, np.zeros(n, np.int64)

        def _reset_one(self, i):
            self.steps[i] = 0
            self.pos[i] = self.table[i, self.count[i]]
            self.count[i] += 1

    env = make("GridWorldEnv", env_num=N, reset_table=table)
    ref = PerEnvTable(N, table)
    o1, _ = env.reset(seed=0)
    o2 = ref.reset()
    assert np.array_equal(o1, o2.astype(np.float32))
    for t in range(400):
        a = rng.integers(0, 5, size=(N, 1, 1))
        o1, r1, d1, _ = env.step(a)
        o2, r2, d2, _ = ref.step(a)
        assert np.array_equal(o1, o2.astype(np.float32)), t
        assert np.array_equal(r1, r2), t
        assert np.array_equal(d1, d2), t
