"""MPE simple_spread (3 agents, shared MLP actor-critic = MAPPO) on the device against the numpy
restatement and the reference trace (tests/golden/trace_mpe_mlp.npz: unmodified reference,
`--use_valuenorm true --use_adv_normalize true`, feed-forward policy)."""
import os

import numpy as np
import pytest

from conftest import GOLDEN

pytestmark = pytest.mark.gpu


def test_simple_spread_env_matches_oracle(cuda):
    from openrl_b200.envs.common import make
    from oracle.envs import SimpleSpreadVec

    N = 8
    env = make("simple_spread", env_num=N)
    ref = SimpleSpreadVec(N)
    assert env.agent_num == 3
    o1, _ = env.reset(seed=11)
    o2 = ref.reset(seed=11)
    np.testing.assert_array_equal(o1["policy"], o2["policy"].astype(np.float32))
    np.testing.assert_array_equal(o1["critic"], o2["critic"].astype(np.float32))
    rng = np.random.default_rng(0)
    for t in range(80):  # crosses three auto-resets (world_length 25)
        a = rng.integers(0, 5, size=(N, 3, 1))
        o1, r1, d1, _ = env.step(a)
        o2, r2, d2, _ = ref.step(a)
        np.testing.assert_allclose(o1["policy"], o2["policy"].astype(np.float32), rtol=0, atol=2e-6, err_msg=str(t))
        np.testing.assert_allclose(o1["critic"], o2["critic"].astype(np.float32), rtol=0, atol=2e-6)
        np.testing.assert_allclose(r1, r2.astype(np.float32), rtol=1e-6, atol=1e-5)
        assert np.array_equal(d1, d2)
        assert d1.all() == ((t + 1) % 25 == 0)


def test_mpe_mappo_train_matches_reference_trace(cuda):
    from openrl_b200.utils.logger import Logger
    from helpers import product

    d = np.load(os.path.join(GOLDEN, "trace_mpe_mlp.npz"), allow_pickle=True)
    iters, N = int(d["meta/iters"]), int(d["meta/env_num"])
    cfg, env, net, agent = product("simple_spread", N, str(d["meta/flags"]).split(), golden=d)
    logger = Logger(quiet=True)
    agent.train(total_time_steps=cfg.episode_length * N * iters, logger=logger)
    train_logs = [h[1] for h in logger.history if "value_loss" in h[1]]
    assert len(train_logs) == iters
    for it in range(iters):
        want = d[f"it{it}/updates"].mean(axis=0)
        for col, name in enumerate(["value_loss", "critic_grad_norm", "policy_loss", "dist_entropy", "actor_grad_norm", "ratio"]):
            np.testing.assert_allclose(train_logs[it][name], want[col], rtol=1e-4, atol=2e-6, err_msg=f"it{it} {name}")
    b = agent.driver.buffer.data
    last = iters - 1
    assert np.array_equal(b.actions.cpu().numpy(), d[f"it{last}/actions"])
    np.testing.assert_allclose(b.policy_obs.cpu().numpy()[1:], d[f"it{last}/policy_obs"][1:], rtol=0, atol=2e-6)
    np.testing.assert_allclose(b.critic_obs.cpu().numpy()[1:], d[f"it{last}/critic_obs"][1:], rtol=0, atol=2e-6)
    np.testing.assert_allclose(b.rewards.cpu().numpy(), d[f"it{last}/rewards"], rtol=1e-6, atol=1e-5)
    assert np.array_equal(b.masks.cpu().numpy(), d[f"it{last}/masks"])


def test_mpe_fast_mode_runs_at_scale(cuda):
    """BASELINE config 3 shape (2048 envs x 3 agents, T=25) in fast mode: finite losses, episodes finish."""
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.common import make
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.logger import Logger

    cfg = create_config_parser().parse_args(["--episode_length", "25", "--ppo_epoch", "2", "--lr", "7e-4", "--critic_lr", "7e-4",
                                             "--use_adv_normalize", "true", "--log_interval", "1"])
    cfg.quiet = True
    env = make("simple_spread", env_num=2048)
    agent = PPOAgent(PPONet(env, cfg=cfg, device="cuda:0"))
    logger = Logger(quiet=True)
    agent.train(total_time_steps=25 * 2048 * 3, logger=logger)
    logs = [h[1] for h in logger.history if "value_loss" in h[1]]
    assert len(logs) == 3 and all(np.isfinite(list(l.values())).all() for l in logs)
    roll = [h[1] for h in logger.history if "rollout_episode_reward" in h[1]]
    assert all(r["rollout_episode_reward"] < 0 for r in roll)
