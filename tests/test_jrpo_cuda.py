"""Joint-action PPO (JRPO, `--use_joint_action_loss true`) on the recurrent MAPPO update, on the device.

- The reference's simple_spread JRPO traces (tests/golden/trace_mpe_jrpo*.npz, the examples/mpe/mpe_jrpo.yaml flags),
  stage by stage at the bars of the other recurrent traces (test_gru_cuda.check_recurrent_trace).
- With one agent JRPO is the ordinary recurrent update: the CartPole GRU trace, recorded without the flag, with it.
- Simple_spread at 2048 envs x 3 agents, the reference's own MPE example flow, the multi-GPU bucket contract, and the
  configurations that stay unbuilt."""
import os

import numpy as np
import pytest

from conftest import GOLDEN

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("tag", ["mpe_jrpo", "mpe_jrpo_mb"])
def test_jrpo_matches_reference_trace(cuda, tag):
    from helpers import check_recurrent_trace

    check_recurrent_trace(tag, "simple_spread")


def test_jrpo_single_agent_reproduces_cartpole_gru_trace(cuda, tmp_path):
    from helpers import check_recurrent_trace

    with np.load(os.path.join(GOLDEN, "trace_cartpole_gru.npz"), allow_pickle=True) as d:
        rec = {k: d[k] for k in d.files}
    rec["meta/flags"] = np.array(str(rec["meta/flags"]) + " --use_joint_action_loss true")
    np.savez(tmp_path / "trace_cartpole_gru.npz", **rec)
    check_recurrent_trace("cartpole_gru", "CartPole-v1", golden_dir=str(tmp_path))


def _mpe_jrpo_cfg(extra=()):
    from openrl_b200.configs.config import create_config_parser

    cfg = create_config_parser().parse_args(["--episode_length", "25", "--lr", "7e-4", "--critic_lr", "7e-4", "--ppo_epoch", "2",
                                             "--use_recurrent_policy", "true", "--use_joint_action_loss", "true",
                                             "--use_valuenorm", "true", "--use_adv_normalize", "true", "--log_interval", "1",
                                             *extra])
    cfg.quiet = True
    return cfg


def test_jrpo_runs_at_c3_scale(cuda):
    """simple_spread JRPO, 2048 envs x 3 agents (the C3 shape with the mpe_jrpo.yaml flags)."""
    from openrl_b200.envs.common import make
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.logger import Logger

    env = make("simple_spread", env_num=2048)
    agent = PPOAgent(PPONet(env, cfg=_mpe_jrpo_cfg(), device="cuda:0"))
    logger = Logger(quiet=True)
    agent.train(total_time_steps=25 * 2048 * 2, logger=logger)
    assert agent.driver.trainer.joint_action
    logs = [h[1] for h in logger.history if "value_loss" in h[1]]
    assert len(logs) == 2 and all(np.isfinite(list(l.values())).all() for l in logs), logs
    assert abs(logs[0]["ratio"] - 1.0) < 1e-3 and logs[0]["dist_entropy"] > 1.5


def test_reference_mpe_example_flow_with_jrpo(cuda, tmp_path):
    """The reference's own MPE example test (tests/test_examples/test_train_mpe.py): simple_spread, 2 envs,
    episode_length 5, GRU + JRPO + ValueNorm + advantage normalisation; train, save, load, act greedily."""
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.common import make
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent

    cfg = create_config_parser().parse_args("--episode_length 5 --use_recurrent_policy true --use_joint_action_loss true"
                                            " --use_valuenorm true --use_adv_normalize true".split())
    cfg.quiet = True
    env = make("simple_spread", env_num=2, asynchronous=True)
    agent = PPOAgent(PPONet(env, cfg=cfg, device="cuda:0"))
    agent.train(total_time_steps=30)
    assert agent.driver.trainer.joint_action
    agent.save(tmp_path / "ppo_agent")
    agent.load(tmp_path / "ppo_agent")
    agent.set_env(env)
    obs, info = env.reset(seed=0)
    for _ in range(5):
        action, _ = agent.act(obs, deterministic=True)
        assert tuple(action.shape) == (2, 3, 1)
        obs, r, done, info = env.step(action)
        if np.any(done):
            break
    env.close()


def test_jrpo_sharded_buckets_sum_to_global_bucket(cuda):
    """Multi-GPU contract of the JRPO update on one GPU: two uneven halves of the v3 chunk list, processed with
    norm_rows = global (chunk, step) groups and the moments of the whole list, give gradient buckets whose SUM is the
    bucket of the whole list."""
    import torch

    from openrl_b200 import lib
    from openrl_b200.utils.logger import Logger
    from helpers import product

    d = np.load(os.path.join(GOLDEN, "trace_mpe_jrpo.npz"), allow_pickle=True)
    cfg, env, net, agent = product("simple_spread", int(d["meta/env_num"]), str(d["meta/flags"]).split(), golden=d)
    agent.train(total_time_steps=0, logger=Logger(quiet=True))
    drv = agent.driver
    drv.actor_rollout()
    drv.compute_returns()
    tr, b = drv.trainer, drv.buffer.data
    Lc, A = cfg.data_chunk_length, b.num_agents
    chunks = b.episode_length * b.n_rollout_threads // Lc
    ids = torch.randperm(chunks).cuda()
    tr.tape = torch.empty(int(tr._lib.orl_rnn_workspace_floats(chunks * Lc * A, tr.rnn_stride)), dtype=torch.float32, device="cuda")
    stats = tr._joint_mb_stats(b, ids).clone()

    def bucket(part, norm_rows):
        a = tr._rnn_args(b, part.contiguous(), stats)
        assert a.flags & lib.PPO_JOINT_ACTION
        a.norm_rows = norm_rows
        lib.check(tr._lib.orl_rnn_fwdbwd(a, lib.current_stream()), "orl_rnn_fwdbwd")
        return tr.rnn_bucket.clone()

    whole = bucket(ids, 0)
    parts = bucket(ids[:chunks // 3], chunks * Lc) + bucket(ids[chunks // 3:], chunks * Lc)
    np.testing.assert_allclose(parts.cpu().numpy(), whole.cpu().numpy(), rtol=2e-4, atol=2e-6)
    assert float(whole[:tr.rnn_stride].abs().max()) > 1e-3 and float(whole[tr.rnn_stride:2 * tr.rnn_stride].abs().max()) > 1e-3


def test_jrpo_limits_are_loud(cuda):
    """JRPO is built on the chunked recurrent generator only; the joint kernels take 3 agents."""
    import torch

    from openrl_b200 import lib
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.common import make
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.logger import Logger
    from helpers import product

    for flags in (["--use_joint_action_loss", "true"],
                  ["--use_joint_action_loss", "true", "--use_naive_recurrent_policy", "true", "--episode_length", "25"]):
        cfg = create_config_parser().parse_args(flags)
        cfg.quiet = True
        agent = PPOAgent(PPONet(make("simple_spread", env_num=2), cfg=cfg, device="cuda:0"))
        with pytest.raises(NotImplementedError, match="use_joint_action_loss"):
            agent.train(total_time_steps=25 * 2 * 2)
    # the kernel entry point refuses the flag with a number of agents it was not built for
    cfg, env, net, agent = product("CartPole-v1", 4, ["--use_recurrent_policy", "true", "--episode_length", "8"])
    agent.train(total_time_steps=0, logger=Logger(quiet=True))
    drv = agent.driver
    drv.actor_rollout()
    drv.compute_returns()
    tr, b = drv.trainer, drv.buffer.data
    ids = torch.arange(4, device="cuda")
    tr.tape = torch.empty(int(tr._lib.orl_rnn_workspace_floats(4 * cfg.data_chunk_length, tr.rnn_stride)), dtype=torch.float32,
                          device="cuda")
    a = tr._rnn_args(b, ids, b.gae_stats[5:8])
    a.flags |= lib.PPO_JOINT_ACTION
    assert tr._lib.orl_rnn_fwdbwd(a, lib.current_stream()) != 0
