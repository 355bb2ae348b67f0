"""Recurrent (GRU) MAPPO on the device against the unmodified reference's trace
(tests/golden/trace_mpe_gru.npz: simple_spread, 4 envs x 3 agents, T=25, data_chunk_length 2,
`--use_recurrent_policy true --use_valuenorm true --use_adv_normalize true`) and against the torch
oracle (oracle/nets.py rnn_layer, pinned to the same trace by tests/test_oracle_loop.py).

Bars: actions / masks bit-exact; hidden states, values and log-probs within 2e-5 absolute (fp32 GRU
with device expf/tanhf); per-iteration losses within 2e-4 relative (float atomics in the tape
reductions make the summation order run-dependent); parameters after the update within 2e-3."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from helpers import check_recurrent_trace

pytestmark = pytest.mark.gpu


def _oracle_params(model):
    return {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}


def _compare_act(a_dev, lp_dev, a_ref, lp_ref, rows):
    """Actions must agree; the one tolerated exception is a single row whose argmax(p / q) is a near-tie, which a 1e-7
    difference between the device and the torch-CPU logits can flip (seen once in ~10 full-suite runs: the orthogonal
    init differs by 1 ulp with the BLAS thread count, so the draw is not the same on every box).  Log-probs are compared
    on the agreeing rows."""
    a_dev = np.asarray(a_dev).astype(np.int64).reshape(rows, -1)
    a_ref = np.asarray(a_ref).astype(np.int64).reshape(rows, -1)
    same = (a_dev == a_ref).all(axis=1)
    assert int(same.sum()) >= rows - 1, f"{rows - int(same.sum())} rows disagree"
    np.testing.assert_allclose(np.asarray(lp_dev).reshape(rows, -1)[same], np.asarray(lp_ref).reshape(rows, -1)[same], rtol=0, atol=2e-6)


def test_recurrent_act_matches_oracle(cuda):
    import torch

    from oracle import nets
    from helpers import product

    cfg, env, net, agent = product("simple_spread", 4, ["--use_recurrent_policy", "true"])
    pol = net.module.models["policy"]
    p = _oracle_params(pol)
    g = torch.Generator().manual_seed(3)
    rows = 37
    obs = torch.randn(rows, 18, generator=g)
    h = torch.randn(rows, 1, 64, generator=g) * 0.5
    masks = (torch.rand(rows, 1, generator=g) > 0.3).float()
    noise = torch.empty(rows, 5).exponential_(1, generator=g)
    for det in (False, True):
        a1, lp1, h1 = net.module.act(obs, h, masks, deterministic=det, exp_noise=noise)
        a2, lp2, h2 = nets.policy_act(p, cfg, obs, None, h, masks, deterministic=det, exp_noise=noise)
        _compare_act(a1.cpu().numpy(), lp1.cpu().numpy(), a2.numpy(), lp2.numpy(), rows)
        np.testing.assert_allclose(h1.cpu().numpy(), h2.numpy(), rtol=0, atol=2e-6)


def test_recurrent_mappo_matches_reference_trace(cuda):
    check_recurrent_trace("mpe_gru", "simple_spread")


def test_naive_recurrent_mpe_matches_reference_trace(cuda):
    """cfg.use_naive_recurrent_policy (whole-trajectory BPTT, naive_recurrent_generator replay_data.py:806-946: minibatches of
    (env, agent) rows, initial hidden state of slot 0) == the chunked path with chunk length = episode_length; the reference's
    simple_spread trace with two minibatches per epoch."""
    check_recurrent_trace("mpe_naive_gru", "simple_spread")


@pytest.mark.parametrize("env_id,chunk,mini", [("CartPole-v1", 4, 2), ("GridWorldEnv", 1, 1), ("simple_spread", 3, 4)])
def test_recurrent_training_runs_and_acts(cuda, env_id, chunk, mini):
    """Fast mode (device Philox), ragged minibatches (chunks that do not divide the buffer, several minibatches):
    finite metrics, hidden states reset with the episodes, and the greedy act() path carries its rnn state."""
    import torch

    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.common import make
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.logger import Logger

    cfg = create_config_parser().parse_args(["--use_recurrent_policy", "true", "--episode_length", "25", "--ppo_epoch", "2",
                                             "--data_chunk_length", str(chunk), "--num_mini_batch", str(mini),
                                             "--log_interval", "1"])
    cfg.quiet = True
    N = 7
    env = make(env_id, env_num=N)
    agent = PPOAgent(PPONet(env, cfg=cfg, device="cuda:0"))
    logger = Logger(quiet=True)
    agent.train(total_time_steps=25 * N * 3, logger=logger)
    logs = [h[1] for h in logger.history if "value_loss" in h[1]]
    assert len(logs) == 3 and all(np.isfinite(list(l.values())).all() for l in logs), logs
    b = agent.driver.buffer.data
    hs, mk = b.rnn_states.cpu().numpy(), b.masks.cpu().numpy()
    assert np.isfinite(hs).all() and np.abs(hs[1:]).max() > 0
    done_slots = mk[1:, ..., 0] == 0
    assert (hs[1:][done_slots] == 0).all()          # rnn_states[dones_env] = 0 (onpolicy_driver.py:262-269)
    obs, _ = env.reset(seed=5)
    agent.net.reset(env)
    a1, _ = agent.act(obs, deterministic=True)
    s1 = torch.as_tensor(agent.net.rnn_states_actor).clone()
    assert a1.shape == (N, env.agent_num, 1) and np.abs(s1.cpu().numpy()).max() > 0
    obs2, _, _, _ = env.step(a1)
    agent.act(obs2, deterministic=True, episode_starts=np.ones(N, dtype=np.float32))
    s_reset = torch.as_tensor(agent.net.rnn_states_actor).clone()
    agent.net.rnn_states_actor = s1 * 0
    agent.act(obs2, deterministic=True)
    np.testing.assert_array_equal(s_reset.cpu().numpy(), torch.as_tensor(agent.net.rnn_states_actor).cpu().numpy())


def test_mpe_gru_runs_at_baseline_scale(cuda):
    """BASELINE configs[2]: simple_spread MAPPO, 3 agents x 2048 envs, shared GRU actor-critic (examples/mpe/mpe_ppo.yaml)."""
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.common import make
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.logger import Logger

    cfg = create_config_parser().parse_args(["--episode_length", "25", "--lr", "7e-4", "--critic_lr", "7e-4", "--ppo_epoch", "2",
                                             "--use_recurrent_policy", "true", "--use_valuenorm", "true",
                                             "--use_adv_normalize", "true", "--log_interval", "1"])
    cfg.quiet = True
    env = make("simple_spread", env_num=2048)
    agent = PPOAgent(PPONet(env, cfg=cfg, device="cuda:0"))
    logger = Logger(quiet=True)
    agent.train(total_time_steps=25 * 2048 * 2, logger=logger)
    logs = [h[1] for h in logger.history if "value_loss" in h[1]]
    assert len(logs) == 2 and all(np.isfinite(list(l.values())).all() for l in logs), logs
    assert abs(logs[0]["ratio"] - 1.0) < 1e-3 and logs[0]["dist_entropy"] > 1.5
    roll = [h[1] for h in logger.history if "rollout_episode_reward" in h[1]]
    assert all(r["rollout_episode_reward"] < 0 for r in roll)


def test_recurrent_sharded_buckets_sum_to_global_bucket(cuda):
    """Multi-GPU contract of the recurrent update on one GPU: two halves of the chunk list processed with
    norm_rows = global row-steps give gradient buckets whose SUM is the bucket of the whole chunk list."""
    import torch

    from openrl_b200 import lib
    from openrl_b200.utils.logger import Logger
    from helpers import product

    d = np.load(os.path.join(GOLDEN, "trace_mpe_gru.npz"), allow_pickle=True)
    cfg, env, net, agent = product("simple_spread", int(d["meta/env_num"]), str(d["meta/flags"]).split(), golden=d)
    agent.train(total_time_steps=0, logger=Logger(quiet=True))
    drv = agent.driver
    drv.actor_rollout()
    drv.compute_returns()
    tr, b = drv.trainer, drv.buffer.data
    Lc = cfg.data_chunk_length
    chunks = b.episode_length * b.n_rollout_threads * b.num_agents // Lc
    ids = torch.randperm(chunks).cuda()
    tr.tape = torch.empty(int(tr._lib.orl_rnn_workspace_floats(chunks * Lc, tr.rnn_stride)), dtype=torch.float32, device="cuda")

    def bucket(part, norm_rows):
        a = tr._rnn_args(b, part.contiguous(), b.gae_stats[5:8])
        a.norm_rows = norm_rows
        lib.check(tr._lib.orl_rnn_fwdbwd(a, lib.current_stream()), "orl_rnn_fwdbwd")
        return tr.rnn_bucket.clone()

    whole = bucket(ids, 0)
    parts = bucket(ids[:chunks // 3], chunks * Lc) + bucket(ids[chunks // 3:], chunks * Lc)   # uneven split: odd chunk counts too
    np.testing.assert_allclose(parts.cpu().numpy(), whole.cpu().numpy(), rtol=2e-4, atol=2e-6)
    assert float(whole[:2 * tr.rnn_stride].abs().max()) > 1e-3


def test_recurrent_limits_are_loud(cuda):
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.common import make
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent

    cfg = create_config_parser().parse_args(["--use_recurrent_policy", "true", "--data_chunk_length", "100"])
    cfg.quiet = True
    agent = PPOAgent(PPONet(make("CartPole-v1", env_num=2), cfg=cfg, device="cuda:0"))
    with pytest.raises(NotImplementedError):
        agent.train(total_time_steps=400)
    # whole-trajectory BPTT is the chunked path with chunk = episode_length: the default episode_length (200) is beyond the 32-step limit
    cfg2 = create_config_parser().parse_args(["--use_naive_recurrent_policy", "true"])
    cfg2.quiet = True
    agent2 = PPOAgent(PPONet(make("CartPole-v1", env_num=2), cfg=cfg2, device="cuda:0"))
    with pytest.raises(NotImplementedError):
        agent2.train(total_time_steps=400)
    cfg3 = create_config_parser().parse_args(["--use_recurrent_policy", "true", "--rnn_type", "lstm"])
    with pytest.raises(NotImplementedError):
        PPONet(make("CartPole-v1", env_num=2), cfg=cfg3, device="cuda:0")
