"""Box action spaces of 9..64 dimensions (cfg.use_wide_gaussian_head) without a GPU: the oracle loop against traces of
the unmodified reference on the envs of tests/wide_gaussian_oracle.py (tests/golden/trace_wide_gaussian_{21,64}.npz,
tools/gen_golden_wide_gaussian.py) — actions and observations bit for bit, the update scalars and parameters at 1e-4;
which head kinds the networks take with and without the option; and the refusals of what keeps 8 dimensions (GRU
policies, use_share_model, JRPO), of every width above 64, and of ORL_HEAD_GAUSSIAN_WIDE on the entries that do not
build it (the tensor-core update, orl_share_*, the self-play rollout and the device envs)."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from helpers import trace_threads  # noqa: F401  (autouse fixture)
from oracle import loop
from wide_gaussian_oracle import TRACES, WideGaussianTrainer

OPT = ["--use_wide_gaussian_head", "true"]


@pytest.mark.parametrize("n", sorted(TRACES))
def test_wide_gaussian_oracle_reproduces_reference_trace(n):
    obs_dim = TRACES[n]
    d = np.load(os.path.join(GOLDEN, f"trace_wide_gaussian_{n}.npz"), allow_pickle=True)
    cfg = loop.cfg_from_flags(str(d["meta/flags"]))
    tr = WideGaussianTrainer(cfg, int(d["meta/env_num"]), obs_dim, n)
    params = lambda: {f"{mk}.{k}": v.detach().numpy() for mk, p in (("policy", tr.pol), ("critic", tr.cri))  # noqa: E731
                      for k, v in p.items()}
    assert d["init/policy.act.action_out.fc_mean.weight"].shape == (n, 64)
    assert d["init/policy.base.mlp.fc1.0.weight"].shape == (64, obs_dim)
    for k, v in params().items():
        np.testing.assert_allclose(v, d[f"init/{k}"], rtol=0, atol=1e-6, err_msg=k)
    last = int(d["meta/iters"]) - 1
    for it in range(int(d["meta/iters"])):
        tr.rollout()
        b = tr.buf
        assert b.actions.shape[-1] == n
        assert np.array_equal(b.actions, d[f"it{it}/actions"])
        assert np.array_equal(b.obs, d[f"it{it}/policy_obs"])
        assert np.array_equal(b.masks, d[f"it{it}/masks"])
        tr.compute_returns()
        np.testing.assert_allclose(b.action_log_probs, d[f"it{it}/action_log_probs"], rtol=0, atol=1e-5)
        np.testing.assert_allclose(b.value_preds, d[f"it{it}/value_preds"], rtol=0, atol=1e-5)
        updates, perms = tr.train()
        assert np.array_equal(perms, d[f"it{it}/perms"])
        np.testing.assert_allclose(updates, d[f"it{it}/updates"], rtol=1e-4, atol=1e-6)
        tr.after_update()
        if it == last:   # the traces keep the weights at init and after the last iteration
            for k, v in params().items():
                np.testing.assert_allclose(v, d[f"it{it}/params/{k}"], rtol=1e-4, atol=1e-6, err_msg=k)


def _cfg(flags):
    from openrl_b200.configs.config import create_config_parser

    return create_config_parser().parse_args(flags)


def _box(n):
    from openrl_b200 import spaces

    return spaces.Box(-1.0, 1.0, (n,), np.float32)


def test_head_kinds_with_and_without_the_option():
    """Without the option Box(9) keeps the refusal that names 8; with it Box(1..8) keeps ORL_HEAD_GAUSSIAN and
    Box(9..64) takes ORL_HEAD_GAUSSIAN_WIDE, whose parameter layout is ORL_HEAD_GAUSSIAN's."""
    from openrl_b200 import lib, spaces
    from openrl_b200.modules.networks.policy_network import PolicyNetwork

    obs = spaces.Box(0.0, 1.0, (27,), np.float32)
    assert _cfg([]).use_wide_gaussian_head is False
    with pytest.raises(NotImplementedError, match="width up to 8"):
        PolicyNetwork(_cfg([]), obs, _box(9))
    for n in (1, 8, 9, 21, 64):
        pol = PolicyNetwork(_cfg(OPT), obs, _box(n))
        assert pol.head_kind == (lib.HEAD_GAUSSIAN_WIDE if n > 8 else lib.HEAD_GAUSSIAN)
        assert lib.is_gaussian(pol.head_kind)
        assert pol.flat_params.numel() == 64 * 27 + 3 * 64 + 64 * 64 + 3 * 64 + n * 64 + 2 * n
    assert not lib.is_gaussian(lib.HEAD_CATEGORICAL)


@pytest.mark.parametrize("what", ["65", "gru", "share", "jrpo"])
def test_modules_refuse_what_keeps_the_limit(what):
    """Box(65) names 64 with the option; GRU policies, the shared policy-value network and JRPO refuse Box(9) with it."""
    from openrl_b200 import spaces
    from openrl_b200.modules.networks.policy_network import PolicyNetwork
    from openrl_b200.modules.networks.policy_value_network import PolicyValueNetwork

    obs = spaces.Box(0.0, 1.0, (9,), np.float32)
    if what == "65":
        with pytest.raises(NotImplementedError, match="up to 64"):
            PolicyNetwork(_cfg(OPT), obs, _box(65))
    elif what == "gru":
        with pytest.raises(NotImplementedError, match="Discrete action spaces"):
            PolicyNetwork(_cfg(OPT + ["--use_recurrent_policy", "true"]), obs, _box(9))
    elif what == "share":
        with pytest.raises(NotImplementedError, match="up to 8"):
            PolicyValueNetwork(_cfg(OPT + ["--use_share_model", "true"]), obs, _box(9))
    else:   # JRPO runs on the chunked recurrent update, whose policy has no DiagGaussian head
        with pytest.raises(NotImplementedError, match="Discrete action spaces"):
            PolicyNetwork(_cfg(OPT + ["--use_recurrent_policy", "true", "--use_joint_action_loss", "true"]), obs, _box(9))


def _ppo_args(lib, n, head_kind, flags=0):
    fake = 1 << 20   # never dereferenced: every refusal happens before a launch
    a = lib.OrlPpoArgs()
    a.obs_dim, a.critic_obs_dim, a.n_actions, a.activation_id, a.head_kind = 9, 9, n, 1, head_kind
    a.grid_per_net, a.batch_rows, a.row_begin, a.total_rows, a.flags = 1, 1024, 0, 1024, flags
    for name in ("policy_params", "critic_params", "partials", "folded", "grads", "policy_obs", "critic_obs", "actions",
                 "old_log_probs", "advantages", "value_preds", "returns", "active_masks", "gae_stats", "mb_stats",
                 "policy_adam_m", "policy_adam_v", "critic_adam_m", "critic_adam_v", "adam_steps", "lrs", "train_info"):
        setattr(a, name, fake)
    return a


def _rollout_args(lib, env_kind, n, head_kind):
    fake = 1 << 20
    r = lib.OrlRolloutArgs()
    r.env_kind, r.n_envs, r.n_agents, r.episode_length, r.t_end = env_kind, 4, 1, 1, 1
    r.obs_dim, r.n_actions, r.head_kind = 9, n, head_kind
    for name in ("policy_params", "policy_obs", "actions", "action_log_probs"):
        setattr(r, name, fake)
    return r


def test_cabi_refusals_of_the_wide_gaussian_kind(orl_lib):
    """ORL_HEAD_GAUSSIAN_WIDE is a bad argument (10001) before any launch on the tensor-core update, the orl_share_*
    entries, every device env and the self-play rollout, and at 65 dimensions everywhere; ORL_HEAD_GAUSSIAN keeps its
    refusal of 9 dimensions with the same message.  (The GRU entries take no head kind: their policies are
    Categorical.)"""
    from openrl_b200 import lib

    W, G = lib.HEAD_GAUSSIAN_WIDE, lib.HEAD_GAUSSIAN
    assert W == 2
    for n in (9, 4):
        assert orl_lib.orl_ppo_fwdbwd(_ppo_args(lib, n, W, lib.PPO_TENSORCORE), None) == 10001
        assert b"ORL_PPO_TENSORCORE" in orl_lib.orl_last_error()
    for fn in (orl_lib.orl_ppo_fwdbwd, orl_lib.orl_ppo_reduce, orl_lib.orl_ppo_apply):
        assert fn(_ppo_args(lib, 65, W), None) == 10001
        assert b"1..64" in orl_lib.orl_last_error()
        assert fn(_ppo_args(lib, 9, G), None) == 10001
        assert b"n_actions must be in 1..8 for Gaussian heads (1..64 for Categorical heads)" in orl_lib.orl_last_error()
    for fn in (orl_lib.orl_share_fwdbwd, orl_lib.orl_share_apply):
        assert fn(_ppo_args(lib, 4, W), None) == 10001
    assert orl_lib.orl_share_rollout(_rollout_args(lib, lib.ENV_NONE, 4, W), None) == 10001
    # device envs: CartPole / GridWorld / simple_spread with the wide kind
    for env, n in ((lib.ENV_CARTPOLE, 2), (lib.ENV_GRIDWORLD, 5), (lib.ENV_MPE_SPREAD, 5)):
        r = _rollout_args(lib, env, n, W)
        if env == lib.ENV_MPE_SPREAD:
            r.n_agents, r.obs_dim, r.critic_obs_dim = 3, 18, 54
        else:
            r.obs_dim = 4
        assert orl_lib.orl_rollout(r, None) == 10001
        assert b"host-stepped" in orl_lib.orl_last_error()
    assert orl_lib.orl_rollout(_rollout_args(lib, lib.ENV_NONE, 65, W), None) == 10001
    sp = lib.OrlSelfPlayArgs()
    sp.rollout = _rollout_args(lib, lib.ENV_GRIDWORLD_2P, 5, W)
    sp.rollout.obs_dim = 4
    sp.rollout.env_i32 = sp.pool_count = sp.pool_stats = 1 << 20
    sp.strategy = lib.SP_RANDOM
    assert orl_lib.orl_selfplay_rollout(sp, None) == 10001
    assert b"Categorical" in orl_lib.orl_last_error()
    fake = 1 << 20
    assert orl_lib.orl_policy_eval(fake, 9, 65, 1, W, fake, fake, None, fake, fake, 16, None) == 10001
    assert orl_lib.orl_policy_eval(fake, 9, 9, 1, G, fake, fake, None, fake, fake, 16, None) == 10001
    assert orl_lib.orl_policy_eval(fake, 9, 9, 1, 3, fake, fake, None, fake, fake, 16, None) == 10001
