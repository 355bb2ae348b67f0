"""Wide Discrete action spaces (9..64 actions) without a GPU: the oracle loop with the reference's mask ingest against
traces of the unmodified reference on the masked env widened to 9 and 64 actions (tests/golden/trace_wide_actions_*.npz,
tools/gen_golden_wide_actions.py); the C-ABI's refusals of heads it does not build; and the module refusals of the
policies that keep the 8-action limit."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from helpers import trace_threads  # noqa: F401  (autouse fixture)
from oracle import loop
from wide_actions_oracle import WIDTHS, WideMaskedTrainer


def _illegal(actions, action_masks):
    a = actions[..., 0].astype(np.int64)
    return int((np.take_along_axis(action_masks[:-1], a[..., None], axis=-1) == 0).sum())


@pytest.mark.parametrize("n", WIDTHS)
def test_wide_oracle_reproduces_reference_trace(n):
    d = np.load(os.path.join(GOLDEN, f"trace_wide_actions_{n}.npz"), allow_pickle=True)
    cfg = loop.cfg_from_flags(str(d["meta/flags"]))
    tr = WideMaskedTrainer(cfg, int(d["meta/env_num"]), n)
    params = lambda: {f"{mk}.{k}": v.detach().numpy() for mk, p in (("policy", tr.pol), ("critic", tr.cri))  # noqa: E731
                      for k, v in p.items()}
    assert d["init/policy.act.action_out.linear.weight"].shape == (n, 64)
    for k, v in params().items():
        np.testing.assert_allclose(v, d[f"init/{k}"], rtol=0, atol=1e-6, err_msg=k)
    for it in range(int(d["meta/iters"])):
        tr.rollout()
        b = tr.buf
        am = d[f"it{it}/action_masks"]
        assert am.shape[-1] == n
        assert np.array_equal(b.actions, d[f"it{it}/actions"])
        assert np.array_equal(b.obs, d[f"it{it}/policy_obs"])
        assert np.array_equal(b.masks, d[f"it{it}/masks"])
        assert np.array_equal(b.action_masks, am)
        assert (am == 0).any() and _illegal(b.actions, am) == 0
        if n > 8:   # actions beyond the 8 the narrow head holds were sampled
            assert b.actions.max() >= 8
        tr.compute_returns()
        np.testing.assert_allclose(b.value_preds, d[f"it{it}/value_preds"], rtol=0, atol=1e-5)
        updates, perms = tr.train()
        assert np.array_equal(perms, d[f"it{it}/perms"])
        np.testing.assert_allclose(updates, d[f"it{it}/updates"], rtol=1e-4, atol=1e-6)
        tr.after_update()
        for k, v in params().items():
            np.testing.assert_allclose(v, d[f"it{it}/params/{k}"], rtol=1e-4, atol=1e-6, err_msg=k)


def _ppo_args(lib, n, flags=0):
    fake = 1 << 20   # never dereferenced: every refusal happens before a launch
    a = lib.OrlPpoArgs()
    a.obs_dim, a.critic_obs_dim, a.n_actions, a.activation_id, a.head_kind = 9, 9, n, 1, lib.HEAD_CATEGORICAL
    a.grid_per_net, a.batch_rows, a.row_begin, a.total_rows, a.flags = 1, 1024, 0, 1024, flags
    for name in ("policy_params", "critic_params", "partials", "folded", "grads", "policy_obs", "critic_obs", "actions",
                 "old_log_probs", "advantages", "value_preds", "returns", "active_masks", "gae_stats", "mb_stats",
                 "policy_adam_m", "policy_adam_v", "critic_adam_m", "critic_adam_v", "adam_steps", "lrs", "train_info"):
        setattr(a, name, fake)
    return a


def test_cabi_refuses_heads_it_does_not_build(orl_lib):
    """65 actions, and 9 actions on the tensor-core update (its head is 8 wide), are bad arguments (10001) before
    any launch; so are 9-wide DiagGaussian heads and 9 actions on a device env."""
    from openrl_b200 import lib

    for fn in (orl_lib.orl_ppo_fwdbwd, orl_lib.orl_ppo_reduce, orl_lib.orl_ppo_apply):
        assert fn(_ppo_args(lib, 65), None) == 10001
        assert b"1..64" in orl_lib.orl_last_error()
    assert orl_lib.orl_ppo_fwdbwd(_ppo_args(lib, 9, lib.PPO_TENSORCORE), None) == 10001
    assert b"ORL_PPO_TENSORCORE" in orl_lib.orl_last_error()
    g = _ppo_args(lib, 9)
    g.head_kind = lib.HEAD_GAUSSIAN
    assert orl_lib.orl_ppo_fwdbwd(g, None) == 10001

    fake = 1 << 20
    r = lib.OrlRolloutArgs()
    r.env_kind, r.n_envs, r.n_agents, r.episode_length, r.t_end = lib.ENV_NONE, 4, 1, 1, 1
    r.obs_dim, r.n_actions, r.head_kind = 9, 65, lib.HEAD_CATEGORICAL
    for name in ("policy_params", "policy_obs", "actions", "action_log_probs"):
        setattr(r, name, fake)
    assert orl_lib.orl_rollout(r, None) == 10001
    r.n_actions, r.head_kind = 9, lib.HEAD_GAUSSIAN
    assert orl_lib.orl_rollout(r, None) == 10001
    r.head_kind, r.env_kind, r.n_agents, r.obs_dim, r.critic_obs_dim = lib.HEAD_CATEGORICAL, lib.ENV_MPE_SPREAD, 3, 18, 54
    assert orl_lib.orl_rollout(r, None) == 10001
    assert orl_lib.orl_policy_eval(fake, 9, 65, 1, lib.HEAD_CATEGORICAL, fake, fake, None, fake, fake, 16, None) == 10001
    assert orl_lib.orl_policy_eval(fake, 9, 9, 1, lib.HEAD_GAUSSIAN, fake, fake, None, fake, fake, 16, None) == 10001
    # the GRU insert keeps the 8-action limit
    assert orl_lib.orl_host_insert_rnn(fake, 4, 1, 9, fake, fake, fake, fake, fake, fake, 9, None, 0, None) == 10001


def _cfg(flags):
    from openrl_b200.configs.config import create_config_parser

    return create_config_parser().parse_args(flags)


@pytest.mark.parametrize("what", ["gru", "share", "gaussian", "65"])
def test_modules_refuse_what_keeps_the_8_action_limit(what):
    """A GRU policy, the shared policy-value network and a DiagGaussian head with 9 actions, and any policy with 65
    actions, raise NotImplementedError naming the limit; a feed-forward Categorical head of 9..64 actions builds."""
    from openrl_b200 import spaces
    from openrl_b200.modules.networks.policy_network import PolicyNetwork
    from openrl_b200.modules.networks.policy_value_network import PolicyValueNetwork

    obs = spaces.Box(0.0, 1.0, (9,), np.float32)
    for n in (9, 64):
        assert PolicyNetwork(_cfg([]), obs, spaces.Discrete(n)).n_actions == n
    if what == "gru":
        with pytest.raises(NotImplementedError, match="up to 8 actions"):
            PolicyNetwork(_cfg(["--use_recurrent_policy", "true"]), obs, spaces.Discrete(9))
    elif what == "share":
        with pytest.raises(NotImplementedError, match="up to 8"):
            PolicyValueNetwork(_cfg(["--use_share_model", "true"]), obs, spaces.Discrete(9))
    elif what == "gaussian":
        with pytest.raises(NotImplementedError, match="width up to 8"):
            PolicyNetwork(_cfg([]), obs, spaces.Box(-1.0, 1.0, (9,), np.float32))
    else:
        with pytest.raises(NotImplementedError, match="up to 64 actions"):
            PolicyNetwork(_cfg([]), obs, spaces.Discrete(65))
