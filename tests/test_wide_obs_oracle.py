"""Observations of 65..256 features (cfg.use_wide_observations) without a GPU: the oracle loops against traces of the
unmodified reference on envs with wide observations (tests/golden/trace_wide_obs_{dict,box_256}.npz,
tools/gen_golden_wide_obs.py) — actions and observations bit for bit, the update scalars and parameters at 1e-4; which
widths the networks, the host vec-env and the C-ABI take with and without the option; and the refusals, with messages
that name the limit, of every path that keeps 64 features (GRU policies, use_share_model, the device envs, the
tensor-core update, orl_host_insert) and of every width above 256."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from helpers import trace_threads  # noqa: F401  (autouse fixture)
from oracle import loop

WIDE = ["--use_wide_observations", "true"]


@pytest.mark.parametrize("tag", ["wide_obs_dict", "wide_obs_box_256"])
def test_wide_obs_oracle_reproduces_reference_trace(tag):
    from wide_obs_oracle import WideBoxTrainer, WideDictObsTrainer

    d = np.load(os.path.join(GOLDEN, f"trace_{tag}.npz"), allow_pickle=True)
    cfg = loop.cfg_from_flags(str(d["meta/flags"]))
    dict_obs = tag == "wide_obs_dict"
    tr = (WideDictObsTrainer if dict_obs else WideBoxTrainer)(cfg, int(d["meta/env_num"]))
    params = lambda: {f"{mk}.{k}": v.detach().numpy() for mk, p in (("policy", tr.pol), ("critic", tr.cri))  # noqa: E731
                      for k, v in p.items()}
    for k, v in params().items():
        np.testing.assert_allclose(v, d[f"init/{k}"], rtol=0, atol=1e-6, err_msg=k)
    widths = (80, 168) if dict_obs else (256, 256)
    assert (tr.pol["base.mlp.fc1.0.weight"].shape[1], tr.cri["base.mlp.fc1.0.weight"].shape[1]) == widths
    for it in range(int(d["meta/iters"])):
        tr.rollout()
        b = tr.buf
        assert np.array_equal(b.actions, d[f"it{it}/actions"])
        assert np.array_equal(b.masks, d[f"it{it}/masks"])
        assert (b.masks[1:] == 0).any()                                   # episodes ended inside the rollout
        if dict_obs:
            assert np.array_equal(b.policy_obs, d[f"it{it}/policy_obs"])
            assert np.array_equal(b.critic_obs, d[f"it{it}/critic_obs"])
            assert np.array_equal(b.critic_obs[..., :80], b.policy_obs)  # the policy sees part of the critic's state
        else:
            assert np.array_equal(b.obs, d[f"it{it}/policy_obs"])
            assert b.actions.shape[-1] == 4
        tr.compute_returns()
        np.testing.assert_allclose(b.value_preds, d[f"it{it}/value_preds"], rtol=0, atol=1e-5)
        updates, perms = tr.train()
        assert np.array_equal(perms, d[f"it{it}/perms"])
        np.testing.assert_allclose(updates, d[f"it{it}/updates"], rtol=1e-4, atol=1e-6)
        tr.after_update()
        for k, v in params().items():
            np.testing.assert_allclose(v, d[f"it{it}/params/{k}"], rtol=1e-4, atol=1e-6, err_msg=k)


def _cfg(flags):
    from openrl_b200.configs.config import create_config_parser

    return create_config_parser().parse_args(flags)


def _box(w):
    from openrl_b200 import spaces

    return spaces.Box(-np.inf, np.inf, (w,), np.float32)


def _dict(d, dc):
    from openrl_b200 import spaces

    return spaces.Dict({"policy": _box(d), "critic": _box(dc)})


def test_option_is_off_by_default():
    assert _cfg([]).use_wide_observations is False and _cfg(WIDE).use_wide_observations is True


def test_networks_keep_64_without_the_option():
    from openrl_b200 import spaces
    from openrl_b200.modules.networks.policy_network import PolicyNetwork
    from openrl_b200.modules.networks.value_network import ValueNetwork

    assert PolicyNetwork(_cfg([]), _box(64), spaces.Discrete(5)).obs_dim == 64
    for build in (lambda: PolicyNetwork(_cfg([]), _box(65), spaces.Discrete(5)), lambda: ValueNetwork(_cfg([]), _box(65)),
                  lambda: ValueNetwork(_cfg([]), _dict(18, 65))):
        with pytest.raises(NotImplementedError, match="width <= 64 only.*use_wide_observations"):
            build()


@pytest.mark.parametrize("d", [65, 80, 168, 256])
def test_feed_forward_networks_take_up_to_256_with_the_option(d):
    """Policy and critic, a flat Box or a Dict entry, Categorical (14, 64 actions) and DiagGaussian (8) heads."""
    from openrl_b200 import spaces
    from openrl_b200.modules.networks.policy_network import PolicyNetwork
    from openrl_b200.modules.networks.value_network import ValueNetwork

    cfg = _cfg(WIDE)
    for act in (spaces.Discrete(14), spaces.Discrete(64), spaces.Box(-1.0, 1.0, (8,), np.float32)):
        pol = PolicyNetwork(cfg, _box(d), act)
        assert pol.obs_dim == d and pol.state_dict()["base.mlp.fc1.0.weight"].shape == (64, d)
    assert PolicyNetwork(cfg, _dict(d, 18), spaces.Discrete(14)).obs_dim == d
    assert ValueNetwork(cfg, _dict(18, d)).obs_dim == d
    assert ValueNetwork(cfg, _box(d)).obs_dim == d


def test_networks_refuse_257_and_the_paths_that_keep_64():
    from openrl_b200 import spaces
    from openrl_b200.modules.networks.policy_network import PolicyNetwork
    from openrl_b200.modules.networks.policy_value_network import PolicyValueNetwork
    from openrl_b200.modules.networks.value_network import ValueNetwork

    cfg = _cfg(WIDE)
    with pytest.raises(NotImplementedError, match="width <= 256 only"):
        PolicyNetwork(cfg, _box(257), spaces.Discrete(5))
    with pytest.raises(NotImplementedError, match="width <= 256 only"):
        ValueNetwork(cfg, _dict(18, 257))
    gru = _cfg(WIDE + ["--use_recurrent_policy", "true"])
    with pytest.raises(NotImplementedError, match="64"):
        PolicyNetwork(gru, _box(65), spaces.Discrete(5))
    with pytest.raises(NotImplementedError, match="64"):
        ValueNetwork(gru, _dict(18, 65))
    with pytest.raises(NotImplementedError, match="64"):
        PolicyValueNetwork(_cfg(WIDE + ["--use_share_model", "true"]), _box(65), spaces.Discrete(5))


def test_dict_obs_dims_with_and_without_the_option():
    from openrl_b200.envs.vec_env.host_venv import dict_obs_dims

    assert dict_obs_dims(_dict(80, 168), wide_observations=True) == (80, 168)
    assert dict_obs_dims(_dict(256, 1), wide_observations=True) == (256, 1)
    with pytest.raises(NotImplementedError, match="'critic' observation has width 65.*use_wide_observations"):
        dict_obs_dims(_dict(3, 65))
    with pytest.raises(NotImplementedError, match="'policy' observation has width 257.*1..256"):
        dict_obs_dims(_dict(257, 3), wide_observations=True)


class _Wide8m:
    """One SMAC-8m-shaped agent's spaces (Dict {"policy": 80, "critic": 168}, Discrete(14)) with a 4-tuple step."""

    def __init__(self):
        from openrl_b200 import spaces

        self.observation_space = _dict(80, 168)
        self.action_space = spaces.Discrete(14)

    def _obs(self):
        return {"policy": np.zeros(80, np.float32), "critic": np.zeros(168, np.float32)}

    def reset(self, seed=None, options=None):
        return self._obs(), {}

    def step(self, action):
        return self._obs(), 0.0, False, {}


def test_make_takes_the_option_from_cfg():
    """make() reads use_wide_observations from kwargs["cfg"], as the reference's make receives cfg, and still hands
    every keyword to make_custom_envs."""
    from openrl_b200.envs.common import make

    seen = []

    def thunks(id, env_num, render_mode=None, **kw):
        seen.append(kw)
        return [_Wide8m for _ in range(env_num)]

    env = make("Wide8m", env_num=2, make_custom_envs=thunks, device="cpu", cfg=_cfg(WIDE))
    assert (env.obs_dim, env.critic_obs_dim) == (80, 168)
    assert "cfg" in seen[0]
    with pytest.raises(NotImplementedError, match="width 80"):
        make("Wide8m", env_num=2, make_custom_envs=thunks, device="cpu", cfg=_cfg([]))
    with pytest.raises(NotImplementedError, match="width 80"):
        make("Wide8m", env_num=2, make_custom_envs=thunks, device="cpu")


def _ppo_args(lib, d, dc, flags=0):
    fake = 1 << 20   # never dereferenced: every refusal happens before a launch
    a = lib.OrlPpoArgs()
    a.obs_dim, a.critic_obs_dim, a.n_actions, a.activation_id, a.head_kind = d, dc, 5, 1, lib.HEAD_CATEGORICAL
    a.grid_per_net, a.batch_rows, a.row_begin, a.total_rows, a.flags = 1, 1024, 0, 1024, flags
    for name in ("policy_params", "critic_params", "partials", "folded", "grads", "policy_obs", "critic_obs", "actions",
                 "old_log_probs", "advantages", "value_preds", "returns", "active_masks", "gae_stats", "mb_stats",
                 "policy_adam_m", "policy_adam_v", "critic_adam_m", "critic_adam_v", "adam_steps", "lrs", "train_info"):
        setattr(a, name, fake)
    return a


def test_cabi_refuses_widths_it_does_not_build(orl_lib):
    """257 anywhere, 65 on the tensor-core update, on a device env's rollout and in orl_host_insert's critic section,
    257 in orl_host_insert_wide_obs: ORL_ERR_BAD_ARG (10001) before any launch, with a message naming the limit."""
    from openrl_b200 import lib

    fake = 1 << 20
    for fn in (orl_lib.orl_ppo_fwdbwd, orl_lib.orl_ppo_reduce, orl_lib.orl_ppo_apply):
        for d, dc in ((257, 18), (18, 257)):
            assert fn(_ppo_args(lib, d, dc), None) == 10001
            assert b"1..256" in orl_lib.orl_last_error()
    assert orl_lib.orl_ppo_fwdbwd(_ppo_args(lib, 65, 8, lib.PPO_TENSORCORE), None) == 10001
    assert b"ORL_PPO_TENSORCORE" in orl_lib.orl_last_error() and b"1..64" in orl_lib.orl_last_error()

    r = lib.OrlRolloutArgs()
    r.env_kind, r.n_envs, r.n_agents, r.episode_length, r.t_end = lib.ENV_NONE, 4, 1, 1, 1
    r.obs_dim, r.n_actions, r.head_kind = 257, 5, lib.HEAD_CATEGORICAL
    for name in ("policy_params", "policy_obs", "actions", "action_log_probs"):
        setattr(r, name, fake)
    assert orl_lib.orl_rollout(r, None) == 10001
    assert b"1..256" in orl_lib.orl_last_error()
    r.env_kind, r.n_agents, r.obs_dim, r.critic_obs_dim = lib.ENV_MPE_SPREAD, 3, 65, 54
    assert orl_lib.orl_rollout(r, None) == 10001
    assert b"1..64" in orl_lib.orl_last_error()

    assert orl_lib.orl_critic_values(fake, 257, 1, fake, fake, 16, None) == 10001
    assert b"1..256" in orl_lib.orl_last_error()
    assert orl_lib.orl_policy_eval(fake, 257, 5, 1, lib.HEAD_CATEGORICAL, fake, fake, None, fake, fake, 16, None) == 10001
    assert b"1..256" in orl_lib.orl_last_error()

    args = lambda dc: (fake, 4, 1, 9, fake, fake, fake, fake, None, 0, fake, dc, None)  # noqa: E731
    assert orl_lib.orl_host_insert(*args(65)) == 10001
    assert b"1..64" in orl_lib.orl_last_error() and b"orl_host_insert_wide_obs" in orl_lib.orl_last_error()
    for dc in (0, 257):
        assert orl_lib.orl_host_insert_wide_obs(*args(dc)) == 10001
        assert b"1..256" in orl_lib.orl_last_error()
    # the GRU entries keep 64
    assert orl_lib.orl_host_insert_rnn_wide(fake, 4, 1, 9, fake, fake, fake, fake, fake, None, 0, fake, 65, None) == 10001
