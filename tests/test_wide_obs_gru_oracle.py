"""Observations of 65..256 features on GRU policies and critics (cfg.use_wide_recurrent_observations) without a GPU: the
recurrent oracle loop against traces of the unmodified reference on envs with wide observations
(tests/golden/trace_wide_obs_gru_{dict,box_256}.npz, tools/gen_golden_wide_obs_gru.py); the option is off by default;
which widths the networks take under each combination of the two wide-observation options; make() opening wide Dict
entries with either option; and the C-ABI refusals, with messages that name the limit, of every
width above 256 and of the paths that keep 64 (the device-env GRU rollout and JRPO)."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from helpers import trace_threads  # noqa: F401  (autouse fixture)
from oracle import loop

WIDE_FF = ["--use_wide_observations", "true"]
WIDE_GRU = ["--use_wide_recurrent_observations", "true"]
GRU = ["--use_recurrent_policy", "true"]


@pytest.mark.parametrize("tag", ["wide_obs_gru_dict", "wide_obs_gru_box_256"])
def test_oracle_reproduces_reference_trace(tag):
    """SMAC 8m's shapes with masks and a GRU (use_recurrent_policy), and Box(256) observations with
    use_naive_recurrent_policy: actions, observations and masks bit for bit, hidden states and values at 1e-5, the update
    scalars and the parameters after the last iteration (the traces keep no earlier ones) at 1e-4."""
    from wide_obs_gru_oracle import WideBoxGRUTrainer, WideDictGRUTrainer

    d = np.load(os.path.join(GOLDEN, f"trace_{tag}.npz"), allow_pickle=True)
    cfg = loop.cfg_from_flags(str(d["meta/flags"]))
    dict_obs = tag == "wide_obs_gru_dict"
    assert (cfg.use_recurrent_policy, cfg.use_naive_recurrent_policy) == ((True, False) if dict_obs else (False, True))
    tr = (WideDictGRUTrainer if dict_obs else WideBoxGRUTrainer)(cfg, int(d["meta/env_num"]))
    params = lambda: {f"{mk}.{k}": v.detach().numpy() for mk, p in (("policy", tr.pol), ("critic", tr.cri))  # noqa: E731
                      for k, v in p.items()}
    widths = (80, 168) if dict_obs else (256, 256)
    assert (d["init/policy.base.mlp.fc1.0.weight"].shape[1], d["init/critic.base.mlp.fc1.0.weight"].shape[1]) == widths
    for k, v in params().items():
        np.testing.assert_allclose(v, d[f"init/{k}"], rtol=0, atol=1e-6, err_msg=k)
    for it in range(int(d["meta/iters"])):
        tr.rollout()
        b = tr.buf
        assert np.array_equal(b.actions, d[f"it{it}/actions"])
        assert np.array_equal(b.policy_obs, d[f"it{it}/policy_obs"])
        assert np.array_equal(b.masks, d[f"it{it}/masks"])
        assert (b.masks[1:] == 0).any()   # episodes ended inside the rollout, so hidden states were reset mid-chunk
        if dict_obs:
            am = d[f"it{it}/action_masks"]
            assert np.array_equal(b.critic_obs, d[f"it{it}/critic_obs"])
            assert np.array_equal(b.action_masks, am) and (am == 0).any()
        np.testing.assert_allclose(b.rnn_states, d[f"it{it}/rnn_states"], rtol=0, atol=1e-5)
        tr.compute_returns()
        np.testing.assert_allclose(b.value_preds, d[f"it{it}/value_preds"], rtol=0, atol=1e-5)
        updates, perms = tr.train()
        assert np.array_equal(perms, d[f"it{it}/perms"])
        np.testing.assert_allclose(updates, d[f"it{it}/updates"], rtol=1e-4, atol=1e-6)
        tr.after_update()
        if it == int(d["meta/iters"]) - 1:
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
    assert _cfg([]).use_wide_recurrent_observations is False
    assert _cfg(WIDE_GRU).use_wide_recurrent_observations is True
    assert _cfg(WIDE_GRU).use_wide_observations is False and _cfg(WIDE_FF).use_wide_recurrent_observations is False


@pytest.mark.parametrize("recurrent", ["--use_recurrent_policy", "--use_naive_recurrent_policy"])
@pytest.mark.parametrize("options", [[], WIDE_FF, WIDE_GRU, WIDE_FF + WIDE_GRU], ids=["none", "ff", "gru", "both"])
def test_networks_check_the_option_of_their_kind(recurrent, options):
    """A GRU net takes 65..256 features only with use_wide_recurrent_observations, a feed-forward net only with
    use_wide_observations; 257 is refused everywhere, naming the bound."""
    from openrl_b200 import spaces
    from openrl_b200.modules.networks.policy_network import PolicyNetwork
    from openrl_b200.modules.networks.value_network import ValueNetwork

    gru_on, ff_on = WIDE_GRU[0] in options, WIDE_FF[0] in options
    for net_flags, on in (([recurrent, "true", "--use_wide_recurrent_head", "true"], gru_on), ([], ff_on)):
        cfg = _cfg(net_flags + options)
        builds = [lambda d: PolicyNetwork(cfg, _box(d), spaces.Discrete(14)),
                  lambda d: PolicyNetwork(cfg, _dict(d, 18), spaces.Discrete(64)),
                  lambda d: ValueNetwork(cfg, _dict(18, d)), lambda d: ValueNetwork(cfg, _box(d))]
        for build in builds:
            assert build(64).obs_dim == 64
            for d in (65, 80, 168, 256):
                if on:
                    net = build(d)
                    assert net.obs_dim == d and net.state_dict()["base.mlp.fc1.0.weight"].shape == (64, d)
                else:
                    with pytest.raises(NotImplementedError, match="64"):
                        build(d)
            with pytest.raises(NotImplementedError, match="256" if on else "64"):
                build(257)


def test_recurrent_refusal_names_the_option():
    from openrl_b200 import spaces
    from openrl_b200.modules.networks.policy_network import PolicyNetwork

    with pytest.raises(NotImplementedError, match="<= 256 only.*use_wide_recurrent_observations"):
        PolicyNetwork(_cfg(GRU + WIDE_GRU), _box(257), spaces.Discrete(5))


def test_shared_model_keeps_64():
    from openrl_b200 import spaces
    from openrl_b200.modules.networks.policy_value_network import PolicyValueNetwork

    with pytest.raises(NotImplementedError, match="64"):
        PolicyValueNetwork(_cfg(WIDE_GRU + ["--use_share_model", "true"]), _box(65), spaces.Discrete(5))
    with pytest.raises(NotImplementedError, match="use_share_model is not built"):
        PolicyValueNetwork(_cfg(GRU + WIDE_GRU + ["--use_share_model", "true"]), _box(65), spaces.Discrete(5))


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


@pytest.mark.parametrize("options", [WIDE_FF, WIDE_GRU, WIDE_FF + WIDE_GRU], ids=["ff", "gru", "both"])
def test_make_opens_wide_dict_entries_with_either_option(options):
    from openrl_b200.envs.common import make

    thunks = lambda id, env_num, render_mode=None, **kw: [_Wide8m for _ in range(env_num)]  # noqa: E731
    env = make("Wide8m", env_num=2, make_custom_envs=thunks, device="cpu", cfg=_cfg(GRU + options))
    assert (env.obs_dim, env.critic_obs_dim) == (80, 168)
    with pytest.raises(NotImplementedError, match="width 80"):
        make("Wide8m", env_num=2, make_custom_envs=thunks, device="cpu", cfg=_cfg(GRU))


def _rnn_args(lib, d, dc, **kw):
    fake = 1 << 20   # never dereferenced: every refusal happens before a launch
    a = lib.OrlRnnArgs()
    a.env_kind, a.n_envs, a.n_agents, a.episode_length = lib.ENV_NONE, 4, 1, 8
    a.obs_dim, a.critic_obs_dim, a.n_actions, a.activation_id = d, dc, 5, 1
    a.chunk_length, a.n_chunks, a.t_begin, a.t_end, a.row_begin, a.row_end = 2, 4, 0, 1, 0, 4
    a.grads_stride = 1 << 18
    for name in ("chunk_ids", "policy_params", "critic_params", "policy_obs", "critic_obs", "rnn_states", "rnn_states_critic",
                 "actions", "action_log_probs", "rewards", "masks", "active_masks", "value_preds", "returns", "advantages",
                 "gae_stats", "mb_stats", "tape", "grads", "loss_acc", "policy_adam_m", "policy_adam_v", "critic_adam_m",
                 "critic_adam_v", "adam_steps", "lrs", "train_info", "ep_return", "ep_length", "episode_stats"):
        setattr(a, name, fake)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def test_rnn_cabi_refuses_widths_it_does_not_build(orl_lib):
    """257 on every host-stepped orl_rnn_* entry, 65 on the device-env rollout and on JRPO: ORL_ERR_BAD_ARG (10001)
    before any launch, with a message naming the limit."""
    from openrl_b200 import lib

    for fn in (orl_lib.orl_rnn_act_rows, orl_lib.orl_rnn_critic, orl_lib.orl_rnn_fwdbwd, orl_lib.orl_rnn_apply):
        for d, dc in ((257, 18), (18, 257), (0, 18)):
            assert fn(_rnn_args(lib, d, dc), None) == 10001
            assert b"1..256" in orl_lib.orl_last_error()
    for d, dc in ((65, 54), (18, 65)):
        a = _rnn_args(lib, d, dc, env_kind=lib.ENV_MPE_SPREAD, n_envs=4, n_agents=3)
        assert orl_lib.orl_rnn_rollout(a, None) == 10001
        assert b"64" in orl_lib.orl_last_error()
        a = _rnn_args(lib, d, dc, n_agents=3, flags=lib.PPO_JOINT_ACTION)
        assert orl_lib.orl_rnn_fwdbwd(a, None) == 10001
        assert b"ORL_PPO_JOINT_ACTION" in orl_lib.orl_last_error() and b"1..64" in orl_lib.orl_last_error()


def test_workspace_entry_keeps_the_narrow_size(orl_lib):
    """orl_rnn_workspace_floats_wide_obs equals orl_rnn_workspace_floats_for at widths <= 64 and adds the X field and the
    dW1 panel buffer beyond."""
    tw = orl_lib.orl_rnn_tape_width()
    for n in (5, 64):
        assert orl_lib.orl_rnn_workspace_floats_wide_obs(3000, 40000, n, 64, 64) == orl_lib.orl_rnn_workspace_floats_for(3000, 40000, n)
    assert orl_lib.orl_rnn_workspace_floats_wide_obs(3000, 40000, 5, 80, 18) == 3000 * (tw + 256) + 3 * 40000 + 64 * 256
    assert orl_lib.orl_rnn_workspace_floats_wide_obs(3000, 40000, 64, 18, 168) == 3000 * (tw + 256) + 3 * 40000 + 64 * 256
    assert orl_lib.orl_rnn_workspace_floats_wide_obs(3000, 40000, 64, 80, 168) == 3000 * (tw + 320) + 3 * 40000 + 64 * 256
