"""GRU policies with DiagGaussian heads (cfg.use_recurrent_gaussian_head) without a GPU: the option's default, the head
kind and parameter count (with logstd) it gives, the refusals that keep their limits, the C-ABI refusals (bad argument,
10001, before any launch) and the workspace entry of the head kind."""
import numpy as np
import pytest

OPT = ["--use_recurrent_policy", "true", "--use_recurrent_gaussian_head", "true"]


def _cfg(flags):
    from openrl_b200.configs.config import create_config_parser

    return create_config_parser().parse_args(flags)


def _box(w, lo=-1.0):
    from openrl_b200 import spaces

    return spaces.Box(lo, 1.0, (w,), np.float32)


def test_option_default_and_head_kinds():
    from openrl_b200 import lib
    from openrl_b200.modules.networks.policy_network import PolicyNetwork

    assert _cfg([]).use_recurrent_gaussian_head is False
    with pytest.raises(NotImplementedError, match="Discrete action spaces"):
        PolicyNetwork(_cfg(["--use_recurrent_policy", "true"]), _box(18), _box(5))
    with pytest.raises(NotImplementedError, match="up to 8"):
        PolicyNetwork(_cfg(OPT), _box(18), _box(9))
    with pytest.raises(NotImplementedError, match="up to 8"):   # the option does not lift the width with the wide-head options
        PolicyNetwork(_cfg(OPT + ["--use_wide_gaussian_head", "true", "--use_wide_recurrent_head", "true"]), _box(18), _box(9))
    for flags in (OPT, ["--use_naive_recurrent_policy", "true", "--use_recurrent_gaussian_head", "true"]):
        for d, n in ((18, 5), (1, 1), (64, 8)):
            pol = PolicyNetwork(_cfg(flags), _box(d), _box(n))
            assert pol.recurrent and pol.head_kind == lib.HEAD_GAUSSIAN and pol.n_actions == n
            rnn = 64 * d + 3 * 64 + 64 * 64 + 3 * 64 + 2 * 192 * 64 + 2 * 192 + 2 * 64
            assert pol.flat_params.numel() == rnn + n * 64 + n + n
            names = [k for k, _ in pol.named_parameters()]
            assert names[-3:] == ["act.action_out.fc_mean.weight", "act.action_out.fc_mean.bias", "act.action_out.logstd._bias"]
    # observations above 64 features take use_wide_recurrent_observations, as for Discrete heads
    with pytest.raises(NotImplementedError):
        PolicyNetwork(_cfg(OPT), _box(65), _box(5))
    pol = PolicyNetwork(_cfg(OPT + ["--use_wide_recurrent_observations", "true"]), _box(256), _box(8))
    assert pol.head_kind == lib.HEAD_GAUSSIAN


def test_param_count_and_workspace_of_the_head_kind(orl_lib):
    from openrl_b200 import lib

    for d, n in ((18, 5), (256, 8), (1, 1)):
        cat = orl_lib.orl_rnn_param_count(d, n)
        assert orl_lib.orl_rnn_param_count_head(d, n, lib.HEAD_CATEGORICAL) == cat
        assert orl_lib.orl_rnn_param_count_head(d, n, lib.HEAD_GAUSSIAN) == cat + n
    w = orl_lib.orl_rnn_tape_width()
    for rows in (1, 1023, 1024, 1025):
        for n, d, dc in ((5, 18, 54), (8, 256, 256), (3, 65, 9), (1, 9, 256)):
            stride = 70000
            old = orl_lib.orl_rnn_workspace_floats_wide_obs(rows, stride, n, d, dc)
            assert orl_lib.orl_rnn_workspace_floats_head(rows, stride, n, d, dc, lib.HEAD_CATEGORICAL) == old
            pol_w = w + 8 + (256 if d > 64 else 0)        # 1752 or 2008: dL/dlogstd before the X field
            cri_w = w + (256 if dc > 64 else 0)
            panels = 64 * 256 if max(d, dc) > 64 else 0
            got = orl_lib.orl_rnn_workspace_floats_head(rows, stride, n, d, dc, lib.HEAD_GAUSSIAN)
            assert got == rows * max(pol_w, cri_w) + -(-rows // 1024) * stride + panels


def _rnn_args(lib, n, **kw):
    fake = 1 << 20   # never dereferenced: every refusal happens before a launch
    a = lib.OrlRnnArgs()
    a.env_kind, a.n_envs, a.n_agents, a.episode_length = lib.ENV_NONE, 4, 1, 8
    a.obs_dim, a.critic_obs_dim, a.n_actions, a.activation_id = 9, 9, n, 1
    a.chunk_length, a.n_chunks, a.t_begin, a.t_end, a.row_begin, a.row_end = 2, 4, 0, 1, 0, 4
    a.grads_stride = 1 << 16
    a.head_kind = lib.HEAD_GAUSSIAN
    for name in ("chunk_ids", "policy_params", "critic_params", "policy_obs", "critic_obs", "rnn_states", "rnn_states_critic",
                 "actions", "action_log_probs", "rewards", "masks", "active_masks", "value_preds", "returns", "advantages",
                 "gae_stats", "mb_stats", "tape", "grads", "loss_acc", "policy_adam_m", "policy_adam_v", "critic_adam_m",
                 "critic_adam_v", "adam_steps", "lrs", "train_info", "ep_return", "ep_length", "episode_stats"):
        setattr(a, name, fake)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def test_rnn_cabi_refusals_of_the_gaussian_head(orl_lib):
    from openrl_b200 import lib

    entries = (orl_lib.orl_rnn_act_rows, orl_lib.orl_rnn_fwdbwd, orl_lib.orl_rnn_critic, orl_lib.orl_rnn_apply)
    for fn in entries:   # neither CATEGORICAL nor GAUSSIAN
        for hk in (lib.HEAD_GAUSSIAN_WIDE, -1, 3):
            assert fn(_rnn_args(lib, 5, head_kind=hk), None) == 10001
            assert b"head_kind" in orl_lib.orl_last_error()
        assert fn(_rnn_args(lib, 9), None) == 10001   # GAUSSIAN keeps 8 dimensions
        assert b"1..8" in orl_lib.orl_last_error()
    # the device envs are Discrete
    r = _rnn_args(lib, 2, env_kind=lib.ENV_CARTPOLE, obs_dim=4, critic_obs_dim=4, n_agents=1)
    assert orl_lib.orl_rnn_rollout(r, None) == 10001
    assert b"ORL_HEAD_CATEGORICAL" in orl_lib.orl_last_error()
    # JRPO is built for Discrete action spaces
    j = _rnn_args(lib, 5, n_agents=3, flags=lib.PPO_JOINT_ACTION)
    assert orl_lib.orl_rnn_fwdbwd(j, None) == 10001
    assert b"JOINT_ACTION" in orl_lib.orl_last_error()
    # a grads_stride that leaves out logstd
    s = _rnn_args(lib, 5, grads_stride=orl_lib.orl_rnn_param_count(9, 5))
    assert orl_lib.orl_rnn_fwdbwd(s, None) == 10001
    assert b"grads_stride" in orl_lib.orl_last_error()


def test_abi_field_appended():
    """head_kind follows action_masks, so every older field keeps its offset and a zeroed struct is Categorical."""
    from openrl_b200 import lib

    names = [f[0] for f in lib.OrlRnnArgs._fields_]
    assert names[-3:] == ["action_masks", "head_kind", "reserved3"]
    assert lib.OrlRnnArgs.head_kind.offset == lib.OrlRnnArgs.action_masks.offset + 8
    assert lib.OrlRnnArgs().head_kind == lib.HEAD_CATEGORICAL
