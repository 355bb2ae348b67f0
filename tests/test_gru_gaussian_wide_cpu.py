"""GRU policies with DiagGaussian heads of 9..64 dimensions (cfg.use_wide_recurrent_gaussian_head) without a GPU: the
option's default, the head kinds and parameter counts (ending in logstd) it gives, the refusals that keep their limits,
the C-ABI refusals (bad argument, 10001, before any launch) and the tape widths of the wide head kind.  The refusals of
PPOAlgorithm (JRPO, use_share_model with a GRU) query the device first and are in tests/test_gru_gaussian_wide_cuda.py."""
import numpy as np
import pytest

REC = ["--use_recurrent_policy", "true", "--use_recurrent_gaussian_head", "true"]
OPT = REC + ["--use_wide_recurrent_gaussian_head", "true"]


def _cfg(flags):
    from openrl_b200.configs.config import create_config_parser

    return create_config_parser().parse_args(flags)


def _box(w):
    from openrl_b200 import spaces

    return spaces.Box(-1.0, 1.0, (w,), np.float32)


def test_option_default_and_head_kinds():
    from openrl_b200 import lib
    from openrl_b200.modules.networks.policy_network import PolicyNetwork

    assert _cfg([]).use_wide_recurrent_gaussian_head is False
    naive = ["--use_naive_recurrent_policy", "true", "--use_recurrent_gaussian_head", "true",
             "--use_wide_recurrent_gaussian_head", "true"]
    for flags in (OPT, naive):
        for n in (1, 8, 9, 21, 64):
            pol = PolicyNetwork(_cfg(flags), _box(18), _box(n))
            want = lib.HEAD_GAUSSIAN if n <= 8 else lib.HEAD_GAUSSIAN_WIDE
            assert pol.recurrent and pol.head_kind == want and pol.n_actions == n and lib.is_gaussian(pol.head_kind)
            rnn = 64 * 18 + 3 * 64 + 64 * 64 + 3 * 64 + 2 * 192 * 64 + 2 * 192 + 2 * 64
            assert pol.flat_params.numel() == rnn + n * 64 + n + n
            names = [k for k, _ in pol.named_parameters()]
            assert names[-3:] == ["act.action_out.fc_mean.weight", "act.action_out.fc_mean.bias", "act.action_out.logstd._bias"]
    # Box(1..8) keeps HEAD_GAUSSIAN with the option off as well
    assert PolicyNetwork(_cfg(REC), _box(18), _box(8)).head_kind == lib.HEAD_GAUSSIAN
    # 65 and beyond are refused, naming 64
    with pytest.raises(NotImplementedError, match="64"):
        PolicyNetwork(_cfg(OPT), _box(18), _box(65))
    # without use_recurrent_gaussian_head the option changes nothing: a GRU policy on a Box space is refused
    with pytest.raises(NotImplementedError, match="Discrete action spaces"):
        PolicyNetwork(_cfg(["--use_recurrent_policy", "true", "--use_wide_recurrent_gaussian_head", "true"]), _box(18), _box(21))
    # without the option Box(9+) keeps its limit of 8, and the message names the option
    with pytest.raises(NotImplementedError, match="up to 8.*use_wide_recurrent_gaussian_head"):
        PolicyNetwork(_cfg(REC + ["--use_wide_gaussian_head", "true", "--use_wide_recurrent_head", "true"]), _box(18), _box(9))
    # observations above 64 features take use_wide_recurrent_observations, as for the other heads
    with pytest.raises(NotImplementedError):
        PolicyNetwork(_cfg(OPT), _box(67), _box(21))
    pol = PolicyNetwork(_cfg(OPT + ["--use_wide_recurrent_observations", "true"]), _box(256), _box(64))
    assert pol.head_kind == lib.HEAD_GAUSSIAN_WIDE and pol.obs_dim == 256


def test_param_count_and_tape_widths(orl_lib):
    from openrl_b200 import lib

    for d, n in ((18, 9), (67, 21), (256, 64)):
        cat = orl_lib.orl_rnn_param_count(d, n)
        assert orl_lib.orl_rnn_param_count_head(d, n, lib.HEAD_GAUSSIAN_WIDE) == cat + n
    for rows in (1, 1023, 1024, 1025):
        for n, d, dc in ((9, 18, 54), (21, 67, 67), (64, 256, 256), (64, 9, 256), (30, 65, 9)):
            stride = 90000
            pol_w = 1872 + (256 if d > 64 else 0)         # dL/dmean at 1744, dL/dlogstd at 1808, then the X field
            cri_w = 1744 + (256 if dc > 64 else 0)
            panels = 64 * 256 if max(d, dc) > 64 else 0
            got = orl_lib.orl_rnn_workspace_floats_head(rows, stride, n, d, dc, lib.HEAD_GAUSSIAN_WIDE)
            assert got == rows * max(pol_w, cri_w) + -(-rows // 1024) * stride + panels


def _rnn_args(lib, n, **kw):
    fake = 1 << 20   # never dereferenced: every refusal happens before a launch
    a = lib.OrlRnnArgs()
    a.env_kind, a.n_envs, a.n_agents, a.episode_length = lib.ENV_NONE, 4, 1, 8
    a.obs_dim, a.critic_obs_dim, a.n_actions, a.activation_id = 9, 9, n, 1
    a.chunk_length, a.n_chunks, a.t_begin, a.t_end, a.row_begin, a.row_end = 2, 4, 0, 1, 0, 4
    a.grads_stride = 1 << 16
    a.head_kind = lib.HEAD_GAUSSIAN_WIDE
    for name in ("chunk_ids", "policy_params", "critic_params", "policy_obs", "critic_obs", "rnn_states", "rnn_states_critic",
                 "actions", "action_log_probs", "rewards", "masks", "active_masks", "value_preds", "returns", "advantages",
                 "gae_stats", "mb_stats", "tape", "grads", "loss_acc", "policy_adam_m", "policy_adam_v", "critic_adam_m",
                 "critic_adam_v", "adam_steps", "lrs", "train_info", "ep_return", "ep_length", "episode_stats"):
        setattr(a, name, fake)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def test_rnn_cabi_refusals_of_the_wide_gaussian_head(orl_lib):
    from openrl_b200 import lib

    for fn in (orl_lib.orl_rnn_act_rows, orl_lib.orl_rnn_fwdbwd, orl_lib.orl_rnn_critic, orl_lib.orl_rnn_apply):
        for n in (1, 5, 8):   # the wide kind is 9..64; 1..8 is ORL_HEAD_GAUSSIAN
            assert fn(_rnn_args(lib, n), None) == 10001
            assert b"head_kind" in orl_lib.orl_last_error()
        assert fn(_rnn_args(lib, 65), None) == 10001
        assert b"1..64" in orl_lib.orl_last_error()
        assert fn(_rnn_args(lib, 9, head_kind=lib.HEAD_GAUSSIAN), None) == 10001   # the 8-wide kind keeps its limit
        assert b"1..8" in orl_lib.orl_last_error()
        for hk in (-1, 3):
            assert fn(_rnn_args(lib, 21, head_kind=hk), None) == 10001
            assert b"head_kind" in orl_lib.orl_last_error()
    # the device envs are Discrete
    r = _rnn_args(lib, 21, env_kind=lib.ENV_CARTPOLE, obs_dim=4, critic_obs_dim=4, n_agents=1)
    assert orl_lib.orl_rnn_rollout(r, None) == 10001
    # JRPO is built for Discrete action spaces of up to 8 actions
    j = _rnn_args(lib, 21, n_agents=3, flags=lib.PPO_JOINT_ACTION)
    assert orl_lib.orl_rnn_fwdbwd(j, None) == 10001
    assert b"JOINT_ACTION" in orl_lib.orl_last_error()
    # a grads_stride that leaves out logstd
    s = _rnn_args(lib, 21, grads_stride=orl_lib.orl_rnn_param_count(9, 21))
    assert orl_lib.orl_rnn_fwdbwd(s, None) == 10001
    assert b"grads_stride" in orl_lib.orl_last_error()
