"""GRU policies at head widths of 9..64 actions, without a GPU: the refusals of the recurrent C-ABI that keep a narrower
limit (65 actions anywhere, the device-env GRU rollout above 8 actions, JRPO above 8 actions, orl_host_insert_rnn's masks
above 8 actions, which orl_host_insert_rnn_wide takes up to 64), every one a bad argument (10001) before any launch;
orl_rnn_workspace_floats_for against orl_rnn_workspace_floats; and the opt-in cfg.use_wide_recurrent_head of the module."""
import numpy as np
import pytest


def _rnn_args(lib, n, **kw):
    fake = 1 << 20   # never dereferenced: every refusal happens before a launch
    a = lib.OrlRnnArgs()
    a.env_kind, a.n_envs, a.n_agents, a.episode_length = lib.ENV_NONE, 4, 1, 8
    a.obs_dim, a.critic_obs_dim, a.n_actions, a.activation_id = 9, 9, n, 1
    a.chunk_length, a.n_chunks, a.t_begin, a.t_end, a.row_begin, a.row_end = 2, 4, 0, 1, 0, 4
    a.grads_stride = 1 << 16
    for name in ("chunk_ids", "policy_params", "critic_params", "policy_obs", "critic_obs", "rnn_states", "rnn_states_critic",
                 "actions", "action_log_probs", "rewards", "masks", "active_masks", "value_preds", "returns", "advantages",
                 "gae_stats", "mb_stats", "tape", "grads", "loss_acc", "policy_adam_m", "policy_adam_v", "critic_adam_m",
                 "critic_adam_v", "adam_steps", "lrs", "train_info", "ep_return", "ep_length", "episode_stats"):
        setattr(a, name, fake)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def test_rnn_cabi_refuses_what_keeps_a_narrower_limit(orl_lib):
    from openrl_b200 import lib

    for fn in (orl_lib.orl_rnn_act_rows, orl_lib.orl_rnn_fwdbwd, orl_lib.orl_rnn_critic, orl_lib.orl_rnn_apply):
        assert fn(_rnn_args(lib, 65), None) == 10001
        assert b"1..64" in orl_lib.orl_last_error()
    # the device envs have at most 5 actions: their fused GRU rollout keeps the 8-wide head
    r = _rnn_args(lib, 9, env_kind=lib.ENV_CARTPOLE, obs_dim=4, critic_obs_dim=4)
    assert orl_lib.orl_rnn_rollout(r, None) == 10001
    assert b"1..8" in orl_lib.orl_last_error()
    # JRPO keeps the 8-wide head
    j = _rnn_args(lib, 9, n_agents=3, flags=lib.PPO_JOINT_ACTION)
    assert orl_lib.orl_rnn_fwdbwd(j, None) == 10001
    assert b"up to 8 actions" in orl_lib.orl_last_error()


def test_rnn_workspace_for_n_actions(orl_lib):
    """The per-width workspace is the old one for every n <= 8 and 64 floats more per tape row above."""
    w = orl_lib.orl_rnn_tape_width()
    for rows in (1, 1023, 1024, 1025, 3 * 1024 + 7):
        for stride in (57480, 61512):
            old = orl_lib.orl_rnn_workspace_floats(rows, stride)
            for n in range(1, 9):
                assert orl_lib.orl_rnn_workspace_floats_for(rows, stride, n) == old
            for n in (9, 17, 64):
                assert orl_lib.orl_rnn_workspace_floats_for(rows, stride, n) == old + 64 * rows
            assert old == rows * w + -(-rows // 1024) * stride


def test_gru_inserts_take_their_mask_widths(orl_lib):
    """orl_host_insert_rnn takes masks of up to 8 actions, orl_host_insert_rnn_wide up to 64: both refuse one more."""
    fake = 1 << 20
    args = lambda n: (fake, 4, 1, 9, fake, fake, fake, fake, fake, fake, n, None, 0, None)  # noqa: E731
    assert orl_lib.orl_host_insert_rnn(*args(9)) == 10001
    assert b"1..8" in orl_lib.orl_last_error()
    assert orl_lib.orl_host_insert_rnn_wide(*args(65)) == 10001
    assert b"1..64" in orl_lib.orl_last_error()


def _cfg(flags):
    from openrl_b200.configs.config import create_config_parser

    return create_config_parser().parse_args(flags)


def test_wide_gru_head_is_opt_in():
    """A GRU policy of 9..64 actions builds with use_wide_recurrent_head and refuses without it, naming the limit; 65
    actions refuse either way."""
    from openrl_b200 import spaces
    from openrl_b200.modules.networks.policy_network import PolicyNetwork

    obs = spaces.Box(0.0, 1.0, (9,), np.float32)
    gru = ["--use_recurrent_policy", "true"]
    assert not _cfg(gru).use_wide_recurrent_head
    for n in (1, 8):
        assert PolicyNetwork(_cfg(gru), obs, spaces.Discrete(n)).n_actions == n
    for n in (9, 33, 64):
        with pytest.raises(NotImplementedError, match="use_wide_recurrent_head"):
            PolicyNetwork(_cfg(gru), obs, spaces.Discrete(n))
        for flags in (gru, ["--use_naive_recurrent_policy", "true"]):
            net = PolicyNetwork(_cfg(flags + ["--use_wide_recurrent_head", "true"]), obs, spaces.Discrete(n))
            assert net.recurrent and net.n_actions == n
    with pytest.raises(NotImplementedError, match="up to 64 actions"):
        PolicyNetwork(_cfg(gru + ["--use_wide_recurrent_head", "true"]), obs, spaces.Discrete(65))
