"""The C-ABI library builds for sm_90a, loads, and exports every symbol the header declares
(no compute calls: this runs without a GPU)."""
import ctypes


def test_every_declared_symbol_is_exported(orl_lib):
    from openrl_b200 import lib

    names = lib.declared_symbols()
    assert "orl_gae" in names
    raw = ctypes.CDLL(lib.LIB_PATH)
    for n in names:
        assert hasattr(raw, n), n
    # and every bound signature is declared in the header
    for n in lib._SIGNATURES:
        assert n in names, n


def test_abi_version(orl_lib):
    assert orl_lib.orl_abi_version() == 1


def test_bad_arguments_are_reported_not_crashed(orl_lib):
    rc = orl_lib.orl_gae(None, None, None, None, None, None, None, None, None, None, 4, 4, 0.99, 0.95, 1, None)
    assert rc == 10001
    assert b"orl_gae" in orl_lib.orl_last_error()
    # the recurrent rollout steps device envs only; a policy-only step goes to orl_rnn_act_rows
    from openrl_b200 import lib

    a = lib.OrlRnnArgs()
    a.env_kind, a.n_envs, a.n_agents, a.episode_length, a.t_end = lib.ENV_NONE, 4, 1, 1, 1
    a.obs_dim, a.critic_obs_dim, a.n_actions = 4, 4, 2
    assert orl_lib.orl_rnn_rollout(a, None) == 10001
    assert b"orl_rnn_act_rows" in orl_lib.orl_last_error()
    # the single-agent device rollouts store each observation as one float4: an observation buffer 4 bytes off a 16-byte
    # boundary is rejected before anything is launched or dereferenced
    fake = 1 << 20   # never dereferenced
    buffers = ("policy_params", "policy_obs", "actions", "action_log_probs", "rewards", "masks", "active_masks", "env_f64",
               "env_u64", "env_i32", "ep_return", "ep_length", "episode_stats")

    def rollout_args(kind, n_actions, **misaligned):
        r = lib.OrlRolloutArgs()
        r.env_kind, r.n_envs, r.n_agents, r.episode_length, r.t_end = kind, 4, 1, 1, 1
        r.obs_dim, r.n_actions, r.head_kind = 4, n_actions, lib.HEAD_CATEGORICAL
        for name in buffers:
            setattr(r, name, fake)
        for name in misaligned:
            setattr(r, name, fake + 4)
        return r

    for fn, args in ((orl_lib.orl_rollout, rollout_args(lib.ENV_CARTPOLE, 2, policy_obs=1)),
                     (orl_lib.orl_rollout, rollout_args(lib.ENV_GRIDWORLD, 5, critic_obs=1)),
                     (orl_lib.orl_share_rollout, rollout_args(lib.ENV_CARTPOLE, 2, policy_obs=1)),
                     (orl_lib.orl_share_rollout, rollout_args(lib.ENV_GRIDWORLD, 5, critic_obs=1))):
        assert fn(args, None) == 10001
        assert b"16-byte aligned" in orl_lib.orl_last_error()
    a.env_kind = lib.ENV_CARTPOLE
    for name in buffers + ("rnn_states",):
        setattr(a, name, fake)
    a.critic_obs = fake + 4
    assert orl_lib.orl_rnn_rollout(a, None) == 10001
    assert b"16-byte aligned" in orl_lib.orl_last_error()


def test_share_update_refuses_what_the_ffma_update_refuses(orl_lib):
    """orl_share_fwdbwd / orl_share_apply refuse, before any launch, ValueNorm without a vn_state (the update reads it
    for the value targets, the optimiser step writes it back) and a contiguous row range past the buffer's end."""
    from openrl_b200 import lib

    fake = 1 << 20   # never dereferenced
    a = lib.OrlPpoArgs()
    a.obs_dim, a.critic_obs_dim, a.n_actions, a.activation_id, a.head_kind = 4, 4, 2, 1, lib.HEAD_CATEGORICAL
    a.grid_per_net, a.batch_rows, a.row_begin, a.total_rows = 1, 1024, 0, 1024
    for name in ("policy_params", "critic_params", "partials", "folded", "grads", "policy_obs", "critic_obs", "actions",
                 "old_log_probs", "advantages", "value_preds", "returns", "active_masks", "gae_stats", "mb_stats",
                 "policy_adam_m", "policy_adam_v", "critic_adam_m", "critic_adam_v", "adam_steps", "lrs", "train_info"):
        setattr(a, name, fake)
    a.flags, a.vn_state = lib.PPO_VALUENORM, None
    for fn in (orl_lib.orl_share_fwdbwd, orl_lib.orl_share_apply):
        assert fn(a, None) == 10001
        assert b"vn_state" in orl_lib.orl_last_error()
    a.vn_state = fake
    for begin, rows in ((1, 1024), (0, 1025), (-1, 4)):
        a.row_begin, a.batch_rows = begin, rows
        assert orl_lib.orl_share_fwdbwd(a, None) == 10001
        assert b"row range" in orl_lib.orl_last_error()
