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
