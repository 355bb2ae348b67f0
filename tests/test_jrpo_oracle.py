"""Joint-action PPO (JRPO) oracle (tests/jrpo_oracle.py) against traces of the unmodified reference:
simple_spread with the examples/mpe/mpe_jrpo.yaml flags (one minibatch of 2-step chunks, and two minibatches of
4-step chunks), and, with one agent, the ordinary recurrent CartPole trace, which JRPO must reproduce as recorded."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from helpers import trace_threads  # noqa: F401  (autouse fixture)
from oracle import loop


@pytest.mark.parametrize("tag,env_id", [("mpe_jrpo", "simple_spread"), ("mpe_jrpo_mb", "simple_spread"),
                                        ("cartpole_gru", "CartPole-v1")])
def test_jrpo_oracle_reproduces_reference_trace(tag, env_id):
    import jrpo_oracle

    d = np.load(os.path.join(GOLDEN, f"trace_{tag}.npz"), allow_pickle=True)
    flags = str(d["meta/flags"])
    assert ("--use_joint_action_loss true" in flags) == tag.startswith("mpe_jrpo")
    cfg = loop.cfg_from_flags(flags)
    tr = jrpo_oracle.JointTrainer(cfg, env_id, int(d["meta/env_num"]))
    for mk, prm in (("policy", tr.pol), ("critic", tr.cri)):
        for k, v in prm.items():
            np.testing.assert_allclose(v.detach().numpy(), d[f"init/{mk}.{k}"], rtol=0, atol=1e-6, err_msg=k)
            v.data.copy_(torch.from_numpy(d[f"init/{mk}.{k}"]))
    for it in range(int(d["meta/iters"])):
        tr.rollout()
        b = tr.buf
        assert np.array_equal(b.actions, d[f"it{it}/actions"])
        assert np.array_equal(b.policy_obs, d[f"it{it}/policy_obs"])
        assert np.array_equal(b.rewards, d[f"it{it}/rewards"])
        assert np.array_equal(b.masks, d[f"it{it}/masks"])
        np.testing.assert_allclose(b.rnn_states, d[f"it{it}/rnn_states"], rtol=0, atol=1e-5)
        np.testing.assert_allclose(b.rnn_states_critic, d[f"it{it}/rnn_states_critic"], rtol=0, atol=1e-5)
        tr.compute_returns()
        np.testing.assert_allclose(b.value_preds, d[f"it{it}/value_preds"], rtol=0, atol=1e-5)
        updates, perms = tr.train()
        assert np.array_equal(perms, d[f"it{it}/perms"])
        np.testing.assert_allclose(tr.last_adv, d[f"it{it}/advantages"], rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(updates, d[f"it{it}/updates"], rtol=2e-4, atol=2e-6)
        tr.after_update()
        for mk, prm in (("policy", tr.pol), ("critic", tr.cri)):
            for k, v in prm.items():
                np.testing.assert_allclose(v.detach().numpy(), d[f"it{it}/params/{mk}.{k}"], rtol=2e-4, atol=2e-6, err_msg=k)


def test_jrpo_traces_use_v3_chunking():
    """The recorded permutations are over the v3 chunk count N*T // L (samples are (env, step) pairs carrying all
    agents), not over the N*T*A // L chunks of the ordinary recurrent generator."""
    for tag, L in (("mpe_jrpo", 2), ("mpe_jrpo_mb", 4)):
        d = np.load(os.path.join(GOLDEN, f"trace_{tag}.npz"), allow_pickle=True)
        N, T = int(d["meta/env_num"]), d["it0/actions"].shape[0]
        assert d["it0/perms"].shape == (2, N * T // L)
