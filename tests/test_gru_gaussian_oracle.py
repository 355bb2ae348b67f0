"""GRU policies with DiagGaussian heads (cfg.use_recurrent_gaussian_head) without a GPU: the recurrent oracle loop of
tests/gru_gaussian_oracle.py against traces of the unmodified reference (tests/golden/trace_gru_gaussian_{spread,box_256}
.npz, tools/gen_golden_gru_gaussian.py) — observations bit for bit, actions at 1e-6, log-probs, hidden states and values at
1e-5, the update scalars and the parameters after the last iteration at 1e-4.  The option, head kinds, parameter count
and refusals are in tests/test_gru_gaussian_cpu.py."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from helpers import trace_threads  # noqa: F401  (autouse fixture)
from oracle import loop


@pytest.mark.parametrize("tag", ["gru_gaussian_spread", "gru_gaussian_box_256"])
def test_oracle_reproduces_reference_trace(tag):
    """3 agents with Dict 18 / 54 observations, Box(5) and agents finishing at different steps (use_recurrent_policy), and
    Box(256) observations with Box(8) (use_naive_recurrent_policy)."""
    from gru_gaussian_oracle import GRUGaussianTrainer

    d = np.load(os.path.join(GOLDEN, f"trace_{tag}.npz"), allow_pickle=True)
    cfg = loop.cfg_from_flags(str(d["meta/flags"]))
    spread = tag == "gru_gaussian_spread"
    assert (cfg.use_recurrent_policy, cfg.use_naive_recurrent_policy) == ((True, False) if spread else (False, True))
    tr = GRUGaussianTrainer(cfg, int(d["meta/env_num"]), tag)
    n = 5 if spread else 8
    assert d["init/policy.act.action_out.fc_mean.weight"].shape == (n, 64)
    assert d["init/policy.act.action_out.logstd._bias"].shape == (n,) or d["init/policy.act.action_out.logstd._bias"].size == n
    params = lambda: {f"{mk}.{k}": v.detach().numpy() for mk, p in (("policy", tr.pol), ("critic", tr.cri))  # noqa: E731
                      for k, v in p.items()}
    for k, v in params().items():
        np.testing.assert_allclose(v, d[f"init/{k}"], rtol=0, atol=1e-6, err_msg=k)
    last = int(d["meta/iters"]) - 1
    for it in range(int(d["meta/iters"])):
        t = f"it{it}"
        tr.rollout()
        b = tr.buf
        assert b.actions.shape[-1] == n
        # float actions carry the GRU's rounding (the oracle's cell vs torch.nn.GRU): 1e-6, not bit for bit
        np.testing.assert_allclose(b.actions, d[f"{t}/actions"], rtol=0, atol=1e-6, err_msg=t)
        assert np.array_equal(b.policy_obs, d[f"{t}/policy_obs"]), t
        assert np.array_equal(b.masks, d[f"{t}/masks"]), t
        assert np.array_equal(b.active_masks, d[f"{t}/active_masks"]), t
        if spread:
            assert np.array_equal(b.critic_obs, d[f"{t}/critic_obs"]), t
            assert (b.active_masks == 0).any()   # agents that finished before their env
        np.testing.assert_allclose(b.action_log_probs, d[f"{t}/action_log_probs"], rtol=0, atol=1e-5, err_msg=t)
        np.testing.assert_allclose(b.rnn_states, d[f"{t}/rnn_states"], rtol=0, atol=1e-5, err_msg=t)
        tr.compute_returns()
        np.testing.assert_allclose(b.value_preds, d[f"{t}/value_preds"], rtol=0, atol=1e-5, err_msg=t)
        updates, perms = tr.train()
        assert np.array_equal(perms, d[f"{t}/perms"]), t
        np.testing.assert_allclose(updates, d[f"{t}/updates"], rtol=1e-4, atol=1e-6, err_msg=t)
        tr.after_update()
        if it == last:   # the traces keep the weights at init and after the last iteration
            for k, v in params().items():
                np.testing.assert_allclose(v, d[f"{t}/params/{k}"], rtol=1e-4, atol=1e-6, err_msg=k)
