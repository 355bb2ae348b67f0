"""Wide Discrete action spaces (9..64 actions) with a GRU policy, without a GPU: the recurrent oracle loop with the
reference's mask ingest against traces of the unmodified reference on the masked env widened to 9 and 64 actions
(tests/golden/trace_wide_actions_gru_*.npz, tools/gen_golden_wide_actions_gru.py)."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from helpers import trace_threads  # noqa: F401  (autouse fixture)
from oracle import loop
from wide_actions_gru_oracle import WideMaskedMATrainer
from wide_actions_oracle import WIDTHS


def _illegal(actions, action_masks):
    a = actions[..., 0].astype(np.int64)
    return int((np.take_along_axis(action_masks[:-1], a[..., None], axis=-1) == 0).sum())


@pytest.mark.parametrize("n", WIDTHS)
def test_wide_gru_oracle_reproduces_reference_trace(n):
    d = np.load(os.path.join(GOLDEN, f"trace_wide_actions_gru_{n}.npz"), allow_pickle=True)
    cfg = loop.cfg_from_flags(str(d["meta/flags"]))
    assert cfg.use_recurrent_policy and cfg.data_chunk_length == 3
    tr = WideMaskedMATrainer(cfg, int(d["meta/env_num"]), n)
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
        assert np.array_equal(b.policy_obs, d[f"it{it}/policy_obs"])
        assert np.array_equal(b.masks, d[f"it{it}/masks"])
        assert np.array_equal(b.action_masks, am)
        assert (am == 0).any() and _illegal(b.actions, am) == 0
        assert (b.masks[1:] == 0).any()   # episodes ended inside the rollout, so hidden states were reset mid-chunk
        assert b.actions.max() >= 8       # actions beyond the 8 the narrow head holds were sampled
        np.testing.assert_allclose(b.rnn_states, d[f"it{it}/rnn_states"], rtol=0, atol=1e-5)
        tr.compute_returns()
        np.testing.assert_allclose(b.value_preds, d[f"it{it}/value_preds"], rtol=0, atol=1e-5)
        updates, perms = tr.train()
        assert np.array_equal(perms, d[f"it{it}/perms"])
        np.testing.assert_allclose(updates, d[f"it{it}/updates"], rtol=1e-4, atol=1e-6)
        tr.after_update()
        for k, v in params().items():
            np.testing.assert_allclose(v, d[f"it{it}/params/{k}"], rtol=1e-4, atol=1e-6, err_msg=k)
