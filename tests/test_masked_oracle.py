"""The oracle loops with the reference's action-mask ingest (tests/masked_oracle.py) against traces of the unmodified
reference on an env that reports legal-move masks (tests/golden/trace_masked_*.npz, tools/gen_golden_masked.py): same
actions, observations, masks and action masks bit for bit, the update scalars and parameters at 1e-4; plus the
mask-building rule of the host vec-env (no GPU)."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from helpers import trace_threads  # noqa: F401  (autouse fixture)
from oracle import loop


def _illegal(actions, action_masks):
    """Count of actions[t] that action_masks[t] forbids."""
    a = actions[..., 0].astype(np.int64)
    return int((np.take_along_axis(action_masks[:-1], a[..., None], axis=-1) == 0).sum())


@pytest.mark.parametrize("tag", ["masked_ff", "masked_gru"])
def test_masked_oracle_reproduces_reference_trace(tag):
    from masked_oracle import MaskedMATrainer, MaskedTrainer

    d = np.load(os.path.join(GOLDEN, f"trace_{tag}.npz"), allow_pickle=True)
    cfg = loop.cfg_from_flags(str(d["meta/flags"]))
    N = int(d["meta/env_num"])
    tr = (MaskedMATrainer if cfg.use_recurrent_policy else MaskedTrainer)(cfg, N)
    params = lambda: {f"{mk}.{k}": v.detach().numpy() for mk, p in (("policy", tr.pol), ("critic", tr.cri))  # noqa: E731
                      for k, v in p.items()}
    for k, v in params().items():
        np.testing.assert_allclose(v, d[f"init/{k}"], rtol=0, atol=1e-6, err_msg=k)
    for it in range(int(d["meta/iters"])):
        tr.rollout()
        b = tr.buf
        obs = b.policy_obs if cfg.use_recurrent_policy else b.obs
        am = d[f"it{it}/action_masks"]
        assert np.array_equal(b.actions, d[f"it{it}/actions"])
        assert np.array_equal(obs, d[f"it{it}/policy_obs"])
        assert np.array_equal(b.masks, d[f"it{it}/masks"])
        assert np.array_equal(b.action_masks, am)
        assert (am == 0).any() and _illegal(b.actions, am) == 0     # the masks are real and were obeyed
        assert (b.masks[1:] == 0).any()                             # episodes ended inside the rollout
        if cfg.use_recurrent_policy:
            np.testing.assert_allclose(b.rnn_states, d[f"it{it}/rnn_states"], rtol=0, atol=1e-5)
        tr.compute_returns()
        np.testing.assert_allclose(b.value_preds, d[f"it{it}/value_preds"], rtol=0, atol=1e-5)
        updates, perms = tr.train()
        assert np.array_equal(perms, d[f"it{it}/perms"])
        np.testing.assert_allclose(updates, d[f"it{it}/updates"], rtol=1e-4, atol=1e-6)
        assert updates[:, 3].max() < np.log(5) - 0.2                 # the entropy is that of the masked distributions
        tr.after_update()
        for k, v in params().items():
            np.testing.assert_allclose(v, d[f"it{it}/params/{k}"], rtol=1e-4, atol=1e-6, err_msg=k)


def test_oracle_keeps_stale_slots_when_masks_are_missing():
    """Steps whose infos lack the key in one env write no masks: the slot keeps what it held (ones, or the previous
    iteration's value)."""
    from masked_oracle import MaskedTrainer

    cfg = loop.make_cfg(episode_length=6, ppo_epoch=1)
    tr = MaskedTrainer(cfg, 3, report=lambda i, t: not (i == 1 and t % 4 == 2))
    before = tr.buf.action_masks.copy()
    tr.rollout()
    am = tr.buf.action_masks
    assert np.array_equal(am[3], before[3])          # step 2 of env 1 lacked the key: slot 3 untouched (all ones)
    assert (am[[1, 2, 4, 5, 6]] == 0).any()


def test_prepare_action_masks_rule():
    """prepare_action_masks (envs/vec_env/utils/util.py:54-88) as the host vec-env stages it: (n,) applies to every
    agent, (A, n) one row per agent, int8 cast (0 = illegal), None when any env lacks the key."""
    from openrl_b200.envs.vec_env.host_venv import prepare_action_masks

    one = {"action_masks": np.array([1, 0, 1])}
    per = {"action_masks": np.array([[1, 1, 0], [0, 1, 1]])}
    assert prepare_action_masks(None) is None
    m = prepare_action_masks([one, one], agent_num=2)
    assert m.dtype == np.int8 and m.shape == (4, 3) and (m == [1, 0, 1]).all()
    m = prepare_action_masks([per, {"action_masks": [[0, 0, 1], [1, 0, 0]]}], agent_num=2)
    assert np.array_equal(m, [[1, 1, 0], [0, 1, 1], [0, 0, 1], [1, 0, 0]])
    assert prepare_action_masks([one, {}], agent_num=1) is None
    assert prepare_action_masks([one, {"final_observation": 0}], agent_num=1) is None
    assert np.array_equal(prepare_action_masks([{"action_masks": [True, False, 2.5]}]), [[1, 0, 2]])


def test_host_env_stages_masks_of_auto_reset_infos_over_env_range():
    """HostVecEnv's staged step of the whole env range stages [obs | rewards | dones | masks] when every env reported
    masks, the auto-reset info's masks for a finished env (the new episode's first observation), and reports their
    absence otherwise."""
    from masked_oracle import MaskedTargetVec
    from openrl_b200 import spaces
    from openrl_b200.envs.vec_env.host_venv import HostVecEnv

    class Host:
        def __init__(self, inner):
            self.inner, self.parallel_env_num, self.agent_num = inner, inner.N, 1
            self.observation_space = spaces.Box(0, 1, (5,), np.float32)
            self.action_space = spaces.Discrete(5)

        def reset(self, seed=None):
            return self.inner.reset(seed=seed), self.inner.last_infos

        def step(self, actions):
            return self.inner.step(actions)

    N = 3
    inner = MaskedTargetVec(N, report=lambda i, t: t != 2)
    env = HostVecEnv(Host(inner), device="cpu")
    obs0 = torch.zeros(N, 5)
    am0 = torch.ones(N, 5)
    assert env.reset_into(obs0, None, am0)
    assert np.array_equal(am0.numpy(), np.stack([i["action_masks"] for i in inner.last_infos]))
    for t in range(6):
        acts = torch.tensor([[float(e.target)] for e in inner.envs])
        env.fetch_actions(0, N, acts)
        dev, obs, rewards, dones, infos, has = env.step_staged(0, N)
        blk = dev.numpy()
        assert has == (t != 2)
        if not has:
            assert blk.size == N * (5 + 2)
            continue
        assert blk.size == N * (5 + 2 + 5)
        want = np.stack([i["action_masks"] for i in infos]).astype(np.float32)
        assert np.array_equal(blk[N * 7:].reshape(N, 5), want)
        # a finished env's masks are those of the reset observation: the target is always legal
        tgt = blk[:N * 5].reshape(N, 5).argmax(1)
        assert (want[np.arange(N), tgt] == 1).all()
        if t == 4:
            assert dones.all()          # horizon 5: every env auto-reset at this step
