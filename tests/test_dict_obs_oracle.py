"""Host envs with a Dict {"policy", "critic"} observation space, without a GPU: the oracle loop (oracle/loop_ma.MATrainer
on tests/dict_obs_oracle.py) against traces of the unmodified reference (tests/golden/trace_dict_obs_*.npz,
tools/gen_golden_dict_obs.py) — actions, both observations and masks bit for bit, the update scalars and parameters at
1e-4 — and the host side of the device path: SyncHostVecEnv's per-key stacking, HostVecEnv's staged block and its
refusals."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from helpers import trace_threads  # noqa: F401  (autouse fixture)
from oracle import loop


@pytest.mark.parametrize("tag", ["dict_obs_ff", "dict_obs_gru"])
def test_dict_obs_oracle_reproduces_reference_trace(tag):
    from dict_obs_oracle import DictObsMATrainer

    d = np.load(os.path.join(GOLDEN, f"trace_{tag}.npz"), allow_pickle=True)
    cfg = loop.cfg_from_flags(str(d["meta/flags"]))
    tr = DictObsMATrainer(cfg, int(d["meta/env_num"]))
    params = lambda: {f"{mk}.{k}": v.detach().numpy() for mk, p in (("policy", tr.pol), ("critic", tr.cri))  # noqa: E731
                      for k, v in p.items()}
    for k, v in params().items():
        np.testing.assert_allclose(v, d[f"init/{k}"], rtol=0, atol=1e-6, err_msg=k)
    assert tr.pol["base.mlp.fc1.0.weight"].shape[1] == 3 and tr.cri["base.mlp.fc1.0.weight"].shape[1] == 7
    for it in range(int(d["meta/iters"])):
        tr.rollout()
        b = tr.buf
        assert np.array_equal(b.actions, d[f"it{it}/actions"])
        assert np.array_equal(b.policy_obs, d[f"it{it}/policy_obs"])
        assert np.array_equal(b.critic_obs, d[f"it{it}/critic_obs"])
        assert np.array_equal(b.masks, d[f"it{it}/masks"])
        assert (b.masks[1:] == 0).any()                                   # episodes ended inside the rollout
        assert np.array_equal(b.critic_obs[..., :3], b.policy_obs)        # the policy sees part of the critic's state
        if cfg.use_recurrent_policy:
            np.testing.assert_allclose(b.rnn_states, d[f"it{it}/rnn_states"], rtol=0, atol=1e-5)
            np.testing.assert_allclose(b.rnn_states_critic, d[f"it{it}/rnn_states_critic"], rtol=0, atol=1e-5)
        tr.compute_returns()
        np.testing.assert_allclose(b.value_preds, d[f"it{it}/value_preds"], rtol=0, atol=1e-5)
        updates, perms = tr.train()
        assert np.array_equal(perms, d[f"it{it}/perms"])
        np.testing.assert_allclose(updates, d[f"it{it}/updates"], rtol=1e-4, atol=1e-6)
        tr.after_update()
        for k, v in params().items():
            np.testing.assert_allclose(v, d[f"it{it}/params/{k}"], rtol=1e-4, atol=1e-6, err_msg=k)


class _MultiDictEnv:
    """A 3-agent env with Dict observations (A, 2) / (A, 5) and horizon 2: agent a of the env with counter c sees
    [c, a] and the critic [c, a, c + a, seed, 7]."""
    agent_num = 3

    def __init__(self):
        from openrl_b200 import spaces

        self.observation_space = spaces.Dict({"policy": spaces.Box(-np.inf, np.inf, (2,), np.float32),
                                              "critic": spaces.Box(-np.inf, np.inf, (5,), np.float32)})
        self.action_space = spaces.Discrete(3)
        self.c, self.seed = 0, 0

    def _obs(self):
        a = np.arange(3, dtype=np.float32)
        c = np.full(3, self.c, np.float32)
        return {"policy": np.stack([c, a], 1), "critic": np.stack([c, a, c + a, np.full(3, self.seed), np.full(3, 7.0)], 1)}

    def reset(self, seed=None, options=None):
        self.c = 0
        if seed is not None:
            self.seed = seed
        return self._obs(), {}

    def step(self, action):
        self.c += 1
        return self._obs(), np.ones(3), np.full(3, self.c >= 2), {}


def test_sync_host_vec_env_stacks_dict_observations():
    """Single-agent (d,) / (dc,) and multi-agent (A, d) / (A, dc) entries stack to {"policy": (N, A, d), "critic":
    (N, A, dc)} float32, in reset and in step_range; an auto-reset env's `final_observation` is its own dict."""
    from dict_obs_oracle import DictTargetEnv, SpacedDictTargetEnv
    from openrl_b200.envs.vec_env.host_sync import SyncHostVecEnv

    env = SyncHostVecEnv([SpacedDictTargetEnv for _ in range(3)])
    obs, _ = env.reset(seed=4)
    assert set(obs) == {"policy", "critic"}
    assert obs["policy"].shape == (3, 1, 3) and obs["critic"].shape == (3, 1, 7) and obs["policy"].dtype == np.float32
    assert np.array_equal(obs["critic"][..., :3], obs["policy"])
    for t in range(DictTargetEnv.HORIZON):
        obs, rewards, dones, infos = env.step_range(1, 3, np.zeros((2, 1, 1), np.int64))
        assert obs["policy"].shape == (2, 1, 3) and obs["critic"].shape == (2, 1, 7)
    assert dones.all()
    fin = infos[0]["final_observation"]
    assert isinstance(fin, dict) and fin["critic"].shape == (7,) and fin["critic"][4] == 1.0   # the last step's state
    assert (obs["critic"][:, 0, 4] == 0).all()                                                  # the new episodes

    env = SyncHostVecEnv([_MultiDictEnv for _ in range(2)])
    obs, _ = env.reset(seed=9)
    assert obs["policy"].shape == (2, 3, 2) and obs["critic"].shape == (2, 3, 5)
    env.step(np.zeros((2, 3, 1), np.int64))
    obs, rewards, dones, infos = env.step(np.zeros((2, 3, 1), np.int64))
    assert dones.all() and infos[1]["final_observation"]["critic"].shape == (3, 5)
    assert np.array_equal(infos[1]["final_observation"]["policy"][:, 0], [2, 2, 2])
    assert np.array_equal(obs["critic"][1], [[0, 0, 0, 9 + 10086, 7], [0, 1, 1, 9 + 10086, 7], [0, 2, 2, 9 + 10086, 7]])


class _Host:
    """The reference's host vec-env duck type over _MultiDictEnv, reporting (A, n) masks on steps where `masked(t)`."""

    def __init__(self, n, masked=lambda t: False, space=None):
        from openrl_b200.envs.vec_env.host_sync import SyncHostVecEnv

        self.inner = SyncHostVecEnv([_MultiDictEnv for _ in range(n)])
        self.parallel_env_num, self.agent_num = n, 3
        self.observation_space = space if space is not None else self.inner.observation_space
        self.action_space = self.inner.action_space
        self.masked, self.t = masked, 0

    def step_range(self, lo, hi, actions):
        return self.inner.step_range(lo, hi, actions)

    def reset(self, seed=None):
        return self.inner.reset(seed=seed)

    def step(self, actions):
        obs, rewards, dones, infos = self.inner.step(actions)
        if self.masked(self.t):
            infos = [dict(info, action_masks=np.eye(3, dtype=np.int8)) for info in infos]
        self.t += 1
        return obs, rewards, dones, infos


def test_host_env_stages_critic_section():
    """HostVecEnv stages [policy obs | critic obs | rewards | dones (| masks)] in one block; reset_into writes the
    critic entry into the given critic slot; a flat Box env's block keeps its length."""
    from openrl_b200.envs.vec_env.host_venv import HostVecEnv

    N, A, d, dc, n = 4, 3, 2, 5, 3
    env = HostVecEnv(_Host(N, masked=lambda t: t == 1), device="cpu")
    assert env.dict_obs and (env.obs_dim, env.critic_obs_dim) == (d, dc)
    B = N * A
    obs0, cobs0 = torch.zeros(B, d), torch.zeros(B, dc)
    assert not env.reset_into(obs0, cobs0, torch.ones(B, n))
    assert np.array_equal(cobs0.numpy()[:3], [[0, 0, 0, 0, 7], [0, 1, 1, 0, 7], [0, 2, 2, 0, 7]])
    assert np.array_equal(obs0.numpy(), cobs0.numpy()[:, :2])
    for t in range(2):
        env.fetch_actions(0, N, torch.zeros(B, 1))
        dev, obs, rewards, dones, infos, has = env.step_staged(0, N)
        blk = dev.numpy()
        assert has == (t == 1)
        assert blk.size == B * (d + dc + 2 + (n if has else 0))
        assert np.array_equal(blk[:B * d], obs["policy"].reshape(-1))
        assert np.array_equal(blk[B * d:B * (d + dc)], obs["critic"].reshape(-1))
        assert np.array_equal(blk[B * (d + dc):B * (d + dc + 1)], np.ones(B))
        assert np.array_equal(blk[B * (d + dc + 1):B * (d + dc + 2)], dones.reshape(-1).astype(np.float32))
        if has:
            assert np.array_equal(blk[B * (d + dc + 2):].reshape(B, n), np.tile(np.eye(3), (N, 1)))
    # a sub-range stages its own rows only
    assert env.supports_groups
    env.fetch_actions(1, 3, torch.zeros(2 * A, 1))
    dev, obs, *_ = env.step_staged(1, 3)
    assert dev.numel() == 2 * A * (d + dc + 2) and obs["critic"].shape == (2, A, dc)

    # flat Box: no critic section, the length is what it was
    from openrl_b200 import spaces
    box = _Host(N, masked=lambda t: t == 0, space=spaces.Box(-np.inf, np.inf, (d,), np.float32))
    box.reset = lambda seed=None: (box.inner.reset(seed=seed)[0]["policy"], [{}] * N)
    step = box.step
    box.step = lambda a: (lambda o, r, dn, i: (o["policy"], r, dn, i))(*step(a))
    env = HostVecEnv(box, device="cpu")
    assert not env.dict_obs and env.critic_obs_dim == d
    env.reset_into(torch.zeros(B, d))
    for t in range(2):
        env.fetch_actions(0, N, torch.zeros(B, 1))
        dev, obs, rewards, dones, infos, has = env.step_staged(0, N)
        assert dev.numel() == B * (d + 2 + (n if has else 0)) and has == (t == 0)
        assert np.array_equal(dev.numpy()[:B * d], obs.reshape(-1))


@pytest.mark.parametrize("case", ["extra_key", "missing_key", "non_box", "wide", "image"])
def test_host_env_refuses_unsupported_dict_spaces(case):
    from openrl_b200 import spaces
    from openrl_b200.envs.vec_env.host_venv import HostVecEnv

    box = lambda w: spaces.Box(-np.inf, np.inf, (w,), np.float32)  # noqa: E731
    space, match = {
        "extra_key": (spaces.Dict({"policy": box(3), "critic": box(7), "goal": box(2)}), "exactly the keys"),
        "missing_key": (spaces.Dict({"policy": box(3)}), "exactly the keys"),
        "non_box": (spaces.Dict({"policy": box(3), "critic": spaces.Discrete(4)}), "'critic' is"),
        "wide": (spaces.Dict({"policy": box(3), "critic": box(65)}), "'critic' observation has width 65"),
        "image": (spaces.Dict({"policy": spaces.Box(0, 1, (4, 4), np.float32), "critic": box(7)}), "'policy' is"),
    }[case]
    host = _Host(2, space=space)
    with pytest.raises(NotImplementedError, match=match):
        HostVecEnv(host, device="cpu")
