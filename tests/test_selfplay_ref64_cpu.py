"""The float64 self-play replay (tests/selfplay_ref64.py) against the oracles it restates.

- Game step, table resets and the outcome tally with scripted actions for both players equal
  oracle.selfplay.GridWorld2P, the numpy oracle the device game step is pinned to bit-exactly.
- The policy forward on the flat parameter layout equals oracle/nets.py (`mlp_base` + the categorical head) in float64
  on the same parameters under their state_dict names, for every activation and for a trunk whose first LayerNorm sees
  zero variance.
- The Philox start cells take the first valid of 16 tries and fall back to (0, 0, 0, 2); the opponent pick follows the
  two strategies."""
import numpy as np
import pytest
import torch

import selfplay_ref64 as ref
from oracle import nets
from oracle.selfplay import GridWorld2P

SEED = 0x5EED_0F_5E1F


def _start_table(rng, N, K):
    t = rng.integers(0, 10, (N, K, 4))
    bad = lambda c: ((c[..., 0] == 1) & (c[..., 1] == 1)) | ((c[..., 2] == 1) & (c[..., 3] == 1)) | (  # noqa: E731
        (c[..., 0] == c[..., 2]) & (c[..., 1] == c[..., 3]))
    while bad(t).any():
        t[bad(t)] = rng.integers(0, 10, (int(bad(t).sum()), 4))
    return t


def test_replay_game_matches_gridworld2p_oracle():
    rng = np.random.default_rng(0)
    N, T, K = 300, 260, 6
    table = _start_table(rng, N, K)
    acts = rng.integers(0, 5, (T, N, 2))
    acts[:, : N // 5] = 0                               # envs that never move: 100-step time-outs
    acts[:, N // 5: N // 3, 0] = np.where(rng.random((T, N // 3 - N // 5)) < 0.5, 1, 3)   # learners drift to the goal
    acts[:, N // 3: N // 2, 1] = np.where(rng.random((T, N // 2 - N // 3)) < 0.5, 1, 3)   # opponents drift to the goal
    ora = GridWorld2P(table)
    obs0 = ora.reset()
    rep = ref.SelfPlayReplay(table[:, 0], np.zeros(N), np.ones(N), -np.ones(N), np.zeros(N), np.zeros(N), seed=SEED, row_offset=0,
                             strategy="RandomOpponent", pool_params=np.zeros((3, ref.param_count())), pool_count=0,
                             activation_id=1, table=table)
    assert np.array_equal(rep.pos.astype(np.float32), obs0)
    res = rep.rollout(np.zeros(ref.param_count()), T, 0, learner_actions=acts[..., 0], opponent_actions=acts[..., 1])
    ep_ret, ep_len = np.zeros(N), np.zeros(N)
    stats = np.zeros(3)
    for t in range(T):
        o, r, d = ora.step(acts[t, :, 0], acts[t, :, 1])
        assert np.array_equal(res.obs[t + 1], o), t
        assert np.array_equal(res.rewards[t], r), t
        assert np.array_equal(res.masks[t + 1] == 0, d), t
        ep_ret += r
        ep_len += 1
        stats += [ep_ret[d].sum(), ep_len[d].sum(), d.sum()]
        ep_ret[d], ep_len[d] = 0, 0
    assert np.array_equal(rep.pool_stats[-1], ora.outcomes) and rep.pool_stats[:-1].sum() == 0
    assert ora.outcomes.min() > 0 and ora.nreset.max() > K          # every outcome, and resets past the table's end
    assert np.array_equal(rep.nreset, ora.nreset) and np.array_equal(rep.steps, ora.steps)
    assert np.array_equal(rep.ep_return, ep_ret) and np.array_equal(rep.ep_length, ep_len)
    assert np.array_equal(rep.episode_stats, stats)


def _random_flat(rng, head_scale):
    p = {}
    for name, shp in ref.param_shapes():
        base = 1.0 if name.endswith(("fc1.2.weight", "fc3.1.weight")) else 0.0
        p[name] = base + rng.normal(0, 0.5, shp)
    p["act.action_out.linear.weight"] *= head_scale
    return p, np.concatenate([v.reshape(-1) for v in p.values()])


@pytest.mark.parametrize("activation_id", [0, 1, 2, 3])
@pytest.mark.parametrize("dead", [False, True])
def test_replay_forward_matches_oracle_nets(activation_id, dead):
    rng = np.random.default_rng(10 + activation_id)
    p, flat = _random_flat(rng, 3.0)
    if dead:                                  # every fc1 unit far below zero: LayerNorm of a (nearly) constant row
        p["base.mlp.fc1.0.weight"] *= 0.1
        p["base.mlp.fc1.0.bias"][:] = -40.0
        flat = np.concatenate([v.reshape(-1) for v in p.values()])
    obs = rng.integers(0, 10, (500, 4)).astype(np.float64)
    got = ref.log_softmax(ref.policy_logits(flat, obs, activation_id))
    sd = {k: torch.from_numpy(v) for k, v in p.items()}
    want = nets.categorical_logits(sd, nets.mlp_base(sd, "base", torch.from_numpy(obs), 1, activation_id)).numpy()
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-10)
    if dead and activation_id != 2:           # the policy no longer depends on the observation (leaky ReLU stays alive)
        assert got.std(0).max() < 1e-6
    else:
        assert got.std(0).max() > 0.1


def test_reset_cells_first_valid_try_and_fallback(monkeypatch):
    key, nreset = np.arange(2000) + 123, np.arange(2000) * 7 + 5
    cells = ref.reset_cells(key, nreset, SEED)
    assert ((cells >= 0) & (cells < 10)).all()
    assert not ((cells[:, 0] == 1) & (cells[:, 1] == 1)).any() and not ((cells[:, 2] == 1) & (cells[:, 3] == 1)).any()
    assert not ((cells[:, 0] == cells[:, 2]) & (cells[:, 1] == cells[:, 3])).any()
    w = ref.philox4x32_10(key, nreset, ref.RESET_TAG, 0, SEED)     # try 0 is valid for almost every env and decides it
    try0 = np.stack([ref._u32_scaled(x, 10) for x in w], -1)
    assert (cells == try0).all(-1).mean() > 0.9

    real = ref.philox4x32_10
    goal = np.uint64(0x1A000000)                                    # (goal * 10) >> 32 == 1: every cell is the goal

    def first_valid_at(k):
        def fake(c0, c1, c2, c3, seed):
            out = real(c0, c1, c2, c3, seed)
            bad = np.asarray(c3, np.uint64) < np.uint64(k)
            return [np.where(bad, goal, x) for x in out]
        return fake

    monkeypatch.setattr(ref, "philox4x32_10", first_valid_at(5))
    w5 = real(key, nreset, ref.RESET_TAG, 5, SEED)
    try5 = np.stack([ref._u32_scaled(x, 10) for x in w5], -1)
    ok5 = ~((try5[:, 0] == 1) & (try5[:, 1] == 1)) & ~((try5[:, 2] == 1) & (try5[:, 3] == 1)) & ~(
        (try5[:, 0] == try5[:, 2]) & (try5[:, 1] == try5[:, 3]))
    assert np.array_equal(ref.reset_cells(key, nreset, SEED)[ok5], try5[ok5])
    monkeypatch.setattr(ref, "philox4x32_10", first_valid_at(16))
    assert (ref.reset_cells(key, nreset, SEED) == np.array(ref.RESET_FALLBACK)).all()


def test_pick_opponent_strategies():
    key, nreset = np.arange(40_000) + 9, np.arange(40_000) % 977
    for strategy in ("RandomOpponent", "LastOpponent"):
        assert (ref.pick_opponent(strategy, 0, 8, key, nreset, SEED) == -1).all()
        assert (ref.pick_opponent(strategy, 3, 0, key, nreset, SEED) == -1).all()
    assert (ref.pick_opponent("LastOpponent", 11, 8, key, nreset, SEED) == 2).all()
    assert (ref.pick_opponent("LastOpponent", 5, 8, key, nreset, SEED) == 4).all()
    for count, avail in ((5, 5), (11, 8)):
        got = ref.pick_opponent("RandomOpponent", count, 8, key, nreset, SEED)
        c = np.bincount(got, minlength=avail)
        assert c.size == avail and c.min() > 0.9 * key.size / avail
