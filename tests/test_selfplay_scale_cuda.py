"""The self-play rollout at C4 scale (GridWorldSelfPlay, 4096 envs, an opponent pool of 8) against the float64 replay
of tests/selfplay_ref64.py.

One launch of `selfplay_rollout_kernel` runs T = 128 steps from a host-written state: distinct random cells, step
counts spread over 0..100 (episodes end all through the launch), random reset counters, and opponents on every ring
slot and on -1 (an episode begun while the pool was empty keeps its random-action opponent).  The pool has taken 11
snapshots, so its ring has wrapped; each has its own weights and a sharp head, and one is dead under ReLU (its first
LayerNorm sees zero variance).  The noise is keyed by a step base above 2^32 and a non-zero env offset (an
env-sharded vec-env).  The replay, teacher-forced on the kernel's learner actions, must reproduce every observation,
reward and mask bit-exactly, the final env state and tallies exactly, the learner's choices up to near-ties and its
log-probs within 1e-5.  Each deliberate replay mistake in `MUTANTS` must show up as mismatches, so the comparison
would notice a kernel that made it.  The vec-env step API is held to the same replay with tanh snapshots."""
import numpy as np
import pytest

import selfplay_ref64 as ref

pytestmark = pytest.mark.gpu

N, T, CAP = 4096, 128, 8
SEED = 0x2545_F491_4F6C_DD1D
STEP_BASE = (3 << 32) + 4321     # the high step word reaches the noise counter
OFFSET = 2 * N                   # this vec-env is shard 2 of a larger one: env_key = env + OFFSET
N_SNAPSHOTS = 11                 # ring of 8 wrapped: slots hold snapshots 8, 9, 10, 3, ..., 7
DEAD_SNAPSHOT = 5                # ring slot 5: every fc1 unit below zero under ReLU
LP_ATOL = 1e-5
TIE_SHARE = 1e-3                 # resolved opponent near-ties per env-step, at most
STRATEGIES = ("RandomOpponent", "LastOpponent")


def _policy(rng, head_scale, dead=False):
    """Flat float32 policy: logits of standard deviation about `head_scale`; `dead`: fc1 pre-activations below -20."""
    p = {}
    for name, shp in ref.param_shapes():
        if name.endswith(("fc1.2.weight", "fc3.1.weight")):
            p[name] = 1.0 + rng.normal(0, 0.2, shp)
        elif name == "base.mlp.fc3.0.weight":
            p[name] = rng.normal(0, 1 / 8, shp)
        elif name == "act.action_out.linear.weight":
            p[name] = rng.normal(0, head_scale / 8, shp)
        else:
            p[name] = rng.normal(0, 0.5, shp)
    if dead:
        p["base.mlp.fc1.0.weight"] *= 0.1
        p["base.mlp.fc1.0.bias"][:] = -30.0
    return np.concatenate([v.reshape(-1) for v in p.values()]).astype(np.float32)


def _make_env(strategy, cap, count, activation_id, n_envs=N):
    """Env with `count` snapshots added to a pool of `cap`; returns it and the snapshots in the order added."""
    import torch

    from openrl_b200.envs.common import make

    env = make("GridWorldSelfPlay", env_num=n_envs, opponent_pool_size=cap, opponent_strategy=strategy, env_index_offset=OFFSET)
    rng = np.random.default_rng(100 + cap)
    snaps = [_policy(rng, 4.0 + 0.5 * k, dead=(k == DEAD_SNAPSHOT)) for k in range(count)]
    for s in snaps:
        env.opponent_pool.add(torch.from_numpy(s).to(env.device), activation_id=activation_id)
    return env, snaps


def _start_state(rng, opp_values):
    pos = rng.integers(0, 10, (N, 4))
    bad = lambda c: ((c[:, 0] == 1) & (c[:, 1] == 1)) | ((c[:, 2] == 1) & (c[:, 3] == 1)) | (  # noqa: E731
        (c[:, 0] == c[:, 2]) & (c[:, 1] == c[:, 3]))
    while bad(pos).any():
        pos[bad(pos)] = rng.integers(0, 10, (int(bad(pos).sum()), 4))
    steps = rng.integers(0, ref.MAX_STEPS + 1, N)
    return dict(pos=pos, steps=steps, nreset=rng.integers(0, 1 << 30, N), opp=rng.permutation(np.resize(np.asarray(opp_values), N)),
                ep_return=-steps.astype(np.float32), ep_length=steps.copy())


def _launch(env, state, learner, activation_id, deterministic):
    """Writes `state` into the env, runs one T-step selfplay rollout launch and returns the recorded buffers and the
    env state / tallies after it."""
    import torch

    from openrl_b200 import lib

    dev = env.device
    s = state
    env.env_i32[:7].copy_(torch.from_numpy(np.stack([*s["pos"].T, s["steps"], s["nreset"], s["opp"]]).astype(np.int32)))
    env.ep_return.copy_(torch.from_numpy(s["ep_return"]))
    env.ep_length.copy_(torch.from_numpy(s["ep_length"].astype(np.int32)))
    env.episode_stats.zero_()
    env.opponent_pool.stats.zero_()
    z = lambda *sh: torch.zeros(*sh, dtype=torch.float32, device=dev)   # noqa: E731
    buf = dict(obs=z(T + 1, N, 4), actions=z(T, N), logp=z(T, N), rewards=z(T, N), masks=z(T + 1, N), active_masks=z(T + 1, N))
    buf["obs"][0].copy_(torch.from_numpy(s["pos"].astype(np.float32)))
    params = torch.from_numpy(learner).to(dev)
    a = lib.OrlRolloutArgs()
    a.env_kind, a.n_envs, a.n_agents, a.episode_length = env.kind, N, 1, T
    a.t_begin, a.t_end, a.obs_dim, a.n_actions = 0, T, 4, ref.N_ACTIONS
    a.activation_id, a.deterministic = activation_id, deterministic
    a.policy_params, a.policy_obs = lib.ptr(params), lib.ptr(buf["obs"])
    a.actions, a.action_log_probs, a.rewards = lib.ptr(buf["actions"]), lib.ptr(buf["logp"]), lib.ptr(buf["rewards"])
    a.masks, a.active_masks = lib.ptr(buf["masks"]), lib.ptr(buf["active_masks"])
    a.rng_seed, a.rng_step_base, a.rng_row_offset = SEED, STEP_BASE, env.env_index_offset
    a.env_i32, a.env_table, a.env_table_len = lib.ptr(env.env_i32), lib.ptr(env.env_table), env.env_table_len
    a.ep_return, a.ep_length, a.episode_stats = lib.ptr(env.ep_return), lib.ptr(env.ep_length), lib.ptr(env.episode_stats)
    lib.check(lib.load().orl_selfplay_rollout(env.selfplay_args(a), lib.current_stream()), "orl_selfplay_rollout")
    torch.cuda.synchronize()
    kernel = {k: v.cpu().numpy() for k, v in buf.items()}
    final = dict(env_i32=env.env_i32.cpu().numpy(), ep_return=env.ep_return.cpu().numpy(), ep_length=env.ep_length.cpu().numpy(),
                 episode_stats=env.episode_stats.cpu().numpy(), pool_stats=env.opponent_pool.stats.cpu().numpy())
    return kernel, final


def _run(activation_id, strategy, cap=CAP, count=N_SNAPSHOTS, deterministic=0):
    import types

    env, snaps = _make_env(strategy, cap, count, activation_id)
    pool_params = env.opponent_pool.params.cpu().numpy()[:cap]
    for slot in range(min(count, cap)):          # the ring: slot s holds the newest snapshot k with k % cap == s
        k = max(k for k in range(count) if k % cap == slot)
        assert np.array_equal(pool_params[slot, :ref.param_count()], snaps[k])
    rng = np.random.default_rng(7 + activation_id)
    state = _start_state(rng, [-1] + list(range(min(count, cap))))
    learner = _policy(rng, 2.0)
    kernel, final = _launch(env, state, learner, activation_id, deterministic)
    return types.SimpleNamespace(activation_id=activation_id, strategy=strategy, cap=cap, count=count, deterministic=deterministic,
                                 state=state, learner=learner, pool_params=pool_params, kernel=kernel, final=final)


@pytest.fixture(scope="module")
def trajectory(cuda):
    """Kernel trajectories by configuration, run once per module (the mutation test replays the one test 1 checked)."""
    cache = {}

    def get(activation_id, strategy, **kw):
        key = (activation_id, strategy, tuple(sorted(kw.items())))
        if key not in cache:
            cache[key] = _run(activation_id, strategy, **kw)
        return cache[key]
    return get


def _replay(tr, cls=ref.SelfPlayReplay):
    s = tr.state
    rep = cls(s["pos"], s["steps"], s["nreset"], s["opp"], s["ep_return"], s["ep_length"], seed=SEED, row_offset=OFFSET,
              strategy=tr.strategy, pool_params=tr.pool_params, pool_count=tr.count, activation_id=tr.activation_id)
    return rep, rep.rollout(tr.learner, T, STEP_BASE, deterministic=tr.deterministic, kernel=tr.kernel)


def _check(tr):
    """The bars every launch is held to; returns the replay for further checks."""
    rep, res = _replay(tr)
    bad = ref.mismatches(rep, res, tr.kernel, tr.final)
    assert not any(bad.values()), bad
    lp_err = float(np.abs(tr.kernel["logp"].astype(np.float64) - res.lp).max())
    assert lp_err <= LP_ATOL, lp_err
    assert (tr.kernel["actions"] == res.want).mean() > 0.99
    assert rep.opponent_runner_up <= rep.opponent_near_ties < TIE_SHARE * N * T, (rep.opponent_near_ties, rep.opponent_runner_up)
    st = tr.final["pool_stats"]
    print(f"\n[selfplay C4] act {tr.activation_id} {tr.strategy} pool {tr.count}/{tr.cap} det {tr.deterministic}: "
          f"max |logp - logp64| {lp_err:.2e}, learner near-ties {int(res.tie.sum())}, opponent near-ties "
          f"{rep.opponent_near_ties} (runner-up kept {rep.opponent_runner_up}) of {N * T} env-steps, episodes {int(st.sum())}")
    return rep


@pytest.mark.parametrize("strategy", STRATEGIES)
@pytest.mark.parametrize("activation_id", [0, 1, 2, 3])
def test_rollout_matches_float64_replay(trajectory, activation_id, strategy):
    tr = trajectory(activation_id, strategy)
    _check(tr)
    st = tr.final["pool_stats"]
    assert (st.sum(0) > 0).all(), st                      # wins, losses and draws
    assert (st.sum(1) > 0).all(), st                      # every ring slot (the dead snapshot too) and the random opponent
    if strategy == "LastOpponent":                        # a new episode meets the newest snapshot only
        assert (tr.final["env_i32"][6][tr.final["env_i32"][5] != tr.state["nreset"]] == (N_SNAPSHOTS - 1) % CAP).all()


@pytest.mark.parametrize("strategy", STRATEGIES)
def test_rollout_empty_pool_matches_float64_replay(trajectory, strategy):
    tr = trajectory(3, strategy, count=0)
    _check(tr)
    st = tr.final["pool_stats"]
    assert st[:CAP].sum() == 0 and (st[CAP] > 0).all() and (tr.final["env_i32"][6] == -1).all()   # every outcome, random row


def test_rollout_capacity_zero_pool_tallies_row_zero(trajectory):
    tr = trajectory(1, "RandomOpponent", cap=0, count=0)
    _check(tr)
    st = tr.final["pool_stats"]
    assert st.shape == (1, 3) and (st[0] > 0).all() and (tr.final["env_i32"][6] == -1).all()


def test_greedy_learner_matches_float64_argmax(trajectory):
    """deterministic bit 1: the learner takes the first max of its float64 probabilities (up to near-ties); the
    opponents still sample."""
    tr = trajectory(2, "RandomOpponent", deterministic=1)
    _check(tr)
    assert tr.final["pool_stats"].sum() > 0


@pytest.mark.parametrize("strategy", STRATEGIES)
@pytest.mark.parametrize("count", [0, 5, N_SNAPSHOTS])
def test_philox_reset_matches_replay(cuda, strategy, count):
    """orl_selfplay_reset without a start table: cells, step count, reset counter and opponent slot of every env."""
    import torch

    env, _ = _make_env(strategy, CAP, count, 1)
    nreset = np.random.default_rng(count).integers(0, 1 << 30, N)
    env.env_i32[5].copy_(torch.from_numpy(nreset.astype(np.int32)))
    obs, _ = env.reset(seed=SEED)
    z = np.zeros(N)
    rep = ref.SelfPlayReplay(z.reshape(-1, 1).repeat(4, 1), z, nreset, z, z, z, seed=SEED, row_offset=OFFSET, strategy=strategy,
                             pool_params=np.zeros((CAP, ref.param_count())), pool_count=count, activation_id=1)
    want_obs = rep.reset()
    assert np.array_equal(env.env_i32.cpu().numpy()[:7], rep.env_i32())
    assert np.array_equal(obs[:, 0, :], want_obs)
    if count and strategy == "RandomOpponent":
        assert set(rep.opp) == set(range(min(count, CAP)))


class _NextSlot(ref.SelfPlayReplay):
    def snapshot(self, slot):
        return self.pool_params[(slot + 1) % self.cap]


class _Unmirrored(ref.SelfPlayReplay):
    def opponent_obs(self, pos):
        return pos


class _LearnerWeights(ref.SelfPlayReplay):
    def snapshot(self, slot):
        return self.learner_params


class _Lanes01(ref.SelfPlayReplay):
    opponent_lanes = (0, 1)


class _Relu(ref.SelfPlayReplay):
    def opponent_activation(self):
        return 1


class _LocalResetKey(ref.SelfPlayReplay):
    def reset_key(self):
        return np.arange(self.N, dtype=np.int64)


class _TallySlot0(ref.SelfPlayReplay):
    def tally_slot(self, opp):
        return np.zeros_like(opp)


# the next ring slot, the unmirrored observation, the learner's weights for the opponent, opponent noise lanes 0 / 1, a
# ReLU opponent in a tanh run, the reset key with the local env index, every outcome tallied under slot 0
MUTANTS = {"next_slot": _NextSlot, "unmirrored_obs": _Unmirrored, "learner_weights": _LearnerWeights, "lanes_0_1": _Lanes01,
           "relu_opponent": _Relu, "local_reset_key": _LocalResetKey, "tally_slot_0": _TallySlot0}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_replay_mistakes_are_detected(trajectory, mutant):
    """Replaying test 1's tanh / RandomOpponent launch with one deliberate mistake: the comparison must fail.  Opponent
    near-ties are still resolved against the kernel, so every mismatch counted is at a step that is not a near-tie."""
    tr = trajectory(0, "RandomOpponent")
    rep, res = _replay(tr, MUTANTS[mutant])
    bad = ref.mismatches(rep, res, tr.kernel, tr.final)
    print(f"\n[selfplay mutant] {mutant}: {bad}")
    assert sum(bad.values()) > 0, bad


def test_step_api_opponent_plays_the_pools_activation(cuda):
    """env.step with a pool of tanh snapshots: the opponent's moves, rewards, dones and the tallies follow the replay
    with the pool's activation (and not ReLU's)."""
    n_envs, cap, n_steps = 2048, 4, 24
    env, _ = _make_env("RandomOpponent", cap, cap, 0, n_envs=n_envs)
    obs, _ = env.reset(seed=SEED)
    e = env.env_i32.cpu().numpy()
    z = np.zeros(n_envs)
    pool_params = env.opponent_pool.params.cpu().numpy()
    reps = [cls(e[:4].T, e[4], e[5], e[6], z, z, seed=SEED, row_offset=OFFSET, strategy="RandomOpponent", pool_params=pool_params,
                pool_count=cap, activation_id=0) for cls in (ref.SelfPlayReplay, _Relu)]
    counts = [0, 0]
    learner = np.zeros(ref.param_count())           # the step API scripts the learner: its parameters are unused
    rng = np.random.default_rng(3)
    ones = np.ones(n_envs, np.float32)
    for _ in range(n_steps):
        acts = rng.integers(0, ref.N_ACTIONS, n_envs)
        o, r, d, _ = env.step(acts.reshape(n_envs, 1, 1))
        kernel = dict(obs=np.stack([obs[:, 0], o[:, 0]]), rewards=r[None, :, 0, 0].astype(np.float32),
                      masks=np.stack([ones, (~d[:, 0]).astype(np.float32)]), active_masks=np.stack([ones, ones]), actions=acts[None])
        step_base = (1 << 40) + env._sp_steps      # the step API's noise key: one step per call above 2^40
        res = [rep.rollout(learner, 1, step_base, deterministic=2, kernel=kernel) for rep in reps]
        for i in range(2):
            counts[i] += sum(ref.mismatches(reps[i], res[i], kernel, check_learner=False).values())
        obs = o
    assert counts[0] == 0, counts
    final = dict(env_i32=env.env_i32.cpu().numpy(), ep_return=env.ep_return.cpu().numpy(), ep_length=env.ep_length.cpu().numpy(),
                 episode_stats=env.episode_stats.cpu().numpy(), pool_stats=env.opponent_pool.stats.cpu().numpy())
    bad = {k: v for k, v in ref.mismatches(reps[0], res[0], kernel, final, check_learner=False).items() if v}
    assert not bad, bad
    assert counts[1] > 0                            # a ReLU opponent would have moved differently
