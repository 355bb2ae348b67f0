"""Float64 host replay of the self-play rollout: `selfplay_rollout_kernel` and `selfplay_reset_kernel` of
csrc/orl_selfplay.cu.

TEST INFRASTRUCTURE, as rnn_ref64.py.  Vectorised over envs in numpy float64.  It restates
- the policy forward of the flat layout of orl_mlp.cuh (W1[64][4] b1 g1 be1 W3[64][64] b3 g3 be3 Wh[n][64] bh), the
  `mlp_base` order of oracle/nets.py, for all four activations;
- the Philox words: reset cells (counter (env_key, nreset, 0x53706c79, try)), the opponent pick (counter
  (env_key, nreset, 0x4f70706f, 0)), the action noise of (step, env_key): lanes 0 / 1 learner, 2 / 3 opponent policy,
  word 0 of lane 4 the random opponent;
- the game of oracle/selfplay.py (its `_move` and constants, vectorised through a move table);
- the bookkeeping: steps, nreset and opponent slot per env, episode return / length, episode_stats[0..2] and the
  pool's win / loss / draw tally per slot (last row: the random opponent).

The replay is teacher-forced on the learner: it takes the kernel's recorded learner actions and computes what the
float64 policy would have done, the float64 log-prob of the taken action, and the opponent's action itself.  At a
near-tie of the opponent's argmax(p / q) (top two float64 ratios within `TIE_RTOL`) the float32 kernel may pick
either action; the replay then keeps whichever candidate reproduces the kernel's step: the opponent's cell in
obs[t+1] while the episode goes on, the outcome in the reward when it ends.

The places a kernel could read the wrong thing are methods (`snapshot`, `opponent_obs`, `opponent_activation`,
`reset_key`, `tally_slot`) and one attribute (`opponent_lanes`), so a test can replay with a deliberate mistake and
check that the comparison notices it."""
import types

import numpy as np

import param_layout as layout
from oracle.selfplay import COLS, GOAL, MAX_STEPS, ROWS, _move
from helpers import philox4x32_10, philox_units

H = layout.H
N_ACTIONS = 5
LN_EPS = 1e-5
TIE_RTOL = 1e-5
RESET_TAG = 0x53706C79        # counter word 2 of the reset-cell draws
PICK_TAG = 0x4F70706F         # counter word 2 of the RandomOpponent draw
RESET_TRIES = 16
RESET_FALLBACK = (0, 0, 0, 2)
M32 = np.uint64(0xFFFFFFFF)

# _MOVE[x, y, a] = cell after action a from (x, y)
_MOVE = np.array([[[_move(x, y, a) for a in range(N_ACTIONS)] for y in range(COLS)] for x in range(ROWS)], np.int64)


def param_shapes(n=N_ACTIONS, d=4):
    """(state_dict name, shape) of the policy in the order of its flat parameter buffer (orl_mlp.cuh net_offsets)."""
    return layout.mlp_trunk(d) + layout.head(n, "categorical")


def param_count(n=N_ACTIONS, d=4):
    return sum(int(np.prod(s)) for _, s in param_shapes(n, d))


def unflatten(flat, n=N_ACTIONS, d=4):
    """{state_dict name: float64 array} of a flat parameter vector (longer vectors, e.g. padded pool rows, are cut)."""
    flat = np.asarray(flat, np.float64)
    out, off = {}, 0
    for name, shp in param_shapes(n, d):
        k = int(np.prod(shp))
        out[name] = flat[off:off + k].reshape(shp)
        off += k
    return out


def activation(z, activation_id):
    """orl_mlp.cuh act_fwd: tanh, ReLU, leaky ReLU (0.01), ELU (alpha 1)."""
    if activation_id == 0:
        return np.tanh(z)
    if activation_id == 1:
        return np.maximum(z, 0.0)
    if activation_id == 2:
        return np.where(z > 0, z, 0.01 * z)
    return np.where(z > 0, z, np.expm1(np.minimum(z, 0.0)))


def _layernorm(h, g, b):
    m = h.mean(-1, keepdims=True)
    v = ((h - m) ** 2).mean(-1, keepdims=True)
    return (h - m) / np.sqrt(v + LN_EPS) * g + b


def policy_logits(flat, obs, activation_id, n=N_ACTIONS):
    """(rows, n) float64 logits of the flat policy on (rows, 4) observations: fc1, activation, LayerNorm, fc3,
    LayerNorm, head."""
    p = unflatten(flat, n, obs.shape[-1])
    h = activation(obs @ p["base.mlp.fc1.0.weight"].T + p["base.mlp.fc1.0.bias"], activation_id)
    h = _layernorm(h, p["base.mlp.fc1.2.weight"], p["base.mlp.fc1.2.bias"])
    h = h @ p["base.mlp.fc3.0.weight"].T + p["base.mlp.fc3.0.bias"]
    h = _layernorm(h, p["base.mlp.fc3.1.weight"], p["base.mlp.fc3.1.bias"])
    return h @ p["act.action_out.linear.weight"].T + p["act.action_out.linear.bias"]


def log_softmax(x):
    m = x.max(-1, keepdims=True)
    return x - m - np.log(np.exp(x - m).sum(-1, keepdims=True))


def top_two(score):
    """First argmax of each row (the kernels' first-max rule), the runner-up, and whether the two are within TIE_RTOL."""
    order = np.argsort(-score, axis=-1, kind="stable")
    first, second = order[:, 0], order[:, 1]
    rows = np.arange(score.shape[0])
    best, next_ = score[rows, first], score[rows, second]
    return first, second, (best - next_) <= TIE_RTOL * best


def _u32_scaled(w, n):
    """(w * n) >> 32 of 32-bit words: a uniform integer in [0, n)."""
    return ((np.asarray(w, np.uint64) * np.uint64(n)) >> np.uint64(32)).astype(np.int64)


def reset_cells(env_key, nreset, seed):
    """sp_reset_cells without a table: (len, 4) start cells x0, y0, x1, y1 of the resets (env_key, nreset).  The first of
    16 Philox tries whose two cells are distinct and off the goal wins; (0, 0, 0, 2) when none is."""
    env_key, nreset = np.asarray(env_key, np.int64), np.asarray(nreset, np.int64)
    out = np.tile(np.asarray(RESET_FALLBACK, np.int64), (env_key.size, 1))
    found = np.zeros(env_key.size, bool)
    for it in range(RESET_TRIES):
        w = philox4x32_10(env_key, nreset, RESET_TAG, it, seed)
        c = np.stack([_u32_scaled(w[0], ROWS), _u32_scaled(w[1], COLS), _u32_scaled(w[2], ROWS), _u32_scaled(w[3], COLS)], -1)
        ok = (~found & ~((c[:, 0] == GOAL[0]) & (c[:, 1] == GOAL[1])) & ~((c[:, 2] == GOAL[0]) & (c[:, 3] == GOAL[1]))
              & ~((c[:, 0] == c[:, 2]) & (c[:, 1] == c[:, 3])))
        out[ok] = c[ok]
        found |= ok
    return out


def pick_opponent(strategy, count, cap, env_key, nreset, seed):
    """sp_pick_opponent: the ring slot of a new episode's opponent, -1 (random-action opponent) while the pool is empty.
    LastOpponent: the newest snapshot; RandomOpponent: uniform over the filled slots."""
    env_key, nreset = np.asarray(env_key, np.int64), np.asarray(nreset, np.int64)
    avail = min(count, cap)
    if avail <= 0:
        return np.full(env_key.size, -1, np.int64)
    if strategy == "LastOpponent":
        return np.full(env_key.size, (count - 1) % cap, np.int64)
    assert strategy == "RandomOpponent", strategy
    return _u32_scaled(philox4x32_10(env_key, nreset, PICK_TAG, 0, seed)[0], avail)


def game_step(pos, steps, act0, act1):
    """The rules of oracle.selfplay.GridWorld2P.step on all envs at once, before any reset: new cells (N, 4), rewards,
    dones, outcomes (0 win, 1 loss, 2 draw of the learner; -1 while the episode goes on) and step counts."""
    p0 = _MOVE[pos[:, 0], pos[:, 1], act0]
    p1 = _MOVE[pos[:, 2], pos[:, 3], act1]
    g0 = (p0[:, 0] == GOAL[0]) & (p0[:, 1] == GOAL[1])
    g1 = (p1[:, 0] == GOAL[0]) & (p1[:, 1] == GOAL[1])
    outcome = np.select([g0 & ~g1, g1 & ~g0, g0 & g1], [0, 1, 2], -1)
    reward = np.select([g0 & ~g1, g1 & ~g0, g0 & g1], [10.0, -10.0, 0.0], -1.0)
    timeout = (outcome < 0) & (steps == MAX_STEPS)
    reward[timeout] -= 10.0
    outcome[timeout] = 2
    done = outcome >= 0
    return np.concatenate([p0, p1], -1), reward, done, outcome, np.where(done, steps, steps + 1)


class SelfPlayReplay:
    """The device env state (env_i32 rows 0..6, ep_return, ep_length) and tallies, advanced by `rollout` as one
    selfplay_rollout_kernel launch advances them.  `pool_params` is (capacity, >= param_count) with ring slot s in
    row s; `table` (N, K, 4) replaces the Philox resets as the kernel's env_table does."""

    opponent_lanes = (2, 3)

    def __init__(self, pos, steps, nreset, opp, ep_return, ep_length, *, seed, row_offset, strategy, pool_params,
                 pool_count, activation_id, table=None, n=N_ACTIONS):
        self.pos = np.array(pos, np.int64).reshape(-1, 4)
        self.N = self.pos.shape[0]
        self.steps, self.nreset, self.opp = (np.array(v, np.int64).reshape(self.N) for v in (steps, nreset, opp))
        self.ep_return = np.array(ep_return, np.float64).reshape(self.N)
        self.ep_length = np.array(ep_length, np.int64).reshape(self.N)
        self.seed, self.row_offset, self.strategy, self.n = int(seed), int(row_offset), strategy, n
        self.pool_params = np.asarray(pool_params, np.float64)
        self.cap, self.count = self.pool_params.shape[0], int(pool_count)
        self.activation_id = activation_id
        self.table = None if table is None else np.asarray(table, np.int64)
        self.pool_stats = np.zeros((self.cap + 1, 3), np.int64)
        self.episode_stats = np.zeros(3, np.float64)
        self.opponent_near_ties = 0       # opponent steps at a near-tie of argmax(p / q)
        self.opponent_runner_up = 0       # ... of which the kernel's step is reproduced by the runner-up only

    # ---- what the kernel reads (tests override these to replay a deliberate mistake) ----
    def env_key(self):
        return np.arange(self.N, dtype=np.int64) + self.row_offset

    def reset_key(self):
        return self.env_key()

    def snapshot(self, slot):
        return self.pool_params[slot]

    def opponent_obs(self, pos):
        return pos[:, [2, 3, 0, 1]]

    def opponent_activation(self):
        return self.activation_id

    def tally_slot(self, opp):
        return np.where(opp >= 0, opp, self.cap)

    # ---- state ----
    def env_i32(self):
        """(7, N) rows 0..6 of the device's env_i32: x0, y0, x1, y1, steps, nreset, opponent slot."""
        return np.concatenate([self.pos.T, self.steps[None], self.nreset[None], self.opp[None]]).astype(np.int64)

    def _reset(self, idx):
        """Start cells of a new episode for envs `idx` (their nreset not yet bumped)."""
        if self.table is not None:
            k = np.minimum(self.nreset[idx], self.table.shape[1] - 1)
            return self.table[idx, k]
        return reset_cells(self.reset_key()[idx], self.nreset[idx], self.seed)

    def reset(self):
        """selfplay_reset_kernel: every env starts a new episode; returns the (N, 4) observations."""
        idx = np.arange(self.N)
        self.pos = self._reset(idx)
        self.opp = pick_opponent(self.strategy, self.count, self.cap, self.env_key(), self.nreset, self.seed)
        self.nreset = self.nreset + 1
        self.steps = np.zeros(self.N, np.int64)
        self.ep_return[:] = 0.0
        self.ep_length[:] = 0
        return self.pos.astype(np.float32)

    # ---- one launch ----
    def rollout(self, learner_params, T, step_base, deterministic=0, kernel=None, learner_actions=None, opponent_actions=None):
        """Steps t < T with Philox step step_base + t.  Learner actions: `kernel["actions"]` (teacher forcing), else
        `learner_actions` (scripted), else the float64 policy's own choice.  `kernel` (the recorded "obs", "rewards",
        "masks", "actions") also resolves opponent near-ties.  `opponent_actions` scripts the opponent (deterministic
        bit 4).  Returns the replay's obs (T+1, N, 4), rewards (T, N), masks (T+1, N) and, per (t, env), the float64
        learner choice `want`, whether that choice is a near-tie, and the float64 log-prob `lp` of the taken action."""
        N, n = self.N, self.n
        lanes = self.opponent_lanes
        q_l = -np.log(philox_units(T, N, self.seed, step_base, self.row_offset, (0, 1))[..., :n].astype(np.float64))
        q_o = -np.log(philox_units(T, N, self.seed, step_base, self.row_offset, lanes)[..., :n].astype(np.float64))
        step = np.uint64(step_base) + np.arange(T, dtype=np.uint64)[:, None]
        rand_act = _u32_scaled(philox4x32_10(step & M32, step >> np.uint64(32), self.env_key()[None, :], 4, self.seed)[0], n)
        self.learner_params = np.asarray(learner_params, np.float64)
        obs = np.zeros((T + 1, N, 4), np.float32)
        obs[0] = self.pos
        rewards = np.zeros((T, N), np.float32)
        masks = np.ones((T + 1, N), np.float32)
        want = np.zeros((T, N), np.int64)
        tie = np.zeros((T, N), bool)
        lp = np.zeros((T, N), np.float64)
        rows = np.arange(N)
        for t in range(T):
            nl = log_softmax(policy_logits(self.learner_params, self.pos.astype(np.float64), self.activation_id, n))
            score = np.exp(nl) if deterministic & 1 else np.exp(nl) / q_l[t]
            want[t], _, tie[t] = top_two(score)
            if kernel is not None:
                a0 = np.asarray(kernel["actions"][t]).astype(np.int64)
            elif learner_actions is not None:
                a0 = np.asarray(learner_actions[t]).astype(np.int64)
            else:
                a0 = want[t]
            lp[t] = nl[rows, a0]
            otie = np.zeros(N, bool)
            if opponent_actions is not None:
                a1 = np.asarray(opponent_actions[t]).astype(np.int64)
                alt = a1
            else:
                a1, alt = rand_act[t].copy(), rand_act[t].copy()
                for slot in np.unique(self.opp[self.opp >= 0]):
                    idx = np.nonzero(self.opp == slot)[0]
                    lo = log_softmax(policy_logits(self.snapshot(slot), self.opponent_obs(self.pos[idx]).astype(np.float64),
                                                   self.opponent_activation(), n))
                    a1[idx], alt[idx], otie[idx] = top_two(np.exp(lo) / q_o[t, idx])
            pos1, rew, done, outcome, steps1 = game_step(self.pos, self.steps, a0, a1)
            self.opponent_near_ties += int(otie.sum())
            if kernel is not None and otie.any():
                k_obs, k_rew, k_done = kernel["obs"][t + 1], kernel["rewards"][t], kernel["masks"][t + 1] == 0
                same = lambda p, r, d: (r == k_rew) & (d == k_done) & (d | (p == k_obs).all(-1))   # noqa: E731
                pos2, rew2, done2, out2, steps2 = game_step(self.pos, self.steps, a0, alt)
                use = otie & ~same(pos1, rew, done) & same(pos2, rew2, done2)
                pos1[use], rew[use], done[use], outcome[use], steps1[use] = pos2[use], rew2[use], done2[use], out2[use], steps2[use]
                self.opponent_runner_up += int(use.sum())
            self.ep_return += rew
            self.ep_length += 1
            d = np.nonzero(done)[0]
            if d.size:
                np.add.at(self.pool_stats, (self.tally_slot(self.opp[d]), outcome[d]), 1)
                self.episode_stats += [self.ep_return[d].sum(), self.ep_length[d].sum(), d.size]
                self.ep_return[d] = 0.0
                self.ep_length[d] = 0
                pos1[d] = self._reset(d)
                self.opp[d] = pick_opponent(self.strategy, self.count, self.cap, self.env_key()[d], self.nreset[d], self.seed)
                self.nreset[d] += 1
                steps1[d] = 0
            self.pos, self.steps = pos1, steps1
            obs[t + 1] = pos1
            rewards[t] = rew
            masks[t + 1] = ~done
        return types.SimpleNamespace(obs=obs, rewards=rewards, masks=masks, want=want, tie=tie, lp=lp)


def mismatches(replay, res, kernel, final=None, check_learner=True):
    """{what: number of entries where the kernel differs from the replay}.  Per (t, env): obs, rewards, masks,
    active_masks and (unless scripted) learner actions that are neither the float64 choice nor at a near-tie.  With
    `final` (the device's env_i32, ep_return, ep_length, episode_stats, pool_stats after the launch) also the state and
    the tallies."""
    out = dict(obs=int((kernel["obs"][1:] != res.obs[1:]).any(-1).sum()),
               rewards=int((kernel["rewards"] != res.rewards).sum()),
               masks=int((kernel["masks"][1:] != res.masks[1:]).sum()),
               active_masks=int((kernel["active_masks"][1:] != 1.0).sum()))
    if check_learner:
        out["learner_actions"] = int(((kernel["actions"].astype(np.int64) != res.want) & ~res.tie).sum())
    if final is not None:
        out["env_i32"] = int((final["env_i32"][:7] != replay.env_i32()).sum())
        out["ep_return"] = int((final["ep_return"] != replay.ep_return.astype(np.float32)).sum())
        out["ep_length"] = int((final["ep_length"] != replay.ep_length).sum())
        out["episode_stats"] = int((final["episode_stats"][:3] != replay.episode_stats).sum())
        out["pool_stats"] = int((final["pool_stats"] != replay.pool_stats).sum())
    return out
