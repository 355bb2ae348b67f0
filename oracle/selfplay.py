"""Oracle: the two-player GridWorld of the device self-play path (csrc/orl_selfplay.cu) restated in numpy.

TEST INFRASTRUCTURE.  The reference ships no 2-player GridWorld (SURVEY.md §8f-2: "define the 2-player GridWorld
(new env — document rules; no reference parity possible)"); the rules extend the reference's single-player
`GridWorldEnv` (openrl/envs/gridworld/gridworld_env.py:21-86: 10x10 grid, goal (1, 1), actions {stay, x-1, x+1, y-1,
y+1}, -1 per step, +10 on the goal, -10 extra on the 100-step time-out) to two simultaneous movers:

  * exactly one player on the goal after the move: it wins; the learner (player 0) gets +10 / -10, episode ends;
  * both on the goal: draw, reward 0, episode ends;
  * otherwise reward -1; when the episode has already taken 100 steps it ends as a draw with reward -1 - 10;
  * on episode end both players restart from the next entry of the start-cell table.

The opponent-selection rules (RandomOpponent / LastOpponent, openrl/selfplay/sample_strategy/*.py), the Philox start
cells and the policy-driven opponent are restated by the float64 replay of the whole rollout, tests/selfplay_ref64.py
(`pick_opponent`, `reset_cells`, `SelfPlayReplay`), which takes its game rules from `_move` and the constants here."""
import numpy as np

ROWS = COLS = 10
GOAL = (1, 1)
MAX_STEPS = 100


def _move(x, y, a):
    if a == 1:
        x -= 1
    elif a == 2:
        x += 1
    elif a == 3:
        y -= 1
    elif a == 4:
        y += 1
    return min(max(x, 0), ROWS - 1), min(max(y, 0), COLS - 1)


class GridWorld2P:
    """N envs stepped with scripted actions; start cells from `table` (N, K, 4) in reset order."""

    def __init__(self, table):
        self.table = np.asarray(table, np.int64)
        self.N, self.K = self.table.shape[:2]
        self.nreset = np.zeros(self.N, np.int64)
        self.pos = np.zeros((self.N, 4), np.int64)
        self.steps = np.zeros(self.N, np.int64)
        self.outcomes = np.zeros(3, np.int64)     # wins, losses, draws of player 0

    def _reset_env(self, e):
        self.pos[e] = self.table[e, min(self.nreset[e], self.K - 1)]
        self.nreset[e] += 1
        self.steps[e] = 0

    def reset(self):
        for e in range(self.N):
            self._reset_env(e)
        return self.pos.astype(np.float32).copy()

    def step(self, act0, act1):
        rewards = np.zeros(self.N, np.float32)
        dones = np.zeros(self.N, bool)
        for e in range(self.N):
            x0, y0, x1, y1 = self.pos[e]
            x0, y0 = _move(x0, y0, int(act0[e]))
            x1, y1 = _move(x1, y1, int(act1[e]))
            g0, g1 = (x0, y0) == GOAL, (x1, y1) == GOAL
            done, outcome = False, -1
            if g0 and not g1:
                r, done, outcome = 10.0, True, 0
            elif g1 and not g0:
                r, done, outcome = -10.0, True, 1
            elif g0 and g1:
                r, done, outcome = 0.0, True, 2
            else:
                r = -1.0
            if not done:
                if self.steps[e] == MAX_STEPS:
                    done, outcome = True, 2
                    r -= 10.0
                else:
                    self.steps[e] += 1
            self.pos[e] = (x0, y0, x1, y1)
            rewards[e], dones[e] = r, done
            if done:
                self.outcomes[outcome] += 1
                self._reset_env(e)
        return self.pos.astype(np.float32).copy(), rewards, dones
