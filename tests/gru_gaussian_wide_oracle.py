"""GRU policies with DiagGaussian heads of 9..64 dimensions (cfg.use_wide_recurrent_gaussian_head): the envs of the two
traces and their registration with the recurrent Gaussian oracle loop.

TEST INFRASTRUCTURE.  The oracle maths (tests/gru_gaussian_oracle.py: policy_act_gaussian, policy_eval_gaussian,
ppo_update, GRUGaussianTrainer) takes any head width; what is bounded there is its table of envs, VECS.  This module adds
the two envs of the wide traces to that table under their own tags:

  gru_gaussian_wide_21          dm_control humanoid's shapes: tests/wide_gaussian_oracle.py's wide_gaussian_env(67, 21)
                                (Box(67) observations, Box(21)), one agent
  gru_gaussian_wide_spread_64   SpreadBox64Env: SpreadBoxEnv's three agents, Dict {"policy": Box(18), "critic": Box(54)}
                                and agents that finish at different steps, with Box(64) actions

Both are pinned to the unmodified reference by tests/test_gru_gaussian_wide_oracle.py (traces
tests/golden/trace_gru_gaussian_wide_{21,spread_64}.npz, recorded by tools/gen_golden_gru_gaussian_wide.py)."""
import numpy as np

import gru_gaussian_oracle as ggo
from gru_gaussian_oracle import SpreadBoxEnv, SpreadBoxVec
from wide_gaussian_oracle import spaced_wide_gaussian_env, wide_gaussian_vec

WIDE_21 = (67, 21)   # (observation features, action dimensions) of trace_gru_gaussian_wide_21


class SpreadBox64Env(SpreadBoxEnv):
    """SpreadBoxEnv with Box(64) actions: dimension j of agent i targets its feature j % 18, and agent i is rewarded by
    1 - mean |target - clip(a, 0, 1)| over the 64 dimensions (float64).  Observations, dones and the episode's end are
    SpreadBoxEnv's."""
    act_dim = 64

    def step(self, action):
        a = np.asarray(action, dtype=np.float32).reshape(self.agent_num, -1)[:, :self.act_dim].astype(np.float64)
        done_before = np.arange(self.agent_num) + 3 <= self.steps
        target = self.state[:, np.arange(self.act_dim) % self.obs_dim].astype(np.float64)
        reward = 1.0 - np.abs(target - np.clip(a, 0.0, 1.0)).mean(-1)
        reward[done_before] = 0.0
        self.steps += 1
        self._draw()
        dones = np.arange(self.agent_num) + 3 <= self.steps
        return self._obs(), reward[:, None], dones, {}


class SpacedSpreadBox64Env(SpreadBox64Env):
    """SpreadBox64Env with the spaces a host vec-env reads (make(..., make_custom_envs=...))."""

    def __init__(self):
        from openrl_b200 import spaces

        super().__init__()
        box = lambda w: spaces.Box(-np.inf, np.inf, (w,), np.float32)  # noqa: E731
        self.observation_space = spaces.Dict({"policy": box(self.obs_dim), "critic": box(self.critic_obs_dim)})
        self.action_space = spaces.Box(-1.0, 1.0, (self.act_dim,), np.float32)


class SpreadBox64Vec(SpreadBoxVec):
    """SpreadBox64Env under SyncVectorEnv (SpreadBoxVec's seeds and auto-reset)."""
    act_dim = n_actions = SpreadBox64Env.act_dim

    def __init__(self, env_num):
        self.N = env_num
        self.envs = [SpreadBox64Env() for _ in range(env_num)]


def _wide_21_vec(env_num):
    v = wide_gaussian_vec(*WIDE_21)(env_num)
    v.n_actions = v.act_dim
    return v


# the host env class a PPOAgent test builds for each tag
SPACED = {"gru_gaussian_wide_21": spaced_wide_gaussian_env(*WIDE_21), "gru_gaussian_wide_spread_64": SpacedSpreadBox64Env}
ggo.VECS.update({"gru_gaussian_wide_21": _wide_21_vec, "gru_gaussian_wide_spread_64": SpreadBox64Vec})
