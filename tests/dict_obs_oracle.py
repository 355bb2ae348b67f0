"""Oracle for host envs whose observation space is Dict {"policy", "critic"}: the critic reads its own observation.

TEST INFRASTRUCTURE: a small env of our own (numpy only) whose policy sees part of the state and whose critic sees all
of it, its vectorised form with the reference's SyncVectorEnv semantics, and the oracle loop (oracle/loop_ma.MATrainer,
which splits Dict observations into policy_obs / critic_obs) on it.  Pinned to the unmodified reference by
tests/test_dict_obs_oracle.py (traces tests/golden/trace_dict_obs_*.npz, recorded by tools/gen_golden_dict_obs.py).
Follows, in the reference,
  get_policy_obs / get_critic_obs       openrl/buffers/utils/util.py:22-55 (the buffer keeps both at their own widths)
  SyncVectorEnv concatenate of a Dict   openrl/envs/vec_env/utils/numpy_utils.py:127-135 (one stacked array per key)
  SyncVectorEnv auto-reset              openrl/envs/vec_env/sync_venv.py:219-227
"""
import numpy as np

from oracle import envs as oenvs
from oracle import loop_ma


class DictTargetEnv:
    """State: four payoffs in [0, 1), one per action, and the elapsed fraction of the episode.  The policy sees the
    first three payoffs (a partial view: the fourth action's payoff is hidden); the critic sees the full state, the four
    payoffs, the elapsed fraction, their mean and their maximum.  Reward: the payoff of the chosen action; new payoffs
    every step; episodes last HORIZON steps.  4-tuple step (the reference's Single2MultiAgentWrapper and SyncVectorEnv
    take it as is)."""
    obs_dim = 3
    critic_obs_dim = 7
    n_actions = 4
    agent_num = 1
    HORIZON = 5

    def __init__(self):
        self.rng = oenvs.pcg64_np_random(None)
        self.steps = 0
        self._draw()

    def _draw(self):
        self.payoff = self.rng.random(self.n_actions).astype(np.float32)

    def _obs(self):
        p = self.payoff
        critic = np.concatenate([p, [self.steps / self.HORIZON, p.mean(), p.max()]]).astype(np.float32)
        return {"policy": p[:self.obs_dim].copy(), "critic": critic}

    def reset(self, seed=None, options=None):
        if seed is not None:
            self.rng = oenvs.pcg64_np_random(seed)
        self.steps = 0
        self._draw()
        return self._obs(), {}

    def step(self, action):
        a = int(np.asarray(action).reshape(-1)[0])
        reward = float(self.payoff[a])
        self.steps += 1
        self._draw()
        return self._obs(), reward, self.steps >= self.HORIZON, {}


class SpacedDictTargetEnv(DictTargetEnv):
    """DictTargetEnv with the spaces a host vec-env reads (make(..., make_custom_envs=...) -> SyncHostVecEnv)."""

    def __init__(self):
        from openrl_b200 import spaces

        super().__init__()
        box = lambda w: spaces.Box(-np.inf, np.inf, (w,), np.float32)  # noqa: E731
        self.observation_space = spaces.Dict({"policy": box(self.obs_dim), "critic": box(self.critic_obs_dim)})
        self.action_space = spaces.Discrete(self.n_actions)


class DictTargetVec:
    """DictTargetEnv under SyncVectorEnv (sync_venv.py:129-247): seeds seed + i*10086, auto-reset.  reset -> obs
    {"policy": (N,1,3), "critic": (N,1,7)}; step -> that obs, rewards (N,1,1) f64, dones (N,1) bool, infos."""
    obs_dim = DictTargetEnv.obs_dim
    critic_obs_dim = DictTargetEnv.critic_obs_dim
    n_actions = DictTargetEnv.n_actions
    agent_num = 1

    def __init__(self, env_num):
        self.N = env_num
        self.envs = [DictTargetEnv() for _ in range(env_num)]

    @staticmethod
    def _stack(obs):
        return {k: np.stack([o[k] for o in obs])[:, None, :] for k in ("policy", "critic")}

    def reset(self, seed=None):
        return self._stack([e.reset(seed=None if seed is None else seed + i * 10086)[0] for i, e in enumerate(self.envs)])

    def step(self, actions):
        obs, infos = [], []
        rewards = np.zeros((self.N, 1, 1), np.float64)
        dones = np.zeros((self.N, 1), bool)
        for i, e in enumerate(self.envs):
            o, r, d, info = e.step(actions[i, 0])
            if d:
                o, info = e.reset()
            obs.append(o)
            infos.append(info)
            rewards[i, 0, 0], dones[i, 0] = r, d
        return self._stack(obs), rewards, dones, infos


class DictObsMATrainer(loop_ma.MATrainer):
    """PPO, feed-forward or recurrent (oracle/loop_ma.MATrainer), on DictTargetVec: policy_obs (T+1, N, 1, 3) and
    critic_obs (T+1, N, 1, 7)."""

    def __init__(self, cfg, env_num):
        saved = oenvs.ENVS.get("DictTarget")
        oenvs.ENVS["DictTarget"] = DictTargetVec
        try:
            super().__init__(cfg, "DictTarget", env_num)
        finally:
            if saved is None:
                del oenvs.ENVS["DictTarget"]
            else:
                oenvs.ENVS["DictTarget"] = saved
