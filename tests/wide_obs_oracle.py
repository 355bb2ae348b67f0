"""Observations of 65..256 features: two envs of the shapes the wide-observation path is built for, and the oracle loops
on them.

TEST INFRASTRUCTURE.  `WideDictTargetEnv` is DictTargetEnv (tests/dict_obs_oracle.py) at SMAC 8m's shapes: a Dict
{"policy": Box(80), "critic": Box(168)} observation and Discrete(14).  `WideBoxTargetEnv` has a flat Box(256)
observation and a Box(4) action (a DiagGaussian head).  Their SyncVectorEnv forms and the oracle trainers on them are
pinned to the unmodified reference by tests/test_wide_obs_oracle.py (traces tests/golden/trace_wide_obs_{dict,box_256}.npz,
recorded by tools/gen_golden_wide_obs.py)."""
import numpy as np

from dict_obs_oracle import DictObsMATrainer, DictTargetEnv, DictTargetVec
from oracle import envs as oenvs
from oracle import loop


class WideDictTargetEnv(DictTargetEnv):
    """State: 168 features in [0, 1) drawn every step, whose first 14 are the payoffs of the 14 actions and whose last is
    the elapsed fraction of the episode.  The policy sees the first 80 features (a partial view: the payoffs and 66
    more), the critic all 168.  Reward: the payoff of the chosen action; episodes last HORIZON steps."""
    obs_dim = 80
    critic_obs_dim = 168
    n_actions = 14

    def _draw(self):
        self.state = self.rng.random(self.critic_obs_dim).astype(np.float32)
        self.payoff = self.state[:self.n_actions]

    def _obs(self):
        c = self.state.copy()
        c[-1] = self.steps / self.HORIZON
        return {"policy": c[:self.obs_dim].copy(), "critic": c}


class SpacedWideDictTargetEnv(WideDictTargetEnv):
    """WideDictTargetEnv with the spaces a host vec-env reads (make(..., make_custom_envs=...) -> SyncHostVecEnv)."""

    def __init__(self):
        from openrl_b200 import spaces

        super().__init__()
        box = lambda w: spaces.Box(-np.inf, np.inf, (w,), np.float32)  # noqa: E731
        self.observation_space = spaces.Dict({"policy": box(self.obs_dim), "critic": box(self.critic_obs_dim)})
        self.action_space = spaces.Discrete(self.n_actions)


class WideDictTargetVec(DictTargetVec):
    """WideDictTargetEnv under SyncVectorEnv: obs {"policy": (N,1,80), "critic": (N,1,168)}."""
    obs_dim = WideDictTargetEnv.obs_dim
    critic_obs_dim = WideDictTargetEnv.critic_obs_dim
    n_actions = WideDictTargetEnv.n_actions

    def __init__(self, env_num):
        super().__init__(env_num)
        self.envs = [WideDictTargetEnv() for _ in range(env_num)]


class WideDictObsTrainer(DictObsMATrainer):
    """Feed-forward or recurrent PPO (oracle/loop_ma.MATrainer) on WideDictTargetVec."""

    def __init__(self, cfg, env_num):
        saved = oenvs.ENVS.get("DictTarget")
        oenvs.ENVS["DictTarget"] = WideDictTargetVec
        try:
            super(DictObsMATrainer, self).__init__(cfg, "DictTarget", env_num)
        finally:
            if saved is None:
                del oenvs.ENVS["DictTarget"]
            else:
                oenvs.ENVS["DictTarget"] = saved


class WideBoxTargetEnv:
    """An observation of 256 features in [0, 1) drawn every step; Box(4) actions, rewarded by 1 - mean |target - clip(a,
    0, 1)| with the target the first 4 features, computed before the next draw (float64); episodes last HORIZON steps.
    4-tuple step."""
    obs_dim = 256
    act_dim = 4
    agent_num = 1
    HORIZON = 5

    def __init__(self):
        self.rng = oenvs.pcg64_np_random(None)
        self.steps = 0
        self._draw()

    def _draw(self):
        self.obs = self.rng.random(self.obs_dim).astype(np.float32)

    def reset(self, seed=None, options=None):
        if seed is not None:
            self.rng = oenvs.pcg64_np_random(seed)
        self.steps = 0
        self._draw()
        return self.obs.copy(), {}

    def step(self, action):
        a = np.asarray(action, dtype=np.float32).reshape(-1)[:self.act_dim].astype(np.float64)
        target = self.obs[:self.act_dim].astype(np.float64)
        reward = float(1.0 - np.abs(target - np.clip(a, 0.0, 1.0)).mean())
        self.steps += 1
        self._draw()
        return self.obs.copy(), reward, self.steps >= self.HORIZON, {}


class SpacedWideBoxTargetEnv(WideBoxTargetEnv):
    """WideBoxTargetEnv with the spaces a host vec-env reads."""

    def __init__(self):
        from openrl_b200 import spaces

        super().__init__()
        self.observation_space = spaces.Box(-np.inf, np.inf, (self.obs_dim,), np.float32)
        self.action_space = spaces.Box(-1.0, 1.0, (self.act_dim,), np.float32)


class WideBoxTargetVec:
    """WideBoxTargetEnv under SyncVectorEnv (seeds seed + i*10086, auto-reset): obs (N,1,256), rewards (N,1,1) f64,
    dones (N,1) bool."""
    obs_dim = WideBoxTargetEnv.obs_dim
    act_dim = WideBoxTargetEnv.act_dim
    agent_num = 1

    def __init__(self, env_num):
        self.N = env_num
        self.envs = [WideBoxTargetEnv() for _ in range(env_num)]

    def reset(self, seed=None):
        return np.stack([e.reset(seed=None if seed is None else seed + i * 10086)[0] for i, e in enumerate(self.envs)])[:, None, :]

    def step(self, actions):
        obs = np.zeros((self.N, 1, self.obs_dim), np.float32)
        rewards = np.zeros((self.N, 1, 1), np.float64)
        dones = np.zeros((self.N, 1), bool)
        for i, e in enumerate(self.envs):
            o, r, d, _ = e.step(actions[i, 0])
            if d:
                o, _ = e.reset()
            obs[i, 0], rewards[i, 0, 0], dones[i, 0] = o, r, d
        return obs, rewards, dones, [{} for _ in range(self.N)]


class WideBoxTrainer(loop.Trainer):
    """Feed-forward PPO with a DiagGaussian head (oracle/loop.Trainer) on WideBoxTargetVec."""

    def __init__(self, cfg, env_num):
        super().__init__(cfg, "WideBoxTarget", env_num, env=WideBoxTargetVec(env_num))
