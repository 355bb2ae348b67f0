"""Observations of 65..256 features with a GRU policy and critic: two envs, and the recurrent oracle loop on them.

TEST INFRASTRUCTURE.  `MaskedWideDictTargetEnv` is WideDictTargetEnv (tests/wide_obs_oracle.py: SMAC 8m's shapes, a Dict
{"policy": Box(80), "critic": Box(168)} observation and Discrete(14)) that also reports legal-move masks in
`info["action_masks"]`.  `WideBoxDiscreteEnv` has a flat Box(256) observation and Discrete(5).  Their SyncVectorEnv forms
and the oracle trainers on them (oracle/loop_ma.MATrainer, recurrent when cfg asks for it, with the reference's mask
ingest of tests/masked_oracle.py) are pinned to the unmodified reference by tests/test_wide_obs_gru_oracle.py (traces
tests/golden/trace_wide_obs_gru_{dict,box_256}.npz, recorded by tools/gen_golden_wide_obs_gru.py)."""
import numpy as np

from dict_obs_oracle import DictObsMATrainer
from masked_oracle import _MaskIngest
from oracle import envs as oenvs
from oracle import loop_ma
from wide_obs_oracle import WideDictTargetEnv, WideDictTargetVec


class MaskedWideDictTargetEnv(WideDictTargetEnv):
    """WideDictTargetEnv whose info carries, on reset and every step, the legal moves of the next observation: a random
    subset of the 14 actions (each legal with probability 0.5) that always holds the best payoff's action."""

    def _draw(self):
        super()._draw()
        m = (self.rng.random(self.n_actions) < 0.5).astype(np.int8)
        m[int(np.argmax(self.payoff))] = 1
        self.mask = m

    def reset(self, seed=None, options=None):
        obs, _ = super().reset(seed=seed, options=options)
        return obs, {"action_masks": self.mask.copy()}

    def step(self, action):
        obs, reward, done, _ = super().step(action)
        return obs, reward, done, {"action_masks": self.mask.copy()}


class SpacedMaskedWideDictTargetEnv(MaskedWideDictTargetEnv):
    """MaskedWideDictTargetEnv with the spaces a host vec-env reads (make(..., make_custom_envs=...) -> SyncHostVecEnv)."""

    def __init__(self):
        from openrl_b200 import spaces

        super().__init__()
        box = lambda w: spaces.Box(-np.inf, np.inf, (w,), np.float32)  # noqa: E731
        self.observation_space = spaces.Dict({"policy": box(self.obs_dim), "critic": box(self.critic_obs_dim)})
        self.action_space = spaces.Discrete(self.n_actions)


class MaskedWideDictTargetVec(WideDictTargetVec):
    """MaskedWideDictTargetEnv under SyncVectorEnv; the reset infos in `last_infos`."""

    def __init__(self, env_num):
        super().__init__(env_num)
        self.envs = [MaskedWideDictTargetEnv() for _ in range(env_num)]
        self.last_infos = None

    def reset(self, seed=None):
        out = [e.reset(seed=None if seed is None else seed + i * 10086) for i, e in enumerate(self.envs)]
        self.last_infos = [info for _, info in out]
        return self._stack([o for o, _ in out])


class WideDictGRUTrainer(_MaskIngest, DictObsMATrainer):
    """PPO (oracle/loop_ma.MATrainer, recurrent per cfg) on MaskedWideDictTargetVec, with the reference's mask ingest."""

    def __init__(self, cfg, env_num):
        saved = oenvs.ENVS.get("DictTarget")
        oenvs.ENVS["DictTarget"] = MaskedWideDictTargetVec
        try:
            super(DictObsMATrainer, self).__init__(cfg, "DictTarget", env_num)
        finally:
            if saved is None:
                del oenvs.ENVS["DictTarget"]
            else:
                oenvs.ENVS["DictTarget"] = saved
        self._ingest_masks(self.A)


class WideBoxDiscreteEnv:
    """An observation of 256 features in [0, 1) drawn every step; Discrete(5), rewarded by the feature of the chosen
    action in the observation it was chosen on; episodes last HORIZON steps.  4-tuple step."""
    obs_dim = 256
    n_actions = 5
    agent_num = 1
    HORIZON = 5

    def __init__(self):
        self.rng = oenvs.pcg64_np_random(None)
        self.steps = 0
        self._draw()

    def _draw(self):
        self.state = self.rng.random(self.obs_dim).astype(np.float32)

    def reset(self, seed=None, options=None):
        if seed is not None:
            self.rng = oenvs.pcg64_np_random(seed)
        self.steps = 0
        self._draw()
        return self.state.copy(), {}

    def step(self, action):
        a = int(np.asarray(action).reshape(-1)[0])
        reward = float(self.state[a])
        self.steps += 1
        self._draw()
        return self.state.copy(), reward, self.steps >= self.HORIZON, {}


class SpacedWideBoxDiscreteEnv(WideBoxDiscreteEnv):
    """WideBoxDiscreteEnv with the spaces a host vec-env reads."""

    def __init__(self):
        from openrl_b200 import spaces

        super().__init__()
        self.observation_space = spaces.Box(-np.inf, np.inf, (self.obs_dim,), np.float32)
        self.action_space = spaces.Discrete(self.n_actions)


class WideBoxDiscreteVec:
    """WideBoxDiscreteEnv under SyncVectorEnv (seeds seed + i*10086, auto-reset): obs (N,1,256), rewards (N,1,1) f64,
    dones (N,1) bool, infos."""
    obs_dim = WideBoxDiscreteEnv.obs_dim
    n_actions = WideBoxDiscreteEnv.n_actions
    agent_num = 1

    def __init__(self, env_num):
        self.N = env_num
        self.envs = [WideBoxDiscreteEnv() for _ in range(env_num)]

    def reset(self, seed=None):
        return np.stack([e.reset(seed=None if seed is None else seed + i * 10086)[0] for i, e in enumerate(self.envs)])[:, None, :]

    def step(self, actions):
        obs = np.zeros((self.N, 1, self.obs_dim), np.float32)
        rewards = np.zeros((self.N, 1, 1), np.float64)
        dones = np.zeros((self.N, 1), bool)
        infos = []
        for i, e in enumerate(self.envs):
            o, r, d, info = e.step(actions[i, 0])
            if d:
                o, info = e.reset()
            obs[i, 0], rewards[i, 0, 0], dones[i, 0] = o, r, d
            infos.append(info)
        return obs, rewards, dones, infos


class WideBoxGRUTrainer(loop_ma.MATrainer):
    """PPO (oracle/loop_ma.MATrainer, recurrent per cfg) on WideBoxDiscreteVec."""

    def __init__(self, cfg, env_num):
        saved = oenvs.ENVS.get("WideBoxDiscrete")
        oenvs.ENVS["WideBoxDiscrete"] = WideBoxDiscreteVec
        try:
            super().__init__(cfg, "WideBoxDiscrete", env_num)
        finally:
            if saved is None:
                del oenvs.ENVS["WideBoxDiscrete"]
            else:
                oenvs.ENVS["WideBoxDiscrete"] = saved
