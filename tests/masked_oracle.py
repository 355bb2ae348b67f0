"""Oracle for legal-move action masks reported by host envs (`info["action_masks"]`).

TEST INFRASTRUCTURE: a small masked env of our own (numpy only), its vectorised form with the reference's SyncVectorEnv
semantics, and the oracle loops (oracle/loop.Trainer, oracle/loop_ma.MATrainer) with the reference's mask ingest.
Pinned to the unmodified reference by tests/test_masked_oracle.py (traces tests/golden/trace_masked_*.npz, recorded by
tools/gen_golden_masked.py).  Follows, in the reference,
  prepare_action_masks                  openrl/envs/vec_env/utils/util.py:54-88 ((n,) or (A, n) per env; None when any
                                        env's info lacks the key; cast to int8)
  reset_and_buffer_init / init_buffer   openrl/drivers/rl_driver.py:118-131, buffers/replay_data.py:286-298 (slot 0)
  add2buffer / insert                   openrl/drivers/onpolicy_driver.py:114-116, buffers/replay_data.py:282-283 (slot
                                        t+1 only when masks are present: otherwise it keeps what it held)
  SyncVectorEnv auto-reset              openrl/envs/vec_env/sync_venv.py:219-227 (the info of a finished env is the
                                        reset info)
"""
import numpy as np

from oracle import envs as oenvs
from oracle import loop, loop_ma


def action_masks_from_infos(infos, agent_num=1):
    """prepare_action_masks: int8 (N, A, n), or None when any env's info lacks `action_masks`."""
    out = []
    for info in infos:
        if info is None or "action_masks" not in info:
            return None
        m = np.asarray(info["action_masks"])
        out.append([m[a] if m.ndim == 2 else m for a in range(agent_num)])
    return np.array(out, dtype=np.int8)


class MaskedTargetEnv:
    """Observation: one-hot of a target action out of 5.  `info["action_masks"]` (reset and every step, for the next
    observation): a random legal subset that always contains the target.  Reward 1 for the target, 0 for another legal
    move, -1 for an illegal one; episodes last HORIZON steps.  4-tuple step (the reference's Single2MultiAgentWrapper
    and SyncVectorEnv take it as is)."""
    obs_dim = 5
    n_actions = 5
    agent_num = 1
    HORIZON = 5

    def __init__(self):
        self.rng = oenvs.pcg64_np_random(None)
        self.steps = 0
        self._draw()

    def _draw(self):
        self.target = int(self.rng.integers(self.n_actions))
        m = (self.rng.random(self.n_actions) < 0.5).astype(np.int8)
        m[self.target] = 1
        self.mask = m

    def _obs(self):
        o = np.zeros(self.obs_dim, np.float32)
        o[self.target] = 1.0
        return o

    def reset(self, seed=None, options=None):
        if seed is not None:
            self.rng = oenvs.pcg64_np_random(seed)
        self.steps = 0
        self._draw()
        return self._obs(), {"action_masks": self.mask.copy()}

    def step(self, action):
        a = int(np.asarray(action).reshape(-1)[0])
        reward = 1.0 if a == self.target else (0.0 if self.mask[a] else -1.0)
        self.steps += 1
        self._draw()
        return self._obs(), reward, self.steps >= self.HORIZON, {"action_masks": self.mask.copy()}


class MaskedTargetVec:
    """MaskedTargetEnv under SyncVectorEnv (sync_venv.py:129-247): seeds seed + i*10086, auto-reset whose info is the
    reset info.  reset -> obs (N,1,5) (its infos in `last_infos`); step -> obs (N,1,5), rewards (N,1,1) f64,
    dones (N,1) bool, infos.  `report(i, t)` (env i, its t-th step call) decides whether env i's info carries masks."""
    obs_dim = MaskedTargetEnv.obs_dim
    n_actions = MaskedTargetEnv.n_actions
    agent_num = 1

    def __init__(self, env_num, report=None):
        self.N = env_num
        self.envs = [MaskedTargetEnv() for _ in range(env_num)]
        self.report = report
        self.calls = 0
        self.last_infos = None

    def _info(self, i, info):
        return info if self.report is None or self.report(i, self.calls) else {}

    def reset(self, seed=None):
        out = [e.reset(seed=None if seed is None else seed + i * 10086) for i, e in enumerate(self.envs)]
        self.last_infos = [info for _, info in out]
        return np.stack([o for o, _ in out])[:, None, :]

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
            infos.append(self._info(i, info))
        self.calls += 1
        self.last_infos = infos
        return obs, rewards, dones, infos


class _MaskIngest:
    """The reference's mask ingest on top of an oracle loop: slot 0 from the reset infos, slot t+1 from the infos of
    step t, each written only when every env reported masks.  The oracle loops' rollout calls env.step once per step,
    for steps 0..T-1 in order; `rollout` checks that it did."""

    def _ingest_masks(self, agent_num):
        env = self.env
        self._insert_masks(0, env.last_infos, agent_num)
        self._slot = None
        step = env.step

        def stepped(actions):
            assert self._slot is not None, "env.step outside a rollout"
            out = step(actions)
            self._slot += 1
            self._insert_masks(self._slot, out[3], agent_num)
            return out

        env.step = stepped

    def rollout(self):
        self._slot = 0
        super().rollout()
        assert self._slot == self.cfg.episode_length, self._slot
        self._slot = None

    def _insert_masks(self, slot, infos, agent_num):
        am = action_masks_from_infos(infos, agent_num)
        if am is not None:
            self.buf.action_masks[slot] = am


class MaskedTrainer(_MaskIngest, loop.Trainer):
    """Feed-forward PPO (oracle/loop.Trainer) on MaskedTargetVec."""

    def __init__(self, cfg, env_num, report=None):
        super().__init__(cfg, "MaskedTarget", env_num, env=MaskedTargetVec(env_num, report))
        self._ingest_masks(1)


class MaskedMATrainer(_MaskIngest, loop_ma.MATrainer):
    """Recurrent PPO (oracle/loop_ma.MATrainer) on MaskedTargetVec."""

    def __init__(self, cfg, env_num, report=None):
        saved = oenvs.ENVS.get("MaskedTarget")
        oenvs.ENVS["MaskedTarget"] = lambda n: MaskedTargetVec(n, report)
        try:
            super().__init__(cfg, "MaskedTarget", env_num)
        finally:
            if saved is None:
                del oenvs.ENVS["MaskedTarget"]
            else:
                oenvs.ENVS["MaskedTarget"] = saved
        self._ingest_masks(self.A)
