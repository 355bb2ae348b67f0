#!/usr/bin/env python
"""Record the wide-observation traces by executing the unmodified reference on envs whose observations are wider than 64.

TEST INFRASTRUCTURE, run where the reference source is present; the outputs are committed under tests/golden/.

    PYTHONPATH=oracle/refstubs:oracle:<reference checkout> python tools/gen_golden_wide_obs.py

Uses `gen_trace` of oracle/gen_golden.py unchanged, with the reference's `make` given `make_custom_envs`, as
tools/gen_golden_dict_obs.py does: the envs of tests/wide_obs_oracle.py behind the reference's build_envs +
Single2MultiAgentWrapper.

  trace_wide_obs_dict      WideDictTargetEnv (SMAC 8m's shapes: Dict {"policy": Box(80), "critic": Box(168)},
                           Discrete(14)), feed-forward PPO, 4 envs, T = 16, 2 epochs, 2 minibatches, 2 iterations
  trace_wide_obs_box_256   WideBoxTargetEnv (Box(256) observations, Box(4) actions: a DiagGaussian head), the same run
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import gen_golden as gg  # noqa: E402
import gymnasium  # noqa: E402  (the stand-in)
from gymnasium.envs.registration import EnvSpec  # noqa: E402
from wide_obs_oracle import WideBoxTargetEnv, WideDictTargetEnv  # noqa: E402

BASE = ["--seed", "0", "--episode_length", "16", "--ppo_epoch", "2", "--num_mini_batch", "2", "--log_interval", "1000"]
ENV_NUM, ITERS = 4, 2


def _box(lo, hi, d):
    return gymnasium.spaces.Box(lo, hi, (d,), np.float32)


class GymWideDict(gymnasium.Env):
    metadata = {"render_modes": []}

    def __init__(self):
        self.inner = WideDictTargetEnv()
        self.observation_space = gymnasium.spaces.Dict({"policy": _box(-np.inf, np.inf, WideDictTargetEnv.obs_dim),
                                                        "critic": _box(-np.inf, np.inf, WideDictTargetEnv.critic_obs_dim)})
        self.action_space = gymnasium.spaces.Discrete(WideDictTargetEnv.n_actions)
        self.spec = EnvSpec("WideDictTarget")
        self.agent_num = 1

    def reset(self, *, seed=None, options=None):
        return self.inner.reset(seed=seed)

    def step(self, action):
        return self.inner.step(action)


class GymWideBox(gymnasium.Env):
    metadata = {"render_modes": []}

    def __init__(self):
        self.inner = WideBoxTargetEnv()
        self.observation_space = _box(-np.inf, np.inf, WideBoxTargetEnv.obs_dim)
        self.action_space = _box(-1.0, 1.0, WideBoxTargetEnv.act_dim)
        self.spec = EnvSpec("WideBoxTarget")
        self.agent_num = 1

    def reset(self, *, seed=None, options=None):
        return self.inner.reset(seed=seed)

    def step(self, action):
        return self.inner.step(action)


def _envs(cls):
    def make_envs(id, env_num=1, render_mode=None, **kwargs):
        from openrl.envs.common import build_envs
        from openrl.envs.wrappers import Single2MultiAgentWrapper

        return build_envs(make=lambda id, render_mode=None, disable_env_checker=None, **kw: cls(), id=id,
                          env_num=env_num, render_mode=render_mode, wrappers=[Single2MultiAgentWrapper], **kwargs)
    return make_envs


def main():
    torch.set_num_threads(8)   # the thread count every other trace was recorded with (tests/test_oracle_loop.py)
    make = gg.make
    try:
        for tag, cls, env_id in (("wide_obs_dict", GymWideDict, "WideDictTarget"), ("wide_obs_box_256", GymWideBox, "WideBoxTarget")):
            gg.make = lambda id, env_num=1, cls=cls, **kw: make(id, env_num=env_num, make_custom_envs=_envs(cls), **kw)
            gg.gen_trace(env_id, ENV_NUM, BASE, ITERS, tag)
    finally:
        gg.make = make


if __name__ == "__main__":
    main()
