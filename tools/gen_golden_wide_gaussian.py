#!/usr/bin/env python
"""Record the wide DiagGaussian traces by executing the unmodified reference on envs whose Box action spaces are wider
than 8.

TEST INFRASTRUCTURE, run where the reference is installed (oracle/_ref, made by build()); the outputs are committed under
tests/golden/.

    PYTHONPATH=oracle/refstubs:oracle:oracle/_ref python tools/gen_golden_wide_gaussian.py

The recipe of tools/gen_golden_wide_obs.py (`gen_trace` of oracle/gen_golden.py unchanged, the reference's `make` given
`make_custom_envs`, the envs behind the reference's build_envs + Single2MultiAgentWrapper) on the envs of
tests/wide_gaussian_oracle.py:

  trace_wide_gaussian_21   d = 67 observations, Box(21) actions (dm_control humanoid's shapes), feed-forward PPO,
                           4 envs, T = 16, 2 epochs, 2 minibatches, 2 iterations
  trace_wide_gaussian_64   d = 256, Box(64) (the update's shared-memory worst case), the same run

Both observation widths are above 64.  The reference has neither `use_wide_gaussian_head` nor `use_wide_observations` (it
needs no opt-in), so the recorded flags leave them out and the tests add both.  `compact` of tools/gen_golden_wide_obs_gru.py keeps the weights at init and after
the last iteration only, which keeps each file under 1 MB.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

import gen_golden as gg  # noqa: E402
import gymnasium  # noqa: E402  (the stand-in)
from gymnasium.envs.registration import EnvSpec  # noqa: E402
from gen_golden_wide_obs_gru import compact  # noqa: E402
from wide_gaussian_oracle import TRACES, wide_gaussian_env  # noqa: E402

BASE = ["--seed", "0", "--episode_length", "16", "--ppo_epoch", "2", "--num_mini_batch", "2", "--log_interval", "1000"]
ENV_NUM, ITERS = 4, 2


def _gym_env(d, n):
    inner_cls = wide_gaussian_env(d, n)

    class GymWideGaussian(gymnasium.Env):
        metadata = {"render_modes": []}

        def __init__(self):
            self.inner = inner_cls()
            self.observation_space = gymnasium.spaces.Box(-np.inf, np.inf, (d,), np.float32)
            self.action_space = gymnasium.spaces.Box(-1.0, 1.0, (n,), np.float32)
            self.spec = EnvSpec("WideGaussianTarget")
            self.agent_num = 1

        def reset(self, *, seed=None, options=None):
            return self.inner.reset(seed=seed)

        def step(self, action):
            return self.inner.step(action)
    return GymWideGaussian


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
        for n, d in TRACES.items():
            cls = _gym_env(d, n)
            gg.make = lambda id, env_num=1, cls=cls, **kw: make(id, env_num=env_num, make_custom_envs=_envs(cls), **kw)
            tag = f"wide_gaussian_{n}"
            gg.gen_trace("WideGaussianTarget", ENV_NUM, BASE, ITERS, tag)
            compact(tag)
    finally:
        gg.make = make


if __name__ == "__main__":
    main()
