#!/usr/bin/env python
"""Record the GRU + DiagGaussian traces by executing the unmodified reference on Box-action envs with recurrent policies.

TEST INFRASTRUCTURE, run where the reference source is present; the outputs are committed under tests/golden/.

    PYTHONPATH=oracle/refstubs:oracle:<reference checkout> python tools/gen_golden_gru_gaussian.py

The recipe of tools/gen_golden_wide_obs_gru.py (`gen_trace` of oracle/gen_golden.py unchanged, the reference's `make`
given `make_custom_envs` over its build_envs) on the envs of tests/gru_gaussian_oracle.py:

  trace_gru_gaussian_spread    SpreadBoxEnv (continuous simple_spread's shapes: 3 agents, Dict {"policy": Box(18),
                               "critic": Box(54)}, Box(5); agents finish at different steps), --use_recurrent_policy true
                               --data_chunk_length 3, 4 envs, T = 16, 2 epochs, 2 minibatches, 2 iterations
  trace_gru_gaussian_box_256   wide_gaussian_env(256, 8) (Box(256) observations, Box(8)) behind
                               Single2MultiAgentWrapper, --use_naive_recurrent_policy true, the same run

The reference has neither `use_recurrent_gaussian_head` nor `use_wide_recurrent_observations` (it needs no opt-in), so the
recorded flags leave them out and the tests add them.  `compact` keeps the weights at init and after the last iteration.
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
from gru_gaussian_oracle import SpreadBoxEnv  # noqa: E402
from wide_gaussian_oracle import wide_gaussian_env  # noqa: E402

BASE = ["--seed", "0", "--episode_length", "16", "--ppo_epoch", "2", "--num_mini_batch", "2", "--log_interval", "1000"]
ENV_NUM, ITERS = 4, 2
TRACES = {
    "gru_gaussian_spread": BASE + ["--use_recurrent_policy", "true", "--data_chunk_length", "3"],
    "gru_gaussian_box_256": BASE + ["--use_naive_recurrent_policy", "true", "--data_chunk_length", "3"],
}


def _box(d):
    return gymnasium.spaces.Box(-np.inf, np.inf, (d,), np.float32)


class GymSpreadBox(gymnasium.Env):
    """SpreadBoxEnv as a three-agent env of the reference (agent axis first, no Single2MultiAgentWrapper)."""
    metadata = {"render_modes": []}

    def __init__(self):
        self.inner = SpreadBoxEnv()
        self.observation_space = gymnasium.spaces.Dict({"policy": _box(SpreadBoxEnv.obs_dim),
                                                        "critic": _box(SpreadBoxEnv.critic_obs_dim)})
        self.action_space = gymnasium.spaces.Box(-1.0, 1.0, (SpreadBoxEnv.act_dim,), np.float32)
        self.spec = EnvSpec("SpreadBox")
        self.agent_num = SpreadBoxEnv.agent_num

    def reset(self, *, seed=None, options=None):
        return self.inner.reset(seed=seed)

    def step(self, action):
        return self.inner.step(action)


class GymWideBox(gymnasium.Env):
    metadata = {"render_modes": []}

    def __init__(self):
        self.inner = wide_gaussian_env(256, 8)()
        self.observation_space = _box(256)
        self.action_space = gymnasium.spaces.Box(-1.0, 1.0, (8,), np.float32)
        self.spec = EnvSpec("WideGaussianTarget")
        self.agent_num = 1

    def reset(self, *, seed=None, options=None):
        return self.inner.reset(seed=seed)

    def step(self, action):
        return self.inner.step(action)


def _envs(cls, multi):
    def make_envs(id, env_num=1, render_mode=None, **kwargs):
        from openrl.envs.common import build_envs
        from openrl.envs.wrappers import Single2MultiAgentWrapper

        return build_envs(make=lambda id, render_mode=None, disable_env_checker=None, **kw: cls(), id=id,
                          env_num=env_num, render_mode=render_mode, wrappers=[] if multi else [Single2MultiAgentWrapper],
                          **kwargs)
    return make_envs


def main():
    torch.set_num_threads(8)   # the thread count every other trace was recorded with (tests/test_oracle_loop.py)
    make = gg.make
    try:
        for tag, cls, multi, env_id in (("gru_gaussian_spread", GymSpreadBox, True, "SpreadBox"),
                                        ("gru_gaussian_box_256", GymWideBox, False, "WideGaussianTarget")):
            gg.make = lambda id, env_num=1, cls=cls, multi=multi, **kw: make(id, env_num=env_num,
                                                                             make_custom_envs=_envs(cls, multi), **kw)
            gg.gen_trace(env_id, ENV_NUM, TRACES[tag], ITERS, tag)
            compact(tag)
    finally:
        gg.make = make


if __name__ == "__main__":
    main()
