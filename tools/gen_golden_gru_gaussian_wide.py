#!/usr/bin/env python
"""Record the traces of GRU policies with DiagGaussian heads of 9..64 dimensions by executing the unmodified reference.

TEST INFRASTRUCTURE, run where the reference source is present; the outputs are committed under tests/golden/.

    PYTHONPATH=oracle/refstubs:oracle:<reference checkout> python tools/gen_golden_gru_gaussian_wide.py

The recipe of tools/gen_golden_gru_gaussian.py (`gen_trace` of oracle/gen_golden.py unchanged, the reference's `make`
given `make_custom_envs` over its build_envs) on the envs of tests/gru_gaussian_wide_oracle.py:

  trace_gru_gaussian_wide_21         wide_gaussian_env(67, 21) (dm_control humanoid's shapes: Box(67) observations,
                                     Box(21)) behind Single2MultiAgentWrapper, --use_recurrent_policy true
                                     --data_chunk_length 3, 4 envs, T = 16, 2 epochs, 2 minibatches, 2 iterations
  trace_gru_gaussian_wide_spread_64  SpreadBox64Env (3 agents, Dict {"policy": Box(18), "critic": Box(54)}, Box(64);
                                     agents finish at different steps), --use_naive_recurrent_policy true, the same run

The reference has none of `use_recurrent_gaussian_head`, `use_wide_recurrent_gaussian_head` or
`use_wide_recurrent_observations` (it needs no opt-in), so the recorded flags leave them out and the tests add them.
`compact` keeps the weights at init and after the last iteration.
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
from gru_gaussian_wide_oracle import WIDE_21, SpreadBox64Env  # noqa: E402
from wide_gaussian_oracle import wide_gaussian_env  # noqa: E402

BASE = ["--seed", "0", "--episode_length", "16", "--ppo_epoch", "2", "--num_mini_batch", "2", "--log_interval", "1000"]
ENV_NUM, ITERS = 4, 2
TRACES = {
    "gru_gaussian_wide_21": BASE + ["--use_recurrent_policy", "true", "--data_chunk_length", "3"],
    "gru_gaussian_wide_spread_64": BASE + ["--use_naive_recurrent_policy", "true", "--data_chunk_length", "3"],
}


def _box(d):
    return gymnasium.spaces.Box(-np.inf, np.inf, (d,), np.float32)


class GymSpreadBox64(gymnasium.Env):
    """SpreadBox64Env as a three-agent env of the reference (agent axis first, no Single2MultiAgentWrapper)."""
    metadata = {"render_modes": []}

    def __init__(self):
        self.inner = SpreadBox64Env()
        self.observation_space = gymnasium.spaces.Dict({"policy": _box(SpreadBox64Env.obs_dim),
                                                        "critic": _box(SpreadBox64Env.critic_obs_dim)})
        self.action_space = gymnasium.spaces.Box(-1.0, 1.0, (SpreadBox64Env.act_dim,), np.float32)
        self.spec = EnvSpec("SpreadBox64")
        self.agent_num = SpreadBox64Env.agent_num

    def reset(self, *, seed=None, options=None):
        return self.inner.reset(seed=seed)

    def step(self, action):
        return self.inner.step(action)


class GymWideBox21(gymnasium.Env):
    metadata = {"render_modes": []}

    def __init__(self):
        d, n = WIDE_21
        self.inner = wide_gaussian_env(d, n)()
        self.observation_space = _box(d)
        self.action_space = gymnasium.spaces.Box(-1.0, 1.0, (n,), np.float32)
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
        for tag, cls, multi, env_id in (("gru_gaussian_wide_21", GymWideBox21, False, "WideGaussianTarget"),
                                        ("gru_gaussian_wide_spread_64", GymSpreadBox64, True, "SpreadBox64")):
            gg.make = lambda id, env_num=1, cls=cls, multi=multi, **kw: make(id, env_num=env_num,
                                                                             make_custom_envs=_envs(cls, multi), **kw)
            gg.gen_trace(env_id, ENV_NUM, TRACES[tag], ITERS, tag)
            compact(tag)
    finally:
        gg.make = make


if __name__ == "__main__":
    main()
