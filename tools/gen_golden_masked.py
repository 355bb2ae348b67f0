#!/usr/bin/env python
"""Record the action-mask traces by executing the unmodified reference on an env that reports legal-move masks.

TEST INFRASTRUCTURE, run where the reference source is present; the outputs are committed under tests/golden/.

    PYTHONPATH=oracle/refstubs:oracle:<reference checkout> python tools/gen_golden_masked.py

Uses `gen_trace` of oracle/gen_golden.py unchanged, with the reference's `make` given `make_custom_envs`: the masked
env of tests/masked_oracle.py (MaskedTargetEnv: Discrete(5), `info["action_masks"]` on reset and every step, horizon
5, so episodes end mid-rollout and mid-chunk) behind the reference's build_envs + Single2MultiAgentWrapper, as its
make_toy_envs builds its toy envs.  gen_trace records `action_masks` with the rest of the buffer.

  trace_masked_ff    feed-forward PPO, 4 envs, T = 16, 2 epochs, 2 minibatches, 2 iterations
  trace_masked_gru   the same with --use_recurrent_policy true --data_chunk_length 3
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
from masked_oracle import MaskedTargetEnv  # noqa: E402

BASE = ["--seed", "0", "--episode_length", "16", "--ppo_epoch", "2", "--num_mini_batch", "2", "--log_interval", "1000"]
TRACES = {"masked_ff": BASE, "masked_gru": BASE + ["--use_recurrent_policy", "true", "--data_chunk_length", "3"]}
ENV_NUM, ITERS = 4, 2


class GymMaskedTarget(gymnasium.Env):
    """MaskedTargetEnv with the gymnasium surface the reference's vec-env reads (spaces, `spec.id`)."""
    metadata = {"render_modes": []}

    def __init__(self):
        self.inner = MaskedTargetEnv()
        self.observation_space = gymnasium.spaces.Box(0.0, 1.0, (MaskedTargetEnv.obs_dim,), np.float32)
        self.action_space = gymnasium.spaces.Discrete(MaskedTargetEnv.n_actions)
        self.spec = EnvSpec("MaskedTarget")
        self.agent_num = 1

    def reset(self, *, seed=None, options=None):
        return self.inner.reset(seed=seed)

    def step(self, action):
        return self.inner.step(action)


def make_masked_envs(id, env_num=1, render_mode=None, **kwargs):
    from openrl.envs.common import build_envs
    from openrl.envs.wrappers import Single2MultiAgentWrapper

    return build_envs(make=lambda id, render_mode=None, disable_env_checker=None, **kw: GymMaskedTarget(), id=id,
                      env_num=env_num, render_mode=render_mode, wrappers=[Single2MultiAgentWrapper], **kwargs)


def main():
    torch.set_num_threads(8)   # the thread count every other trace was recorded with (tests/test_oracle_loop.py)
    make = gg.make
    gg.make = lambda id, env_num=1, **kw: make(id, env_num=env_num, make_custom_envs=make_masked_envs, **kw)
    try:
        for tag, flags in TRACES.items():
            gg.gen_trace("MaskedTarget", ENV_NUM, flags, ITERS, tag)
    finally:
        gg.make = make


if __name__ == "__main__":
    main()
