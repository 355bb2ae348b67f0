#!/usr/bin/env python
"""Record the Dict-observation traces by executing the unmodified reference on an env whose critic has its own observation.

TEST INFRASTRUCTURE, run where the reference source is present; the outputs are committed under tests/golden/.

    PYTHONPATH=oracle/refstubs:oracle:<reference checkout> python tools/gen_golden_dict_obs.py

Uses `gen_trace` of oracle/gen_golden.py unchanged, with the reference's `make` given `make_custom_envs`: the env of
tests/dict_obs_oracle.py (DictTargetEnv: Dict {"policy": Box(3), "critic": Box(7)}, Discrete(4), horizon 5, so episodes
end mid-rollout and mid-chunk) behind the reference's build_envs + Single2MultiAgentWrapper, as its make_toy_envs
builds its toy envs.  No wrapper carries the Dict: as in the reference's SMAC example (examples/smac/smac_env, whose env
returns {"policy": local_obs, "critic": global_state} and is given only a Monitor), the reference's SyncVectorEnv
stacks a Dict space key by key; Single2MultiAgentWrapper only adds the agent axis to each entry (nest_expand_dim).
gen_trace records the "policy" and "critic" entries of the buffer as policy_obs / critic_obs.

  trace_dict_obs_ff    feed-forward PPO, 4 envs, T = 16, 2 epochs, 2 minibatches, 2 iterations
  trace_dict_obs_gru   the same with --use_recurrent_policy true --data_chunk_length 3
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import gen_golden as gg  # noqa: E402
import gymnasium  # noqa: E402  (the stand-in)
from dict_obs_oracle import DictTargetEnv  # noqa: E402
from gymnasium.envs.registration import EnvSpec  # noqa: E402

BASE = ["--seed", "0", "--episode_length", "16", "--ppo_epoch", "2", "--num_mini_batch", "2", "--log_interval", "1000"]
TRACES = {"dict_obs_ff": BASE, "dict_obs_gru": BASE + ["--use_recurrent_policy", "true", "--data_chunk_length", "3"]}
ENV_NUM, ITERS = 4, 2


class GymDictTarget(gymnasium.Env):
    """DictTargetEnv with the gymnasium surface the reference's vec-env reads (spaces, `spec.id`)."""
    metadata = {"render_modes": []}

    def __init__(self):
        self.inner = DictTargetEnv()
        box = lambda d: gymnasium.spaces.Box(-np.inf, np.inf, (d,), np.float32)  # noqa: E731
        self.observation_space = gymnasium.spaces.Dict({"policy": box(DictTargetEnv.obs_dim),
                                                        "critic": box(DictTargetEnv.critic_obs_dim)})
        self.action_space = gymnasium.spaces.Discrete(DictTargetEnv.n_actions)
        self.spec = EnvSpec("DictTarget")
        self.agent_num = 1

    def reset(self, *, seed=None, options=None):
        return self.inner.reset(seed=seed)

    def step(self, action):
        return self.inner.step(action)


def make_dict_obs_envs(id, env_num=1, render_mode=None, **kwargs):
    from openrl.envs.common import build_envs
    from openrl.envs.wrappers import Single2MultiAgentWrapper

    return build_envs(make=lambda id, render_mode=None, disable_env_checker=None, **kw: GymDictTarget(), id=id,
                      env_num=env_num, render_mode=render_mode, wrappers=[Single2MultiAgentWrapper], **kwargs)


def main():
    torch.set_num_threads(8)   # the thread count every other trace was recorded with (tests/test_oracle_loop.py)
    make = gg.make
    gg.make = lambda id, env_num=1, **kw: make(id, env_num=env_num, make_custom_envs=make_dict_obs_envs, **kw)
    try:
        for tag, flags in TRACES.items():
            gg.gen_trace("DictTarget", ENV_NUM, flags, ITERS, tag)
    finally:
        gg.make = make


if __name__ == "__main__":
    main()
