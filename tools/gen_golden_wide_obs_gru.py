#!/usr/bin/env python
"""Record the wide-observation GRU traces by executing the unmodified reference on envs whose observations are wider
than 64, with recurrent policies.

TEST INFRASTRUCTURE, run where the reference source is present; the outputs are committed under tests/golden/.

    PYTHONPATH=oracle/refstubs:oracle:<reference checkout> python tools/gen_golden_wide_obs_gru.py

The recipe of tools/gen_golden_wide_obs.py (`gen_trace` of oracle/gen_golden.py unchanged, the reference's `make` given
`make_custom_envs`, the envs behind the reference's build_envs + Single2MultiAgentWrapper) on the envs of
tests/wide_obs_gru_oracle.py:

  trace_wide_obs_gru_dict      MaskedWideDictTargetEnv (SMAC 8m's shapes: Dict {"policy": Box(80), "critic": Box(168)},
                               Discrete(14), legal-move masks in info["action_masks"]), --use_recurrent_policy true
                               --data_chunk_length 3, 4 envs, T = 16, 2 epochs, 2 minibatches, 2 iterations
  trace_wide_obs_gru_box_256   WideBoxDiscreteEnv (Box(256) observations, Discrete(5)), --use_naive_recurrent_policy
                               true, the same run

Both nets' weights are random float32 that barely compress, three snapshots of them (init and after each iteration)
would put either file above 1 MB.  `compact` keeps the initial weights and those after the last iteration, which depend on
every update before them, and drops a critic_obs that equals policy_obs (a flat Box env's).
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
from wide_obs_gru_oracle import MaskedWideDictTargetEnv, WideBoxDiscreteEnv  # noqa: E402

BASE = ["--seed", "0", "--episode_length", "16", "--ppo_epoch", "2", "--num_mini_batch", "2", "--log_interval", "1000"]
ENV_NUM, ITERS = 4, 2
TRACES = {
    "wide_obs_gru_dict": BASE + ["--use_recurrent_policy", "true", "--data_chunk_length", "3"],
    "wide_obs_gru_box_256": BASE + ["--use_naive_recurrent_policy", "true", "--data_chunk_length", "3"],
}


def _box(d):
    return gymnasium.spaces.Box(-np.inf, np.inf, (d,), np.float32)


class GymMaskedWideDict(gymnasium.Env):
    metadata = {"render_modes": []}

    def __init__(self):
        self.inner = MaskedWideDictTargetEnv()
        self.observation_space = gymnasium.spaces.Dict({"policy": _box(MaskedWideDictTargetEnv.obs_dim),
                                                        "critic": _box(MaskedWideDictTargetEnv.critic_obs_dim)})
        self.action_space = gymnasium.spaces.Discrete(MaskedWideDictTargetEnv.n_actions)
        self.spec = EnvSpec("MaskedWideDictTarget")
        self.agent_num = 1

    def reset(self, *, seed=None, options=None):
        return self.inner.reset(seed=seed)

    def step(self, action):
        return self.inner.step(action)


class GymWideBoxDiscrete(gymnasium.Env):
    metadata = {"render_modes": []}

    def __init__(self):
        self.inner = WideBoxDiscreteEnv()
        self.observation_space = _box(WideBoxDiscreteEnv.obs_dim)
        self.action_space = gymnasium.spaces.Discrete(WideBoxDiscreteEnv.n_actions)
        self.spec = EnvSpec("WideBoxDiscrete")
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


def compact(tag):
    """Rewrite tests/golden/trace_<tag>.npz without the weights of the iterations before the last and without a critic_obs
    equal to policy_obs."""
    path = os.path.join(gg.OUT, f"trace_{tag}.npz")
    with np.load(path, allow_pickle=True) as z:
        rec = {k: z[k] for k in z.files}
    last = int(rec["meta/iters"]) - 1
    for k in list(rec):
        it = k.split("/")[0]
        if it.startswith("it") and "/params/" in k and int(it[2:]) != last:
            del rec[k]
        elif k.endswith("/critic_obs") and np.array_equal(rec[k], rec[f"{it}/policy_obs"]):
            del rec[k]
    np.savez_compressed(path, **rec)
    print("compacted", os.path.basename(path), "bytes", os.path.getsize(path))


def main():
    torch.set_num_threads(8)   # the thread count every other trace was recorded with (tests/test_oracle_loop.py)
    make = gg.make
    try:
        for tag, cls, env_id in (("wide_obs_gru_dict", GymMaskedWideDict, "MaskedWideDictTarget"),
                                 ("wide_obs_gru_box_256", GymWideBoxDiscrete, "WideBoxDiscrete")):
            gg.make = lambda id, env_num=1, cls=cls, **kw: make(id, env_num=env_num, make_custom_envs=_envs(cls), **kw)
            gg.gen_trace(env_id, ENV_NUM, TRACES[tag], ITERS, tag)
            compact(tag)
    finally:
        gg.make = make


if __name__ == "__main__":
    main()
