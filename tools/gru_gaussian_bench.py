#!/usr/bin/env python
"""Device time of a GRU policy's DiagGaussian head (ORL_HEAD_GAUSSIAN, n in {1, 6, 8}) against its Categorical head at
n = 8, at the shapes of tools/wide_actions_gru_bench.py: 1024 host-stepped envs x 128 steps, obs width 27, chunks of 8.
Both heads are the same 8-row mat-vec of the GRU kernels; the Gaussian one adds gaussian_act / gaussian_row and one
8-float tape field.

    python tools/gru_gaussian_bench.py [--reps 20]

Per head it reports the host act of one step (PPOModule.act_rows over the 1024 rows of a buffer slot, the
orl_rnn_act_rows launch the host rollout issues each step) and one recurrent update epoch over the whole buffer
(ppo_epoch 1, num_mini_batch 1), both timed with CUDA events around `reps` repetitions after a warm-up, with the card's
name and power limit read in the same run.  Prints one JSON line.  Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

from wide_actions_gru_bench import device_ms  # noqa: E402

N_ENVS, T, D = 1024, 128, 27


class Host:
    """obs ~ N(0, 1) (N, 1, D), Box(n) or Discrete(n) actions, done ~ Bernoulli(0.01)."""

    def __init__(self, n_envs, n, box, seed=0):
        from openrl_b200 import spaces

        self.parallel_env_num, self.agent_num = n_envs, 1
        self.observation_space = spaces.Box(-np.inf, np.inf, (D,), np.float32)
        self.action_space = spaces.Box(-1.0, 1.0, (n,), np.float32) if box else spaces.Discrete(n)
        self.rng = np.random.default_rng(seed)

    def reset(self, seed=None):
        return self.rng.standard_normal((self.parallel_env_num, 1, D)).astype(np.float32)

    def step(self, actions):
        n = self.parallel_env_num
        return (self.rng.standard_normal((n, 1, D)).astype(np.float32), self.rng.standard_normal((n, 1, 1)),
                self.rng.random((n, 1)) < 0.01, [{} for _ in range(n)])


def measure(n, box, reps):
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.vec_env import HostVecEnv
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.logger import Logger

    cfg = create_config_parser().parse_args(["--seed", "0", "--episode_length", str(T), "--ppo_epoch", "1", "--num_mini_batch",
                                             "1", "--log_interval", "1000", "--host_env_groups", "false",
                                             "--use_recurrent_policy", "true", "--data_chunk_length", "8",
                                             "--use_recurrent_gaussian_head", "true"])
    cfg.quiet = True
    net = PPONet(HostVecEnv(Host(N_ENVS, n, box)), cfg=cfg, device="cuda:0")
    agent = PPOAgent(net)
    agent.train(total_time_steps=0, logger=Logger(quiet=True))
    drv = agent.driver
    drv.actor_rollout()
    drv.compute_returns()
    b, tr, m = drv.buffer.data, drv.trainer, drv.trainer.algo_module
    assert tr.recurrent and tr.head_kind == (1 if box else 0)
    B, w = N_ENVS, b.actions.shape[-1]
    obs, acts, logp = b.policy_obs[0].view(B, D), b.actions[0].view(B, w), b.action_log_probs[0].view(B, w)
    masks = b.masks[0].view(B)
    states = b.rnn_states[0:2].clone()   # slot 0 is read, slot 1 written: a copy, so the buffer keeps its rollout
    step = [0]

    def act():
        step[0] += 1
        m.act_rows(obs, acts, logp, 0, B, 7, step[0], masks=masks, rnn_states=states)

    act_ms = device_ms(act, reps * 20)
    update_ms = device_ms(lambda: tr.train(b), reps)
    return dict(head="gaussian" if box else "categorical", n=n, act_ms_per_step=round(act_ms, 4),
                update_ms_per_epoch=round(update_ms, 3))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gru_gaussian_bench.py needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    rows = [measure(8, False, args.reps)] + [measure(n, True, args.reps) for n in (1, 6, 8)]
    print(json.dumps(dict(gpu=card, n_envs=N_ENVS, steps=T, obs_dim=D, results=rows)))


if __name__ == "__main__":
    main()
