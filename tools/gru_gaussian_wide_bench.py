#!/usr/bin/env python
"""Device time of a GRU policy's wide DiagGaussian head (ORL_HEAD_GAUSSIAN_WIDE, n in {9, 21, 64}) against its 8-wide
DiagGaussian head (ORL_HEAD_GAUSSIAN, n = 8), at C5-like sizes: 1024 host-stepped envs x 128 steps, 17 observation
features (SyntheticHost's), chunks of 8.  The wide head runs the 64-row head block of the GRU kernels whatever n is, so
its times should depend little on n.

    python tools/gru_gaussian_wide_bench.py [--reps 20]

Per head it reports the host act of one step (PPOModule.act_rows over the 1024 rows of a buffer slot, the
orl_rnn_act_rows launch the host rollout issues each step) and one update minibatch (ppo_epoch 1, num_mini_batch 1: the
whole 131072-row buffer in 16384 chunks), both timed with CUDA events around `reps` repetitions after a warm-up, with
the card's name and power limit read in the same run.  Prints one JSON line.  Needs a GPU.
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

N_ENVS, T, D = 1024, 128, 17


class Host:
    """obs ~ N(0, 1) (N, 1, D), Box(n) actions, done ~ Bernoulli(0.01)."""

    def __init__(self, n_envs, n, seed=0):
        from openrl_b200 import spaces

        self.parallel_env_num, self.agent_num = n_envs, 1
        self.observation_space = spaces.Box(-np.inf, np.inf, (D,), np.float32)
        self.action_space = spaces.Box(-1.0, 1.0, (n,), np.float32)
        self.rng = np.random.default_rng(seed)

    def reset(self, seed=None):
        return self.rng.standard_normal((self.parallel_env_num, 1, D)).astype(np.float32)

    def step(self, actions):
        n = self.parallel_env_num
        return (self.rng.standard_normal((n, 1, D)).astype(np.float32), self.rng.standard_normal((n, 1, 1)),
                self.rng.random((n, 1)) < 0.01, [{} for _ in range(n)])


def measure(n, reps):
    from openrl_b200 import lib
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.vec_env import HostVecEnv
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.logger import Logger

    cfg = create_config_parser().parse_args(["--seed", "0", "--episode_length", str(T), "--ppo_epoch", "1", "--num_mini_batch",
                                             "1", "--log_interval", "1000", "--host_env_groups", "false",
                                             "--use_recurrent_policy", "true", "--data_chunk_length", "8",
                                             "--use_recurrent_gaussian_head", "true",
                                             "--use_wide_recurrent_gaussian_head", "true"])
    cfg.quiet = True
    net = PPONet(HostVecEnv(Host(N_ENVS, n)), cfg=cfg, device="cuda:0")
    agent = PPOAgent(net)
    agent.train(total_time_steps=0, logger=Logger(quiet=True))
    drv = agent.driver
    drv.actor_rollout()
    drv.compute_returns()
    b, tr, m = drv.buffer.data, drv.trainer, drv.trainer.algo_module
    assert tr.recurrent and tr.head_kind == (lib.HEAD_GAUSSIAN if n <= 8 else lib.HEAD_GAUSSIAN_WIDE)
    B = N_ENVS
    obs, acts, logp = b.policy_obs[0].view(B, D), b.actions[0].view(B, n), b.action_log_probs[0].view(B, n)
    masks = b.masks[0].view(B)
    states = b.rnn_states[0:2].clone()   # slot 0 is read, slot 1 written: a copy, so the buffer keeps its rollout
    step = [0]

    def act():
        step[0] += 1
        m.act_rows(obs, acts, logp, 0, B, 7, step[0], masks=masks, rnn_states=states)

    act_ms = device_ms(act, reps * 20)
    update_ms = device_ms(lambda: tr.train(b), reps)
    return dict(head="gaussian_wide" if n > 8 else "gaussian", n=n, act_ms_per_step=round(act_ms, 4),
                update_ms_per_minibatch=round(update_ms, 3))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gru_gaussian_wide_bench.py needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    rows = [measure(n, args.reps) for n in (8, 9, 21, 64)]
    print(json.dumps(dict(gpu=card, n_envs=N_ENVS, steps=T, obs_dim=D, results=rows)))


if __name__ == "__main__":
    main()
