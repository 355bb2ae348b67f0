#!/usr/bin/env python
"""Device time of the feed-forward Categorical head at head widths on both sides of the wide head (n <= 8: the per-thread
head; 9..64: the logits tile), at C5's size: 1024 host-stepped envs x 128 steps, obs width 27.

    python tools/wide_actions_bench.py [--reps 50] [--widths 8 9 18 64]

Per width it reports the host act of one step (PPOModule.act_rows over the 1024 rows of a buffer slot, the launch the
host rollout issues each step) and one FFMA update epoch over the whole buffer (ppo_epoch 1, num_mini_batch 1), both
timed with CUDA events around `reps` repetitions after a warm-up, with the card's name and power limit read in the same
run.  Prints one JSON line.  Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_ENVS, T, D = 1024, 128, 27


class MaskedHost:
    """obs ~ N(0, 1) (N, 1, D), Discrete(n), a random legal subset in info["action_masks"], done ~ Bernoulli(0.01)."""

    def __init__(self, n_envs, n_actions, seed=0):
        from openrl_b200 import spaces

        self.parallel_env_num, self.agent_num, self.n = n_envs, 1, n_actions
        self.observation_space = spaces.Box(-np.inf, np.inf, (D,), np.float32)
        self.action_space = spaces.Discrete(n_actions)
        self.rng = np.random.default_rng(seed)

    def _infos(self):
        m = (self.rng.random((self.parallel_env_num, self.n)) < 0.7).astype(np.int8)
        m[:, 0] = 1
        return [{"action_masks": m[i]} for i in range(self.parallel_env_num)]

    def reset(self, seed=None):
        return self.rng.standard_normal((self.parallel_env_num, 1, D)).astype(np.float32), self._infos()

    def step(self, actions):
        n = self.parallel_env_num
        return (self.rng.standard_normal((n, 1, D)).astype(np.float32), self.rng.standard_normal((n, 1, 1)),
                self.rng.random((n, 1)) < 0.01, self._infos())


def device_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def measure(n, reps):
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.vec_env import HostVecEnv
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.logger import Logger

    cfg = create_config_parser().parse_args(["--seed", "0", "--episode_length", str(T), "--ppo_epoch", "1", "--num_mini_batch",
                                             "1", "--log_interval", "1000", "--host_env_groups", "false"])
    cfg.quiet = True
    net = PPONet(HostVecEnv(MaskedHost(N_ENVS, n)), cfg=cfg, device="cuda:0")
    agent = PPOAgent(net)
    agent.train(total_time_steps=0, logger=Logger(quiet=True))
    drv = agent.driver
    drv.actor_rollout()
    drv.compute_returns()
    b, tr, m = drv.buffer.data, drv.trainer, drv.trainer.algo_module
    assert not tr.use_tensor_cores and not b.action_masks_trivial
    B = N_ENVS
    obs, acts, logp = b.policy_obs[0].view(B, D), b.actions[0].view(B, 1), b.action_log_probs[0].view(B, 1)
    am = b.action_masks[0].view(B, n)
    step = [0]

    def act():
        step[0] += 1
        m.act_rows(obs, acts, logp, 0, B, 7, step[0], action_masks=am)

    act_ms = device_ms(act, reps * 20)
    update_ms = device_ms(lambda: tr.train(b), reps)
    return dict(n=n, act_ms_per_step=round(act_ms, 4), update_ms_per_epoch=round(update_ms, 3))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--widths", type=int, nargs="+", default=[8, 9, 18, 64])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("wide_actions_bench.py needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    rows = [measure(n, args.reps) for n in args.widths]
    print(json.dumps(dict(gpu=card, n_envs=N_ENVS, steps=T, obs_dim=D, results=rows)))


if __name__ == "__main__":
    main()
