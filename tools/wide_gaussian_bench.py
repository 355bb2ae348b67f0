#!/usr/bin/env python
"""Device time of the feed-forward DiagGaussian head on both sides of the wide head (n = 8: the per-thread head,
ORL_HEAD_GAUSSIAN; 9..64: the head tile, ORL_HEAD_GAUSSIAN_WIDE), at C5's size: 1024 host-stepped envs x 128 steps, obs
widths 67 and 256.

    python tools/wide_gaussian_bench.py [--reps 20] [--widths 8 9 21 38 64] [--obs 67 256]

Per (obs width, head width) it reports the host act of one step (PPOModule.act_rows over the 1024 rows of a buffer slot,
the launch the host rollout issues each step), orl_policy_eval over the whole buffer (131072 rows) and one FFMA update
epoch over the whole buffer (ppo_epoch 1, num_mini_batch 1), each timed with CUDA events around `reps` repetitions after
a warm-up, with the card's name and power limit read in the same run.  Prints one JSON line.  Needs a GPU.
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

N_ENVS, T = 1024, 128


class BoxHost:
    """obs ~ N(0, 1) (N, 1, d), Box(n) actions, reward ~ N(0, 1), done ~ Bernoulli(0.001)."""

    def __init__(self, n_envs, d, n, seed=0):
        from openrl_b200 import spaces

        self.parallel_env_num, self.agent_num, self.d = n_envs, 1, d
        self.observation_space = spaces.Box(-np.inf, np.inf, (d,), np.float32)
        self.action_space = spaces.Box(-1.0, 1.0, (n,), np.float32)
        self.rng = np.random.default_rng(seed)

    def reset(self, seed=None):
        return self.rng.standard_normal((self.parallel_env_num, 1, self.d)).astype(np.float32)

    def step(self, actions):
        n = self.parallel_env_num
        return (self.rng.standard_normal((n, 1, self.d)).astype(np.float32), self.rng.standard_normal((n, 1, 1)),
                self.rng.random((n, 1)) < 1e-3, [{} for _ in range(n)])


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


def measure(d, n, reps):
    from openrl_b200 import lib
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.vec_env import HostVecEnv
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.logger import Logger

    cfg = create_config_parser().parse_args(["--seed", "0", "--episode_length", str(T), "--ppo_epoch", "1", "--num_mini_batch",
                                             "1", "--log_interval", "1000", "--host_env_groups", "false",
                                             "--use_wide_observations", "true", "--use_wide_gaussian_head", "true"])
    cfg.quiet = True
    net = PPONet(HostVecEnv(BoxHost(N_ENVS, d, n)), cfg=cfg, device="cuda:0")
    agent = PPOAgent(net)
    agent.train(total_time_steps=0, logger=Logger(quiet=True))
    drv = agent.driver
    drv.actor_rollout()
    drv.compute_returns()
    b, tr, m = drv.buffer.data, drv.trainer, drv.trainer.algo_module
    pol = m.models["policy"]
    assert not tr.use_tensor_cores and pol.head_kind == (lib.HEAD_GAUSSIAN_WIDE if n > 8 else lib.HEAD_GAUSSIAN)
    B, rows = N_ENVS, N_ENVS * T
    obs, acts, logp = b.policy_obs[0].view(B, d), b.actions[0].view(B, n), b.action_log_probs[0].view(B, n)
    step = [0]

    def act():
        step[0] += 1
        m.act_rows(obs, acts, logp, 0, B, 7, step[0])

    all_obs, all_acts = b.policy_obs[:T].reshape(rows, d), b.actions.reshape(rows, n)
    lp, ent = torch.empty(rows, n, device="cuda"), torch.empty(rows, n, device="cuda")

    def evaluate():
        lib.check(m._lib.orl_policy_eval(lib.ptr(pol.flat_params), d, n, pol.activation_id, pol.head_kind, lib.ptr(all_obs),
                                         lib.ptr(all_acts), None, lib.ptr(lp), lib.ptr(ent), rows, lib.current_stream()),
                  "orl_policy_eval")

    act_ms = device_ms(act, reps * 20)
    eval_ms = device_ms(evaluate, reps)
    update_ms = device_ms(lambda: tr.train(b), reps)
    return dict(d=d, n=n, head_kind=int(pol.head_kind), act_ms_per_step=round(act_ms, 4), eval_ms=round(eval_ms, 3),
                update_ms_per_epoch=round(update_ms, 3))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--widths", type=int, nargs="+", default=[8, 9, 21, 38, 64])
    ap.add_argument("--obs", type=int, nargs="+", default=[67, 256])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("wide_gaussian_bench.py needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    rows = [measure(d, n, args.reps) for d in args.obs for n in args.widths]
    print(json.dumps(dict(gpu=card, n_envs=N_ENVS, steps=T, results=rows)))


if __name__ == "__main__":
    main()
