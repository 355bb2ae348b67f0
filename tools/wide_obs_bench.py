#!/usr/bin/env python
"""Device time of the feed-forward nets at observation widths on both sides of the panelled fc1 (d <= 64: all of W1 in
shared memory; 65..256: fc1 over 64-wide panels of the observation), at C5's size: 1024 host-stepped envs x 128 steps,
Dict observations with d = dc, Discrete(14) with masks (SMAC 8m's head).

    python tools/wide_obs_bench.py [--reps 20] [--widths 64 65 128 168 256]

Per width it reports the host act of one step (PPOModule.act_rows over the 1024 rows of a buffer slot, the launch the
host rollout issues each step), orl_critic_values over the buffer's T + 1 slots (PPOModule.get_values, as
compute_returns runs it) and one FFMA update epoch over the whole buffer (ppo_epoch 1, num_mini_batch 1), each timed
with CUDA events around its repetitions after a warm-up, with the card's name and power limit read in the same run.
Prints one JSON line.  Needs a GPU.
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

N_ENVS, T, N_ACT = 1024, 128, 14


class DictHost:
    """obs {"policy": (N, 1, d), "critic": (N, 1, d)} ~ N(0, 1), Discrete(14), a random legal subset in
    info["action_masks"], done ~ Bernoulli(0.01)."""

    def __init__(self, n_envs, d, seed=0):
        from openrl_b200 import spaces

        box = spaces.Box(-np.inf, np.inf, (d,), np.float32)
        self.parallel_env_num, self.agent_num, self.d = n_envs, 1, d
        self.observation_space = spaces.Dict({"policy": box, "critic": box})
        self.action_space = spaces.Discrete(N_ACT)
        self.rng = np.random.default_rng(seed)

    def _obs(self):
        n = self.parallel_env_num
        return {k: self.rng.standard_normal((n, 1, self.d)).astype(np.float32) for k in ("policy", "critic")}

    def _infos(self):
        m = (self.rng.random((self.parallel_env_num, N_ACT)) < 0.7).astype(np.int8)
        m[:, 0] = 1
        return [{"action_masks": m[i]} for i in range(self.parallel_env_num)]

    def reset(self, seed=None):
        return self._obs(), self._infos()

    def step(self, actions):
        n = self.parallel_env_num
        return self._obs(), self.rng.standard_normal((n, 1, 1)), self.rng.random((n, 1)) < 0.01, self._infos()


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


def measure(d, reps):
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.vec_env import HostVecEnv
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.logger import Logger

    cfg = create_config_parser().parse_args(["--seed", "0", "--episode_length", str(T), "--ppo_epoch", "1", "--num_mini_batch",
                                             "1", "--log_interval", "1000", "--host_env_groups", "false",
                                             "--use_wide_observations", "true"])
    cfg.quiet = True
    net = PPONet(HostVecEnv(DictHost(N_ENVS, d), wide_observations=True), cfg=cfg, device="cuda:0")
    agent = PPOAgent(net)
    agent.train(total_time_steps=0, logger=Logger(quiet=True))
    drv = agent.driver
    drv.actor_rollout()
    drv.compute_returns()
    b, tr, m = drv.buffer.data, drv.trainer, drv.trainer.algo_module
    assert not tr.use_tensor_cores and (tr.d, tr.dc, tr.n) == (d, d, N_ACT)
    B = N_ENVS
    obs, acts, logp = b.policy_obs[0].view(B, d), b.actions[0].view(B, 1), b.action_log_probs[0].view(B, 1)
    am = b.action_masks[0].view(B, N_ACT)
    cobs = b.critic_obs.view(-1, d)
    step = [0]

    def act():
        step[0] += 1
        m.act_rows(obs, acts, logp, 0, B, 7, step[0], action_masks=am)

    act_ms = device_ms(act, reps * 20)
    values_ms = device_ms(lambda: m.get_values(cobs), reps * 5)
    update_ms = device_ms(lambda: tr.train(b), reps)
    return dict(d=d, act_ms_per_step=round(act_ms, 4), critic_values_ms=round(values_ms, 4),
                update_ms_per_epoch=round(update_ms, 3))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--widths", type=int, nargs="+", default=[64, 65, 128, 168, 256])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("wide_obs_bench.py needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    rows = [measure(d, args.reps) for d in args.widths]
    print(json.dumps(dict(gpu=card, n_envs=N_ENVS, steps=T, n_actions=N_ACT, results=rows)))


if __name__ == "__main__":
    main()
