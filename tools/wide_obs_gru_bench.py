#!/usr/bin/env python
"""Device time of GRU policies and critics over observations of 64..256 features (cfg.use_wide_recurrent_observations)
on a SMAC-8m-shaped buffer: 128 host-stepped envs x 8 agents (1024 rows) x 128 steps, Dict {"policy": d, "critic": d},
Discrete(14) with masks, chunks of 8.

    python tools/wide_obs_gru_bench.py [--reps 20] [--widths 64 80 168 256]

Per width it reports the host act of one step (PPOModule.act_rows over the 1024 rows of a buffer slot, the orl_rnn_act_rows
launch the host rollout issues each step), the recurrent critic over the T + 1 slots (orl_rnn_critic) and one recurrent
update epoch over the whole buffer (ppo_epoch 1, num_mini_batch 1: the chunk kernels, the tape reductions, the dW1
panels and the optimizer), timed with CUDA events around repetitions after a warm-up, with the card's name and power
limit read in the same run.  d = 64 runs the narrow kernels.  Prints one JSON line.  Needs a GPU.
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

N_ENVS, A, T, N_ACT = 128, 8, 128, 14


class SmacShapedHost:
    """N envs x 8 agents, Dict obs ~ N(0, 1) of width d for both entries, Discrete(14), a random legal subset in
    info["action_masks"], done ~ Bernoulli(0.01)."""

    def __init__(self, d, seed=0):
        from openrl_b200 import spaces

        box = spaces.Box(-np.inf, np.inf, (d,), np.float32)
        self.parallel_env_num, self.agent_num, self.d = N_ENVS, A, d
        self.observation_space = spaces.Dict({"policy": box, "critic": box})
        self.action_space = spaces.Discrete(N_ACT)
        self.rng = np.random.default_rng(seed)

    def _obs(self):
        x = lambda: self.rng.standard_normal((N_ENVS, A, self.d)).astype(np.float32)  # noqa: E731
        return {"policy": x(), "critic": x()}

    def _infos(self):
        m = (self.rng.random((N_ENVS, A, N_ACT)) < 0.7).astype(np.int8)
        m[..., 0] = 1
        return [{"action_masks": m[i]} for i in range(N_ENVS)]

    def reset(self, seed=None):
        return self._obs(), self._infos()

    def step(self, actions):
        done = np.repeat(self.rng.random((N_ENVS, 1)) < 0.01, A, axis=1)
        return self._obs(), self.rng.standard_normal((N_ENVS, A, 1)), done, self._infos()


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
    from openrl_b200 import lib
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.vec_env import HostVecEnv
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.logger import Logger

    cfg = create_config_parser().parse_args(["--seed", "0", "--episode_length", str(T), "--ppo_epoch", "1", "--num_mini_batch",
                                             "1", "--log_interval", "1000", "--host_env_groups", "false",
                                             "--use_recurrent_policy", "true", "--data_chunk_length", "8",
                                             "--use_wide_recurrent_head", "true", "--use_wide_recurrent_observations", "true"])
    cfg.quiet = True
    net = PPONet(HostVecEnv(SmacShapedHost(d), wide_observations=True), cfg=cfg, device="cuda:0")
    agent = PPOAgent(net)
    agent.train(total_time_steps=0, logger=Logger(quiet=True))
    drv = agent.driver
    drv.actor_rollout()
    drv.compute_returns()
    b, tr, m = drv.buffer.data, drv.trainer, drv.trainer.algo_module
    assert tr.recurrent and (tr.d, tr.dc, tr.n) == (d, d, N_ACT)
    B = N_ENVS * A
    obs, acts, logp = b.policy_obs[0].view(B, d), b.actions[0].view(B, 1), b.action_log_probs[0].view(B, 1)
    am, masks = b.action_masks[0].view(B, N_ACT), b.masks[0].view(B)
    states = b.rnn_states[0:2].clone()   # slot 0 is read, slot 1 written: a copy, so the buffer keeps its rollout
    step = [0]

    def act():
        step[0] += 1
        m.act_rows(obs, acts, logp, 0, B, 7, step[0], action_masks=am, masks=masks, rnn_states=states)

    def critic():
        lib.check(drv._lib.orl_rnn_critic(drv._rnn_args(0, T, None), lib.current_stream()), "orl_rnn_critic")

    act_ms = device_ms(act, reps * 20)
    critic_ms = device_ms(critic, reps)
    update_ms = device_ms(lambda: tr.train(b), reps)
    return dict(d=d, act_ms_per_step=round(act_ms, 4), critic_ms=round(critic_ms, 3), update_ms_per_epoch=round(update_ms, 3))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--widths", type=int, nargs="+", default=[64, 80, 168, 256])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("wide_obs_gru_bench.py needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    rows = [measure(d, args.reps) for d in args.widths]
    print(json.dumps(dict(gpu=card, n_envs=N_ENVS, agents=A, steps=T, n_actions=N_ACT, chunk=8, results=rows)))


if __name__ == "__main__":
    main()
