#!/usr/bin/env python
"""One training iteration of CartPole-GRU PPO with the env stepped on the host, both host loops, and the feed-forward
host path at the same shape for context.

1024 envs, T = 128, the numpy CartPole of oracle/envs.py stepped in a Python loop (the host side of the path), Philox
sampling, data_chunk_length 16, the default epochs / minibatches.  Per mode: CUDA events around every act launch
(orl_rnn_act_rows, or orl_rollout with ORL_ENV_NONE for the MLP), around the critic and update phases and around the
whole iteration (rollout -> returns -> update -> after_update); the numpy env alone is timed over T steps with uniform
random actions.  An act event pair also spans the Python that fills the launch arguments.  Modes are timed alternately: `--rounds` rounds of `--iters` iterations each, after `--warmup` iterations of
each.  Prints the card name, power limit and clocks read in the same run, and one JSON line.  `--masked`: every env
reports `info["action_masks"]` on every step (a fixed random row per env, action 0 always legal), so the iteration also
stages, uploads, inserts and applies the masks: the per-step cost of mask ingest is the difference to a run without.
`--dict-obs`: instead, a SMAC-3m-shaped GRU MAPPO workload (3 agents, policy obs 30, 8 actions, per-agent masks every
step, an env ends every 20 steps, staggered) whose host env replays a fixed pool of observations, timed with a flat
Box(30) observation and with Dict {"policy": Box(30), "critic": Box(48)}: the cost of the critic section (staged,
uploaded, inserted, and read by the critic and the update) is the difference between the two.

    python tools/rnn_host_bench.py [--envs 1024 --T 128 --iters 3 --rounds 2 --warmup 2 --masked | --dict-obs]
"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    import torch

    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                            f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


class CartPoleHost:
    """The numpy CartPole vec-env with the reference's duck type; `step_range` steps envs [lo, hi) (two-group loop)."""

    def __init__(self, n, masked=False):
        from openrl_b200 import spaces
        from oracle.envs import CartPoleVec

        self.inner = CartPoleVec(n)
        self.mask_rows = None
        if masked:
            self.mask_rows = (np.random.default_rng(1).random((n, 2)) < 0.5).astype(np.int8)
            self.mask_rows[:, 0] = 1
        self.parallel_env_num, self.agent_num = n, 1
        self.observation_space = spaces.Box(-np.inf, np.inf, (4,), np.float32)
        self.action_space = spaces.Discrete(2)

    def reset(self, seed=None):
        return self.inner.reset(seed=seed)

    def step(self, actions):
        return self.step_range(0, self.parallel_env_num, actions)

    def step_range(self, lo, hi, actions):
        sub = copy.copy(self.inner)
        sub.N, sub.rng, sub.state, sub.elapsed = hi - lo, self.inner.rng[lo:hi], self.inner.state[lo:hi], self.inner.elapsed[lo:hi]
        o, r, d, _ = sub.step(actions)
        if self.mask_rows is not None:
            return o, r, d, [{"action_masks": m} for m in self.mask_rows[lo:hi]]
        return o, r, d, [{} for _ in range(hi - lo)]


class Smac3mHost:
    """SMAC-3m-shaped host vec-env: A = 3 agents, policy obs 30 and, with `critic`, a Dict space with a 48-wide critic
    obs; Discrete(8) with per-agent (A, 8) masks on every step; env e ends at steps where (t + e) % 20 == 19.  The
    observations replay a fixed random pool, so the host side costs little beyond the staging."""
    A, D, DC, N_ACT, POOL = 3, 30, 48, 8, 8

    def __init__(self, n, critic=False):
        from openrl_b200 import spaces

        g = np.random.default_rng(0)
        box = lambda w: spaces.Box(-np.inf, np.inf, (w,), np.float32)  # noqa: E731
        self.parallel_env_num, self.agent_num, self.critic = n, self.A, critic
        self.observation_space = spaces.Dict({"policy": box(self.D), "critic": box(self.DC)}) if critic else box(self.D)
        self.action_space = spaces.Discrete(self.N_ACT)
        self.pol = g.standard_normal((self.POOL, n, self.A, self.D)).astype(np.float32)
        self.cri = g.standard_normal((self.POOL, n, self.A, self.DC)).astype(np.float32)
        m = (g.random((n, self.A, self.N_ACT)) < 0.6).astype(np.int8)
        m[..., 0] = 1
        self.infos = [{"action_masks": m[e]} for e in range(n)]
        self.rewards = g.standard_normal((n, self.A, 1))
        self.t = 0

    def _obs(self, lo, hi):
        k = self.t % self.POOL
        return {"policy": self.pol[k, lo:hi], "critic": self.cri[k, lo:hi]} if self.critic else self.pol[k, lo:hi]

    def reset(self, seed=None):
        self.t = 0
        return self._obs(0, self.parallel_env_num), self.infos

    def step(self, actions):
        return self.step_range(0, self.parallel_env_num, actions)

    def step_range(self, lo, hi, actions):
        if hi == self.parallel_env_num:
            self.t += 1
        dones = np.repeat(((self.t + np.arange(lo, hi)) % 20 == 19)[:, None], self.A, axis=1)
        return self._obs(lo, hi), self.rewards[lo:hi], dones, self.infos[lo:hi]


def build(n, T, recurrent, grouped, masked=False, dict_obs=None):
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.vec_env import HostVecEnv
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.logger import Logger

    cfg = create_config_parser().parse_args(["--seed", "1", "--episode_length", str(T), "--data_chunk_length", "16",
                                             "--use_recurrent_policy", "true" if recurrent else "false",
                                             "--host_env_groups", "true" if grouped else "false"])
    cfg.quiet = True
    host = CartPoleHost(n, masked) if dict_obs is None else Smac3mHost(n, critic=dict_obs)
    agent = PPOAgent(PPONet(HostVecEnv(host), cfg=cfg, device="cuda:0"))
    agent.train(total_time_steps=0, logger=Logger(quiet=True))   # trainer / buffer / driver, envs reset
    drv = agent.driver
    assert drv.recurrent == recurrent
    acts = []
    inner = drv._act   # the act launches: one per group and step

    def timed(*a, **k):
        import torch

        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = inner(*a, **k)
        e1.record()
        acts.append((e0, e1))
        return out

    drv._act = timed
    return drv, acts


def iteration(drv, acts):
    """One iteration; returns {iteration, act (sum), critic, update} in ms and the number of act launches timed."""
    import torch

    drv.phase_events = []
    acts.clear()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    drv.actor_rollout()
    drv.learner_update()
    drv.buffer.after_update()
    e1.record()
    torch.cuda.synchronize()
    out = {"iteration": e0.elapsed_time(e1), "act": 0.0, "critic": 0.0, "update": 0.0}
    n_act = 0
    for name, a, b in drv.phase_events:
        if name in ("critic", "update"):
            out[name] += a.elapsed_time(b)
    for a, b in acts:
        out["act"] += a.elapsed_time(b)
        n_act += 1
    drv.phase_events = None
    drv.episode += 1
    return out, n_act


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=1024)
    ap.add_argument("--T", type=int, default=128)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--masked", action="store_true", help="the envs report action masks on every step")
    ap.add_argument("--dict-obs", action="store_true",
                    help="a SMAC-3m-shaped GRU workload, with and without a 48-wide critic observation")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("rnn_host_bench needs a CUDA device")
    modes = {}
    variants = [(True, None), (False, None)] if not args.dict_obs else [(True, False), (True, True)]
    for recurrent, dict_obs in variants:
        for grouped in (False, True):
            drv, acts = build(args.envs, args.T, recurrent, grouped, args.masked, dict_obs)
            for _ in range(args.warmup):
                iteration(drv, acts)
            tag = "gru" if recurrent else "mlp"
            if dict_obs is not None:
                tag += "_critic48" if dict_obs else "_box"
            modes[tag + ("_grouped" if grouped else "_sync")] = (drv, acts)
    samples = {m: [] for m in modes}
    for _ in range(args.rounds):
        for m, (drv, acts) in modes.items():
            for _ in range(args.iters):
                samples[m].append(iteration(drv, acts))
    # the host env alone: T steps of the numpy CartPole with uniform random actions (what an untrained policy takes)
    host = CartPoleHost(args.envs) if not args.dict_obs else Smac3mHost(args.envs, critic=True)
    host.reset(seed=0)
    acts_host = np.random.default_rng(0).integers(0, 2, size=(args.T, args.envs, host.agent_num, 1))
    t0 = time.perf_counter()
    for t in range(args.T):
        host.step(acts_host[t])
    env_ms = (time.perf_counter() - t0) * 1e3
    name, q = card()
    workload = (f"CartPole host-stepped (numpy env), {args.envs} envs" if not args.dict_obs else
                f"SMAC-3m-shaped host env (3 agents, obs 30, 8 actions, masks every step; critic obs 48 in the critic48 "
                f"modes), {args.envs} envs")
    res = {"workload": workload + f", T={args.T}, Philox sampling, data_chunk_length 16"
                       + (", action masks reported on every step" if args.masked else ""),
           "card": name, "power_limit,clocks.sm,clocks.max.sm": q, "host_env_only_ms_per_iteration": round(env_ms, 2),
           "iterations_per_mode": args.rounds * args.iters, "modes": {}}
    for m, s in samples.items():
        it = [x["iteration"] for x, _ in s]
        n_act = s[0][1]
        act = [x["act"] for x, _ in s]
        res["modes"][m] = {"iteration_ms_median": round(statistics.median(it), 2), "iteration_ms_min": round(min(it), 2),
                           "iteration_ms_max": round(max(it), 2),
                           "env_steps_per_s": round(args.envs * args.T / (statistics.median(it) * 1e-3)),
                           "act_launches_per_iteration": n_act, "act_ms_per_iteration_median": round(statistics.median(act), 3),
                           "act_us_per_launch": round(statistics.median(act) / max(n_act, 1) * 1e3, 2),
                           "critic_ms_median": round(statistics.median(x["critic"] for x, _ in s), 3),
                           "update_ms_median": round(statistics.median(x["update"] for x, _ in s), 3)}
    print(f"[rnn_host_bench] {name} | power.limit, clocks.sm, clocks.max.sm: {q}", file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
