#!/usr/bin/env python
"""Whole-iteration time of recurrent MAPPO with and without joint-action PPO (JRPO) at the C3 shape.

simple_spread, 2048 envs x 3 agents, T = 25, data_chunk_length 2, the examples/mpe/mpe_jrpo.yaml flags (GRU, ValueNorm,
advantage normalisation), 10 epochs (the default) x 1 minibatch: bench.py's C3 extra plus the JRPO flag.  The two trainers live in one process and are timed
alternately: `--rounds` rounds of `--iters` iterations each (collect + GAE + update through
OnPolicyDriver.device_iteration, the captured CUDA graph when eligible), CUDA events around every iteration, after
`--warmup` iterations of each.  Prints the card name and power limit and one JSON line.

    python tools/jrpo_bench.py [--iters 10 --rounds 3 --warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    import torch

    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                            f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--envs", type=int, default=2048)
    args = ap.parse_args()

    import torch

    import bench

    if not torch.cuda.is_available():
        raise SystemExit("jrpo_bench needs a CUDA device")
    drivers = {}
    for mode, extra in (("mappo", []), ("jrpo", ["--use_joint_action_loss", "true"])):
        cfg, env, net, agent = bench.build_agent(0, 1, "c3", args.envs, extra)
        drv = bench.make_driver(cfg, env, net, agent, 0, 1)
        assert drv.trainer.joint_action == (mode == "jrpo")
        for _ in range(args.warmup):
            drv.device_iteration()
        drivers[mode] = drv
    torch.cuda.synchronize()
    times = {m: [] for m in drivers}
    for _ in range(args.rounds):
        for mode, drv in drivers.items():
            ev = []
            for _ in range(args.iters):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                drv.device_iteration()
                e1.record()
                ev.append((e0, e1))
            torch.cuda.synchronize()
            times[mode].append(sum(a.elapsed_time(b) for a, b in ev) / args.iters)
    name, power = card()
    out = {"card": name, "power_limit,max_sm_clock": power,
           "workload": f"simple_spread {args.envs} envs x 3 agents, T=25, L=2, mpe_jrpo.yaml flags, "
                       f"{drivers['mappo'].trainer.ppo_epoch} epochs x 1 minibatch",
           "ms_per_iteration": {m: [round(t, 3) for t in v] for m, v in times.items()},
           "median_ms": {m: round(sorted(v)[len(v) // 2], 3) for m, v in times.items()},
           "cuda_graph": {m: getattr(d.trainer, "_iter_graph", None) is not None for m, d in drivers.items()}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
