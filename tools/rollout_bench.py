#!/usr/bin/env python
"""Time of the fused device rollout (`orl_rollout`, one launch over T steps) alone, at the C2 shape.

bench.py's C2 workload (T = 128, MLP 64x64, device sampling) on `--env` (default CartPole-v1; GridWorldEnv runs
rollout_tc_kernel, which no bench workload times) at each of `--envs` (default 128 and 4096: the latency of one CTA's
step chain, and the full grid).  CUDA events around each of `--launches` launches after
`--warmup` launches; the env state simply carries on from launch to launch.  Reports microseconds per step (median and
range over launches), SM cycles per step at the SM clock read right after the timed launches, and the card's name, power
limit, maximum SM clock and active clock-event (throttle) reasons, read in the same run.  Prints one JSON line.

    python tools/rollout_bench.py [--env CartPole-v1 --envs 128,4096 --launches 50 --warmup 10]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def smi(fields):
    import torch

    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader", f"--id={torch.cuda.current_device()}"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--env", default="CartPole-v1")
    ap.add_argument("--envs", default="128,4096")
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()

    import torch

    import bench
    from openrl_b200 import lib

    if not torch.cuda.is_available():
        raise SystemExit("rollout_bench needs a CUDA device")
    workload = "c2" if args.env == bench.WORKLOADS["c2"]["env"] else "c2_" + args.env
    bench.WORKLOADS.setdefault(workload, dict(bench.WORKLOADS["c2"], env=args.env))
    out = {"card": torch.cuda.get_device_name(), "name,power_limit,max_sm_clock": smi("name,power.limit,clocks.max.sm"),
           "env": args.env, "T": bench.T, "results": {}}
    for n in (int(x) for x in args.envs.split(",")):
        cfg, env, net, agent = bench.build_agent(0, 1, workload, n)
        drv = bench.make_driver(cfg, env, net, agent, 0, 1)
        drv.trainer.prep_rollout()
        L, s, T = lib.load(), lib.current_stream(), drv.episode_length
        a = drv._rollout_args(0, T, None)
        for _ in range(args.warmup):
            lib.check(L.orl_rollout(a, s), "orl_rollout")
        ev = []
        for _ in range(args.launches):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            lib.check(L.orl_rollout(a, s), "orl_rollout")
            e1.record()
            ev.append((e0, e1))
        torch.cuda.synchronize()
        clock = smi("clocks.sm,clocks_event_reasons.active")
        us = sorted(e0.elapsed_time(e1) * 1e3 / T for e0, e1 in ev)
        med = us[len(us) // 2]
        try:
            mhz = float(clock.split(",")[0].split()[0])
        except (ValueError, IndexError):
            mhz = float("nan")
        out["results"][str(n)] = {"us_per_step_median": round(med, 3), "us_per_step_range": [round(us[0], 3), round(us[-1], 3)],
                                  "ms_per_launch_median": round(med * T * 1e-3, 4), "sm_clock_mhz,event_reasons": clock,
                                  "cycles_per_step": round(med * mhz)}
        del drv, agent, net, env
    print(json.dumps(out))


if __name__ == "__main__":
    main()
