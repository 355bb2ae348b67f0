"""Time the C2 PPO update (CartPole-v1, 4096 envs, T = 128: one 524 288-row minibatch through the tensor-core update
kernel, reduce and apply) with CUDA events, on one real rollout buffer.  Prints the GPU, its power limit, and the median
and spread of per-update times over several windows.
    python tools/tc_update_time.py [--updates 200] [--windows 5]"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=200)
    ap.add_argument("--windows", type=int, default=5)
    args = ap.parse_args()
    cfg, env, net, agent = bench.build_agent(0, 1, "c2")
    drv = bench.make_driver(cfg, env, net, agent, 0, 1)
    drv.device_iteration()                    # warm every kernel once
    drv.actor_rollout()
    drv.compute_returns()
    tr, b = drv.trainer, drv.buffer.data
    assert tr.use_tensor_cores
    rows = b.episode_length * b.n_rollout_threads * b.num_agents
    stats = b.gae_stats[5:8]
    for _ in range(20):
        tr.ppo_update(b, rows, None, 0, mb_stats=stats)
    torch.cuda.synchronize()
    times = []
    for _ in range(args.windows):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.updates):
            tr.ppo_update(b, rows, None, 0, mb_stats=stats)
        t1.record()
        torch.cuda.synchronize()
        times.append(t0.elapsed_time(t1) * 1e3 / args.updates)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    times.sort()
    print(f"GPU: {gpu}")
    print(f"C2 update ({rows} rows, {tr.grid_per_net} CTAs per net): median {times[len(times) // 2]:.1f} us, "
          f"min {times[0]:.1f} us, max {times[-1]:.1f} us over {args.windows} windows of {args.updates} updates")


if __name__ == "__main__":
    main()
