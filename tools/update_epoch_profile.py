"""Where one epoch of the C2 tensor-core PPO update spends its time (CartPole-v1, 4096 envs, T = 128, built exactly as
bench.py builds it: one 524 288-row minibatch through ppo_fwdbwd_tc_kernel, ppo_reduce_kernel and ppo_apply_kernel).

Part 1 (the library as built): a few eager iterations under torch.profiler with CUDA activities; the mean time of each
of the three update kernels, the gaps between them, and their sum against bench's `phases_ms.update` (CUDA events
around the update phase of the same kind of eager iteration).

Part 2 (phase stamps): a copy of the library whose orl_ppo_tc.cu is compiled with -DORL_PROFILE_PHASES, built in a
temporary directory and run in a child process.  Every CTA of ppo_fwdbwd_tc_kernel stamps kernel entry, first tile
staged, tile loop end and kernel exit; per update epoch the script reports the prologue (entry -> first tile) and the
epilogue (loop end -> exit) of the policy and critic CTAs, their share of the kernel, and the wave-switch gap per SM
(the policy CTA's loop end to the critic CTA's first tile on the same SM).

The card's name, power limit and SM clock are read in the same run.
    python tools/update_epoch_profile.py [--iters 5] [--epochs 40] [--out DIR]"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KERNELS = ("ppo_fwdbwd_tc_kernel", "ppo_reduce_kernel", "ppo_apply_kernel")
PH_MAX_CTAS, PH_WORDS = 1024, 9   # orl_ppo_tc.cu: g_phases


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return r.stdout.strip()


def c2_driver():
    import torch

    import bench

    cfg, env, net, agent = bench.build_agent(0, 1, "c2")
    drv = bench.make_driver(cfg, env, net, agent, 0, 1)
    for _ in range(3):
        drv.device_iteration()
    torch.cuda.synchronize()
    assert drv.trainer.use_tensor_cores
    return drv


def kernel_name(name):
    for k in KERNELS:
        if k in name:
            return k
    return None


def profile_kernels(iters, out_dir):
    """Part 1: per-kernel means and the gaps fwdbwd -> reduce -> apply -> next fwdbwd, from a torch.profiler trace."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    drv = c2_driver()
    drv.phase_events = []   # eager iterations with CUDA events around each phase (as bench.py's phases_ms)
    for _ in range(iters):
        drv.device_iteration()
    torch.cuda.synchronize()
    upd = [a.elapsed_time(b) for name, a, b in drv.phase_events if name == "update"]
    drv.phase_events = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            drv.device_iteration()
        torch.cuda.synchronize()
    drv.phase_events = None
    path = os.path.join(out_dir, "update_epoch.pt.trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"]
    ev.sort(key=lambda e: e["ts"])
    dur = {k: [] for k in KERNELS}
    gaps = {"fwdbwd->reduce": [], "reduce->apply": [], "apply->next fwdbwd": []}
    for i, e in enumerate(ev):
        k = kernel_name(e["name"])
        if k is None:
            continue
        dur[k].append(e["dur"])
        nxt = ev[i + 1] if i + 1 < len(ev) else None
        if nxt is None:
            continue
        kn = kernel_name(nxt["name"])
        gap = nxt["ts"] - (e["ts"] + e["dur"])
        if k == KERNELS[0] and kn == KERNELS[1]:
            gaps["fwdbwd->reduce"].append(gap)
        elif k == KERNELS[1] and kn == KERNELS[2]:
            gaps["reduce->apply"].append(gap)
        elif k == KERNELS[2] and kn == KERNELS[0]:
            gaps["apply->next fwdbwd"].append(gap)
    epochs = len(dur[KERNELS[0]]) / max(iters, 1)
    print(f"part 1: {iters} eager iterations, {epochs:g} update epochs each")
    per_epoch = 0.0
    for k in KERNELS:
        m = statistics.mean(dur[k]) if dur[k] else float("nan")
        per_epoch += m
        print(f"  {k:24s} mean {m:8.2f} us  (n = {len(dur[k])}, min {min(dur[k]):.2f}, max {max(dur[k]):.2f})")
    gap_sum = 0.0
    for g, v in gaps.items():
        m = statistics.mean(v) if v else 0.0
        gap_sum += m
        print(f"  gap {g:20s} mean {m:8.2f} us  (n = {len(v)})")
    print(f"  per epoch: kernels {per_epoch:.1f} us + gaps {gap_sum:.1f} us = {per_epoch + gap_sum:.1f} us;"
          f" x {epochs:g} epochs = {(per_epoch + gap_sum) * epochs / 1e3:.3f} ms"
          f" against phases_ms.update {statistics.mean(upd):.3f} ms (mean of {len(upd)} eager iterations)")


def build_stamped_lib(tmp):
    """libopenrl_b200.so with orl_ppo_tc.cu compiled under -DORL_PROFILE_PHASES, the other objects as built."""
    from openrl_b200 import build as b

    b.build()
    objs = []
    for src in b.sources():
        if src == "orl_ppo_tc.cu":
            obj = os.path.join(tmp, "orl_ppo_tc_phases.o")
            cmd = [b.NVCC] + b.ARCH + b.COMMON + ["-DORL_PROFILE_PHASES", "-c", os.path.join(b.CSRC, src), "-o", obj]
            subprocess.run(cmd, check=True)
        else:
            obj = os.path.join(b.BUILD, src[:-3] + ".o")
        objs.append(obj)
    so = os.path.join(tmp, "libopenrl_b200_phases.so")
    subprocess.run([b.NVCC] + b.ARCH + ["-shared", "-Xcompiler", "-fPIC", "-o", so] + objs, check=True)
    return so


def summarize(xs):
    return f"mean {statistics.mean(xs):7.2f}  median {statistics.median(xs):7.2f}  max {max(xs):7.2f}"


def phase_stamps(lib_path, epochs):
    """Part 2 (child process): run `epochs` single update epochs on the stamped library and read the stamps of each."""
    import numpy as np
    import torch

    from openrl_b200 import lib

    lib._lib = lib.load(lib_path)
    read = lib._lib.orl_profile_phases_read
    read.argtypes = [ctypes.c_void_p]
    drv = c2_driver()
    tr, b = drv.trainer, drv.buffer.data
    G = tr.grid_per_net
    rows = b.episode_length * b.n_rollout_threads * b.num_agents
    stats = b.gae_stats[5:8]
    host = np.zeros((PH_MAX_CTAS, PH_WORDS), dtype=np.uint64)
    for _ in range(5):
        tr.ppo_update(b, rows, None, 0, mb_stats=stats)
    torch.cuda.synchronize()
    res = {k: [] for k in ("span", "pro_p", "pro_c", "epi_p", "epi_c", "pro_p_clk", "pro_c_clk", "epi_p_clk", "epi_c_clk",
                           "switch", "crit_path")}
    for _ in range(epochs):
        tr.ppo_update(b, rows, None, 0, mb_stats=stats)
        torch.cuda.synchronize()
        lib.check(read(host.ctypes.data), "orl_profile_phases_read")
        s = host[:2 * G].astype(np.int64)
        t0 = s[:, 0].min()
        gt, ck, sm = s[:, 0:4] - t0, s[:, 4:8], s[:, 8]
        pol, cri = slice(0, G), slice(G, 2 * G)
        res["span"].append((gt[:, 3].max() - gt[:, 0].min()) / 1e3)
        res["pro_p"].append((gt[pol, 1] - gt[pol, 0]).mean() / 1e3)
        res["pro_c"].append((gt[cri, 1] - gt[cri, 0]).mean() / 1e3)
        res["epi_p"].append((gt[pol, 3] - gt[pol, 2]).mean() / 1e3)
        res["epi_c"].append((gt[cri, 3] - gt[cri, 2]).mean() / 1e3)
        res["pro_p_clk"].append(float((ck[pol, 1] - ck[pol, 0]).mean()))
        res["pro_c_clk"].append(float((ck[cri, 1] - ck[cri, 0]).mean()))
        res["epi_p_clk"].append(float((ck[pol, 3] - ck[pol, 2]).mean()))
        res["epi_c_clk"].append(float((ck[cri, 3] - ck[cri, 2]).mean()))
        sw = []
        for c in range(G, 2 * G):   # the policy CTA that last left this critic CTA's SM before it started
            prev = [p for p in range(G) if sm[p] == sm[c] and gt[p, 3] <= gt[c, 0]]
            if prev:
                p = max(prev, key=lambda i: gt[i, 3])
                sw.append((gt[c, 1] - gt[p, 2]) / 1e3)
        res["switch"].append(statistics.mean(sw) if sw else float("nan"))
        res["crit_path"].append(res["pro_p"][-1] + res["epi_p"][-1] + res["pro_c"][-1] + res["epi_c"][-1])
    span = statistics.mean(res["span"])
    print(f"part 2: phase stamps of ppo_fwdbwd_tc_kernel, {epochs} update epochs, {G} CTAs per net "
          f"(globaltimer us; clock64 cycles for the per-CTA durations)")
    print(f"  kernel span (first entry -> last exit)      {summarize(res['span'])} us")
    for key, label in (("pro_p", "prologue, policy CTAs"), ("pro_c", "prologue, critic CTAs"),
                       ("epi_p", "epilogue, policy CTAs"), ("epi_c", "epilogue, critic CTAs")):
        print(f"  {label:42s} {summarize(res[key])} us  |  {statistics.mean(res[key + '_clk']):8.0f} cycles")
    print(f"  wave switch per SM (policy loop end -> critic first tile) {summarize(res['switch'])} us")
    cp = statistics.mean(res["crit_path"])
    print(f"  prologue + epilogue of both waves: {cp:.2f} us = {100 * cp / span:.1f} % of the kernel span "
          f"(prologues {statistics.mean(res['pro_p']) + statistics.mean(res['pro_c']):.2f} us, "
          f"epilogues {statistics.mean(res['epi_p']) + statistics.mean(res['epi_c']):.2f} us)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5, help="eager iterations under torch.profiler")
    ap.add_argument("--epochs", type=int, default=40, help="single update epochs read with phase stamps")
    ap.add_argument("--out", default=None, help="directory for the profiler trace (default: a temporary directory)")
    ap.add_argument("--stamped-lib", default=None, help=argparse.SUPPRESS)   # the child process of part 2
    args = ap.parse_args()
    if args.stamped_lib:
        phase_stamps(args.stamped_lib, args.epochs)
        return
    print(f"GPU: {gpu_info()}")
    with tempfile.TemporaryDirectory() as tmp:
        out = args.out or tmp
        os.makedirs(out, exist_ok=True)
        profile_kernels(args.iters, out)
        so = build_stamped_lib(tmp)
        sys.stdout.flush()
        subprocess.run([sys.executable, os.path.abspath(__file__), "--stamped-lib", so, "--epochs", str(args.epochs)], check=True)
    print(f"GPU: {gpu_info()}")


if __name__ == "__main__":
    main()
