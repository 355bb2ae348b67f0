"""GAE kernel micro-benchmark: CUDA-event timing of orl_gae at the BASELINE config shapes and
at a >= 1 GB shape, reported against the HBM peak (MEASURED_PEAKS.json, else the H100 SXM data sheet).
Prints one JSON line per shape; `python tools/gae_micro.py OUT.json` also writes the list to OUT.json."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from openrl_b200 import lib  # noqa: E402


def peak_hbm():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        return json.load(open(p))["hbm_gbs"], "measured"
    return 3350.0, "datasheet"


def bench_shape(L, T, B, flags=5, adv=True, stats=True, iters=20, flush=None):
    dev = torch.device("cuda:0")
    r = torch.randn(T, B, device=dev)
    vp = torch.randn(T + 1, B, device=dev)
    m = (torch.rand(T + 1, B, device=dev) > 0.01).float()
    act = torch.ones(T + 1, B, device=dev)
    nv = torch.randn(B, device=dev)
    vn = torch.tensor([0.3, 2.0, 0.5], device=dev)
    ret = torch.empty(T + 1, B, device=dev)
    a = torch.empty(T, B, device=dev) if adv else None
    st = torch.empty(8, dtype=torch.float64, device=dev) if stats else None
    s = torch.cuda.current_stream().cuda_stream

    def call():
        lib.check(L.orl_gae(lib.ptr(r), lib.ptr(vp), lib.ptr(m), None, lib.ptr(act) if stats else None, lib.ptr(nv),
                            lib.ptr(vn), lib.ptr(ret), lib.ptr(a), lib.ptr(st), T, B, 0.99, 0.95, flags, s), "gae")

    for _ in range(3):
        call()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1e-3)
    times.sort()
    med = times[len(times) // 2]
    per_el = 16 + (4 if adv else 0) + (4 if stats else 0)
    return {"T": T, "B": B, "bytes_per_el": per_el, "median_s": med, "min_s": times[0],
            "GBps_median": T * B * per_el / med / 1e9, "GBps_best": T * B * per_el / times[0] / 1e9}


def main():
    L = lib.load()
    peak, how = peak_hbm()
    flush = torch.empty(256 * 1024 * 1024 // 4, device="cuda:0")  # 256 MB > 50 MB L2
    out = []
    for name, T, B in [("C2 cartpole 4096", 128, 4096), ("C3 mpe 2048x3", 25, 6144), ("C4 gridworld 4096x2", 128, 8192),
                       ("C5 cheetah 1024", 128, 1024), ("1GB+ T128 B2^21", 128, 1 << 21)]:
        for adv, stats in [(False, False), (True, True)]:
            r = bench_shape(L, T, B, adv=adv, stats=stats, flush=flush)
            r["name"] = name
            r["frac_of_%s_hbm_peak" % how] = r["GBps_median"] / peak
            out.append(r)
            print(json.dumps(r))
    if len(sys.argv) > 1:
        json.dump(out, open(sys.argv[1], "w"), indent=1)


if __name__ == "__main__":
    main()
