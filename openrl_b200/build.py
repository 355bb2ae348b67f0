"""In-tree nvcc build of libopenrl_b200.so for sm_90a (H100).

`python -m openrl_b200.build` (or __graft_entry__.build()).  nvcc cross-compiles without a
GPU; the .so is git-ignored but travels to the GPU box with the repo snapshot.
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")
BUILD = os.path.join(CSRC, "build")
LIB = os.path.join(CSRC, "libopenrl_b200.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-I", INCLUDE, "-I", CSRC]
# per-file extra flags: the GAE scan must reproduce numpy's unfused float32 arithmetic
EXTRA = {"orl_gae.cu": ["--fmad=false"]}


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(paths):
    h = hashlib.sha256()
    for p in paths:
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def _deps():
    hdrs = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cuh", ".h"))]
    hdrs += [os.path.join(INCLUDE, f) for f in sorted(os.listdir(INCLUDE))]
    return hdrs


def build(verbose=False, force=False):
    os.makedirs(BUILD, exist_ok=True)
    hdr_digest = _digest(_deps() + [os.path.abspath(__file__)])
    objs, jobs = [], []
    for src in sources():
        spath = os.path.join(CSRC, src)
        obj = os.path.join(BUILD, src[:-3] + ".o")
        stamp = obj + ".sha"
        want = _digest([spath]) + hdr_digest
        objs.append(obj)
        have = open(stamp).read() if os.path.exists(stamp) and os.path.exists(obj) else ""
        if force or have != want:
            cmd = [NVCC] + ARCH + COMMON + EXTRA.get(src, []) + (["-Xptxas", "-v"] if verbose else []) + ["-c", spath, "-o", obj]
            jobs.append((cmd, stamp, want))

    def run(job):
        cmd, stamp, want = job
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        if verbose:
            sys.stderr.write(r.stderr)
        with open(stamp, "w") as f:
            f.write(want)

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(run, jobs))
    if jobs or not os.path.exists(LIB):
        cmd = [NVCC] + ARCH + ["-shared", "-Xcompiler", "-fPIC", "-o", LIB] + objs
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    return LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
