"""Multi-GPU plumbing: one process per GPU, torch.distributed (NCCL over NVLink) for the two
exchange steps of the path (SURVEY.md §8e):

  1. once per iteration: SUM all-reduce of the 8 float64 rollout moments (advantage / return sums
     and counts, `orl_gae` stats) so that advantage normalisation (ppo.py:402-409), masked-mean
     denominators (ppo.py:213-217,315-317) and ValueNorm batch moments (valuenorm.py:64-65) are the
     global-batch values;
  2. once per update: SUM of the folded gradient bucket `folded` (2*stride floats, 37 KB for CartPole) between the
     reduce and the optimiser step.
For the feed-forward update both steps run INSIDE our kernels over NVLink peer memory (`PeerBucket` below,
orl_ppo_reduce_peer / orl_ppo_apply_peer / orl_peer_sum_f64; DESIGN.md §4.5); the NCCL all-reduce is the fallback (ORL_PEER_APPLY=0 or no peer mapping) and carries the recurrent and
shared-network buckets.

Rollouts shard over envs: rank r owns global envs [r*N, (r+1)*N) and seeds them exactly as the
unsharded vec-env would (seed + global_index*10086, sync_venv.py:137); no exchange during
collection or GAE.  The reference has no working distributed path (SURVEY.md §0.3): this is new
design.  The same functions run on CPU tensors with the gloo backend (tests/test_multiproc_cpu.py).
"""
import os

import torch.distributed as dist


_FORCE_SINGLE = False


def force_single_process(on=True):
    """Make this process behave as an unsharded run even though a process group exists (used by the multi-GPU
    equivalence check, which runs the global-batch reference on rank 0 next to the sharded run)."""
    global _FORCE_SINGLE
    _FORCE_SINGLE = bool(on)


def is_distributed():
    return (not _FORCE_SINGLE) and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


def world_size():
    return dist.get_world_size() if is_distributed() else 1


def rank():
    return dist.get_rank() if is_distributed() else 0


def allreduce_sum_(t):
    """In-place SUM all-reduce (no-op for a single process)."""
    if is_distributed():
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return t


# ---- alternative for the fallback path: torch's symmetric-memory one-shot all-reduce -----------------------------------
# ORL_SYMM_ALLREDUCE=1 (with ORL_PEER_APPLY=0): every rank reads all peers' buffers over NVLink and sums locally (signal-pad
# barriers, graph-capturable) instead of NCCL; the fused PeerBucket path supersedes it.  Any failure to set the
# symmetric path up falls back to NCCL.
_SYMM = {}   # data_ptr -> (symmetric input tensor, output tensor, group name)


def symmetric_buffer(shape, dtype, device):
    """A tensor to be SUM-all-reduced with `allreduce_sum_into`: symmetric memory when available (> 1 rank, float32),
    else a plain tensor.  Returns (buffer, reduced) — `reduced` receives the sum (the buffer itself in the NCCL path)."""
    import os

    import torch

    t = None
    if is_distributed() and dtype == torch.float32 and os.environ.get("ORL_SYMM_ALLREDUCE", "0") == "1":
        try:
            import torch.distributed._symmetric_memory as symm_mem

            group = dist.group.WORLD
            t = symm_mem.empty(*shape, dtype=dtype, device=device)
            t.zero_()
            symm_mem.rendezvous(t, group.group_name)
            out = torch.zeros(*shape, dtype=dtype, device=device)
            torch.ops.symm_mem.one_shot_all_reduce_out(t, "sum", group.group_name, out)   # first use: sets up / validates the path
            torch.cuda.synchronize()
            _SYMM[t.data_ptr()] = (t, out, group.group_name)
            return t, out
        except Exception as e:  # noqa: BLE001
            import warnings

            warnings.warn(f"openrl_b200: symmetric-memory all-reduce unavailable ({type(e).__name__}: {e}); using NCCL")
            t = None
    import torch as _t

    t = _t.zeros(*shape, dtype=dtype, device=device)
    return t, t


def allreduce_sum_into(t):
    """SUM all-reduce of a buffer from `symmetric_buffer`; returns the tensor that holds the result."""
    ent = _SYMM.get(t.data_ptr())
    if ent is not None and is_distributed():
        import torch

        torch.ops.symm_mem.one_shot_all_reduce_out(ent[0], "sum", ent[2], ent[1])
        return ent[1]
    return allreduce_sum_(t)


class PeerBucket:
    """The gradient bucket of the feed-forward update as a symmetric allocation mapped into every peer over NVLink:
    orl_ppo_reduce_peer pushes this rank's bucket into every rank's copy, orl_ppo_apply_peer signals / waits / sums the slots and applies
    the optimiser step in the same kernel (include/openrl_b200.h, OrlPeerArgs) — no separate collective per update.
    `create` returns None (callers then use the all-reduce path) when there is one process, when ORL_PEER_APPLY=0, or
    when ANY rank fails to set the symmetric mapping up (the ranks agree on that with one MIN all-reduce)."""

    def __init__(self, sym, handle, stride, device):
        import torch

        from . import lib

        self.sym, self.handle = sym, handle        # keep the allocation and its rendezvous handle alive
        self.epochs = torch.zeros(4, dtype=torch.int32, device=device)
        self.error_flag = torch.zeros(1, dtype=torch.int32, device=device)
        self.summed = torch.zeros(2, stride, dtype=torch.float32, device=device)
        a = lib.OrlPeerArgs()
        a.peer_buffers = int(handle.buffer_ptrs_dev)
        a.local_buffer = sym.data_ptr()
        a.epochs, a.error_flag, a.summed = lib.ptr(self.epochs), lib.ptr(self.error_flag), lib.ptr(self.summed)
        a.world, a.rank = int(handle.world_size), int(handle.rank)
        a.timeout_ms = int(os.environ.get("ORL_PEER_TIMEOUT_MS", "60000"))
        self.args = a

    def check(self):
        """Raise if a peer's bucket did not arrive in time (called when the poisoned statistics are read back)."""
        e = int(self.error_flag.item())
        if e:
            raise RuntimeError(f"openrl_b200: rank {e - 1} did not deliver its gradient bucket within "
                               f"{self.args.timeout_ms} ms (orl_ppo_apply_peer); the ranks are out of step or one has died")

    @staticmethod
    def create(nbytes, stride, device):
        import torch

        if not is_distributed() or os.environ.get("ORL_PEER_APPLY", "1") == "0":
            return None
        from . import lib

        ok, sym, handle, why = 1, None, None, ""
        try:
            if dist.get_world_size() > lib.PEER_MAX_WORLD:
                raise RuntimeError(f"world size > {lib.PEER_MAX_WORLD}")
            import torch.distributed._symmetric_memory as symm_mem

            group = dist.group.WORLD
            sym = symm_mem.empty((nbytes + 3) // 4, dtype=torch.float32, device=device)
            sym.zero_()
            handle = symm_mem.rendezvous(sym, group.group_name)
            int(handle.buffer_ptrs_dev)
        except Exception as e:  # noqa: BLE001
            ok, why = 0, f"{type(e).__name__}: {e}"
        flag = torch.tensor([ok], dtype=torch.int32, device=device)
        if torch.device(device).type == "cuda":
            torch.cuda.synchronize(device)        # the zero-fill has landed before any peer may signal into it
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        if int(flag.item()) == 0:
            import warnings

            warnings.warn("openrl_b200: NVLink peer-memory gradient exchange unavailable"
                          + (f" ({why})" if why else " (on another rank)") + "; using the NCCL all-reduce")
            return None
        return PeerBucket(sym, handle, stride, device)


def env_shard(global_envs, r=None, w=None):
    """(first global env index, number of envs) of rank r when `global_envs` envs are split evenly."""
    r = rank() if r is None else r
    w = world_size() if w is None else w
    if global_envs % w != 0:
        raise ValueError(f"global env count {global_envs} must be divisible by the world size {w}")
    n = global_envs // w
    return r * n, n
