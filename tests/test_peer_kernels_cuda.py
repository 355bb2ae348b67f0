"""Single-GPU checks of the peer-memory exchange kernels (include/openrl_b200.h: OrlPeerArgs).  The multi-process,
multi-GPU behaviour is covered by tests/test_multi_gpu_cuda.py / tools/multi_gpu_check.py; here a two-rank world is
emulated inside one process (two buffers on the same device stand for the two ranks' symmetric allocations), which is
enough for the push half: orl_ppo_reduce_peer must write exactly the sums orl_ppo_reduce writes, into slot
[parity of epochs[net]][rank][net] of EVERY rank's allocation, and nothing else."""
import numpy as np
import pytest

from conftest import GOLDEN

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("rank", [0, 1])
@pytest.mark.parametrize("epochs", [(0, 0), (1, 0), (2, 5)])
def test_reduce_peer_pushes_the_sums_of_reduce_into_every_ranks_slot(cuda, rank, epochs):
    import os

    import torch

    from openrl_b200 import lib
    from helpers import load_buffer, ppo_update_setup

    d = np.load(os.path.join(GOLDEN, "trace_cartpole.npz"), allow_pickle=True)
    cfg, net, trainer, buf = ppo_update_setup(d)
    load_buffer(buf, d, 0)
    L, s = lib.load(), lib.current_stream()
    stride, G, W = trainer.stride, trainer.grid_per_net, 2
    gen = torch.Generator(device="cuda").manual_seed(3)
    trainer.partials.copy_(torch.randn(trainer.partials.shape, device="cuda", generator=gen))
    total = cfg.episode_length * int(d["meta/env_num"])
    a = trainer._args(buf.data, total, None, 0)
    lib.check(L.orl_ppo_reduce(a, s), "orl_ppo_reduce")
    want = trainer.folded.clone()

    nbytes = L.orl_ppo_peer_bucket_bytes(trainer.d, trainer.dc, trainer.n, W)
    bufs = [torch.zeros(nbytes // 4, dtype=torch.float32, device="cuda") for _ in range(W)]
    ptrs = torch.tensor([b.data_ptr() for b in bufs], dtype=torch.int64, device="cuda")
    ep = torch.tensor(list(epochs) + [0, 0], dtype=torch.int32, device="cuda")
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    summed = torch.zeros(2, stride, dtype=torch.float32, device="cuda")
    pa = lib.OrlPeerArgs()
    pa.peer_buffers, pa.local_buffer = ptrs.data_ptr(), bufs[rank].data_ptr()
    pa.epochs, pa.error_flag, pa.summed = ep.data_ptr(), err.data_ptr(), summed.data_ptr()
    pa.world, pa.rank, pa.timeout_ms = W, rank, 1000
    lib.check(L.orl_ppo_reduce_peer(a, pa, s), "orl_ppo_reduce_peer")
    torch.cuda.synchronize()
    for b in bufs:
        slots = b[: 2 * W * 2 * stride].view(2, W, 2, stride)
        expect = torch.zeros_like(slots)
        for net in (0, 1):
            expect[epochs[net] & 1, rank, net] = want[net]
        assert torch.equal(slots, expect)
        assert int(b[2 * W * 2 * stride:].abs().sum().item()) == 0      # flags / small area untouched
    assert ep.tolist()[:2] == list(epochs) and int(err.item()) == 0
