"""CPU emulation of the DEVICE recurrent update pipeline against the unmodified reference's trace
(tests/golden/trace_cartpole_gru.npz: single agent, data_chunk_length 4, two minibatches per epoch, ValueNorm,
episodes ending inside chunks).

Everything the device does is replayed with the same building blocks and the same assembly, on the CPU:
  chunk -> buffer-row mapping            openrl_b200.buffers.replay_data.chunk_row_indices (the product helper)
  chunked forward / BPTT, per-row tape   openrl_b200/csrc/orl_rnn_core.h compiled by g++ (the sequential statement of the
                                         step that orl_rnn_warp.cuh runs warp-cooperatively and is checked against)
  per-step losses and dL/dout            numpy restatement of orl_loss.cuh (pg_term, value_term) as used in
                                         rnn_chunk_warp_kernel: active-mask weights 1/sum(active), entropy bonus
  dW = sum P^T Q tape reductions         the job table of orl_rnn.cu::make_jobs
  clip + Adam + ValueNorm commit         rnn_apply_kernel
and the six scalars of every update plus the parameters after the iteration must equal the reference's."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import loop, nets, ppo
import rnn_pipeline_helpers as hp
from helpers import gxx_shim


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return gxx_shim(tmp_path_factory, "rnn", "rnn_core_shim.cpp")


def test_device_recurrent_pipeline_on_cpu_matches_reference_trace(shim):
    d = np.load(os.path.join(GOLDEN, "trace_cartpole_gru.npz"), allow_pickle=True)
    cfg = loop.cfg_from_flags(str(d["meta/flags"]))
    N, T, L, dim, n = int(d["meta/env_num"]), cfg.episode_length, cfg.data_chunk_length, 4, 2
    B = N
    torch.manual_seed(0)
    order_p = list(nets.init_policy(cfg, dim, "Discrete", n).keys())
    order_c = list(nets.init_critic(cfg, dim).keys())
    Pp = np.concatenate([d[f"init/policy.{k}"].reshape(-1) for k in order_p]).astype(np.float64)
    Pc = np.concatenate([d[f"init/critic.{k}"].reshape(-1) for k in order_c]).astype(np.float64)
    assert shim.shim_param_count(dim, n) == Pp.size and shim.shim_param_count(dim, 1) == Pc.size
    opt_p, opt_c = hp._Adam(Pp.size, cfg.lr, cfg.opti_eps), hp._Adam(Pc.size, cfg.critic_lr, cfg.opti_eps)
    vn = ppo.ValueNormState()

    def targets(rb):   # ValueNorm.update with this minibatch's returns, then normalise them (valuenorm.py:59-90)
        x = torch.from_numpy(rb.astype(np.float32)).view(-1, 1)
        vn.update(x)
        return vn.normalize(x).numpy()[:, 0].astype(np.float64)

    for it in range(int(d["meta/iters"])):
        g = lambda k: d[f"it{it}/{k}"]  # noqa: E731
        buf = hp.load_trace_buffers(d, it, B)
        np.testing.assert_allclose(vn.state(), g("vn_before_update"), rtol=1e-6, atol=1e-7)
        chunks = (T * B) // L
        mbc = chunks // cfg.num_mini_batch
        got = []
        for e in range(cfg.ppo_epoch):
            perm = g("perms")[e]
            for i in range(cfg.num_mini_batch):
                gp, gc, sums, stats = hp.minibatch_buckets(shim, cfg, Pp, Pc, buf, perm[i * mbc:(i + 1) * mbc], dim, n, targets)
                agn, cgn = float(np.sqrt((gp * gp).sum())), float(np.sqrt((gc * gc).sum()))
                Pp = opt_p.step(Pp, gp * min(cfg.max_grad_norm / (agn + 1e-6), 1.0))
                Pc = opt_c.step(Pc, gc * min(cfg.max_grad_norm / (cgn + 1e-6), 1.0))
                got.append([sums[0], cgn, sums[1], sums[2], agn, sums[3] / stats[3]])
        np.testing.assert_allclose(np.array(got), g("updates"), rtol=3e-4, atol=3e-6)
        for P, order, mk in ((Pp, order_p, "policy"), (Pc, order_c, "critic")):
            off = 0
            for k in order:
                want = g(f"params/{mk}.{k}")
                np.testing.assert_allclose(P[off:off + want.size].reshape(want.shape), want, rtol=2e-3, atol=1e-5, err_msg=k)
                off += want.size
        np.testing.assert_allclose(vn.state(), g("vn_after_update"), rtol=1e-5, atol=1e-7)
