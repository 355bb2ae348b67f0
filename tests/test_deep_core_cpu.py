"""The sequential shared policy-value network core used by the cfg.use_share_model CUDA kernels
(openrl_b200/csrc/orl_deep_core.h) compiled with g++ and checked on the CPU against torch autograd of the oracle
(oracle/nets.py: PolicyValueNetwork restatement, pinned to the reference trace tests/golden/trace_share_model.npz):
forward heads, and every parameter gradient obtained from the per-row tape as dW = sum_rows P^T Q / column sums."""
import numpy as np
import pytest
import torch

from helpers import grads_from_tape, gxx_shim, ptr
from oracle import loop, nets


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return gxx_shim(tmp_path_factory, "deep", "deep_core_shim.cpp")


# tape field offsets (orl_deep_core.h)
@pytest.mark.parametrize("d,n,act", [(4, 2, 1), (7, 5, 0), (18, 3, 3), (4, 8, 2)])
def test_deep_core_forward_backward_matches_torch(shim, d, n, act):
    torch.manual_seed(0)
    cfg = loop.make_cfg(use_share_model=True, activation_id=act)
    params = nets.init_policy_value(cfg, d, "Discrete", n)
    g = torch.Generator().manual_seed(1)
    for v in params.values():   # non-trivial LayerNorm affine / biases
        v.add_(0.1 * torch.randn(v.shape, generator=g))
        v.requires_grad_(True)
    assert shim.shim_deep_param_count(d, n) == sum(v.numel() for v in params.values())
    rows = 37
    X = torch.randn(rows, d, generator=g)
    dv = torch.randn(rows, 1, generator=g)
    dlog = torch.randn(rows, n, generator=g)
    feat = nets.shared_trunk(params, cfg, X)
    values = torch.nn.functional.linear(feat, params["v_out.weight"], params["v_out.bias"])
    logits = torch.nn.functional.linear(feat, params["act.action_out.linear.weight"], params["act.action_out.linear.bias"])
    ((values * dv).sum() + (logits * dlog).sum()).backward()
    P = np.concatenate([v.detach().numpy().reshape(-1) for v in params.values()]).astype(np.float32)
    T = shim.shim_deep_tape_width()
    tape = np.zeros((rows, T), np.float32)
    v_out, l_out = np.zeros(rows, np.float32), np.zeros((rows, n), np.float32)
    Xn, dvn, dln = X.numpy().copy(), dv.numpy().reshape(-1).copy(), dlog.numpy().copy()
    shim.shim_deep_rows(ptr(P), d, n, act, rows, ptr(Xn), ptr(v_out), ptr(l_out), ptr(dvn), ptr(dln), ptr(tape))
    np.testing.assert_allclose(v_out, values.detach().numpy().reshape(-1), rtol=1e-5, atol=5e-6)
    np.testing.assert_allclose(l_out, logits.detach().numpy(), rtol=1e-5, atol=5e-6)
    got = grads_from_tape(tape.astype(np.float64), d, n)
    for k, p in params.items():
        want = p.grad.numpy()
        np.testing.assert_allclose(got[k].reshape(want.shape), want, rtol=2e-4, atol=2e-5 * max(1.0, float(np.abs(want).max())), err_msg=k)
