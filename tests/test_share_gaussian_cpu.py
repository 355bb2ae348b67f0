"""The shared policy-value network with a DiagGaussian head (cfg.use_share_model on Box action spaces), on the CPU.

- The oracle (oracle/loop.py, oracle/nets.py) reproduces the reference's trace tests/golden/trace_share_gaussian.npz
  (IdentityEnvcontinuous, 4 envs, T = 16, 2 epochs, 2 minibatches, 2 iterations; recorded by
  tools/gen_golden_share_gaussian.py): initial parameters, actions and observations bit for bit, the six update scalars
  within 1e-4.
- The sequential core of the CUDA kernels (openrl_b200/csrc/orl_deep_core.h), compiled with g++, against torch autograd
  of the oracle: the Gaussian parameter layout (logstd after the mean head's bias), the mean, and every parameter
  gradient from the Gaussian tape as dW = sum_rows P^T Q / column sums, logstd from the rows' dL/dlogstd field."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from helpers import TRACE_THREADS, grads_from_tape, gxx_shim, ptr
from oracle import loop, nets


def test_oracle_reproduces_reference_share_gaussian_trace():
    before = torch.get_num_threads()
    torch.set_num_threads(TRACE_THREADS)
    try:
        d = np.load(os.path.join(GOLDEN, "trace_share_gaussian.npz"), allow_pickle=True)
        cfg = loop.cfg_from_flags(str(d["meta/flags"]))
        assert cfg.use_share_model
        tr = loop.Trainer(cfg, "IdentityEnvcontinuous", int(d["meta/env_num"]))
        assert list(tr.pol)[-3:] == ["act.action_out.fc_mean.weight", "act.action_out.fc_mean.bias", "act.action_out.logstd._bias"]
        for k, v in tr.pol.items():
            assert np.array_equal(v.detach().numpy(), d[f"init/model.{k}"]), k
        for it in range(int(d["meta/iters"])):
            tr.rollout()
            b = tr.buf
            assert b.actions.shape == d[f"it{it}/actions"].shape == (16, 4, 1, 1)
            assert np.array_equal(b.actions, d[f"it{it}/actions"])
            assert np.array_equal(b.obs, d[f"it{it}/policy_obs"])
            np.testing.assert_allclose(b.action_log_probs, d[f"it{it}/action_log_probs"], rtol=0, atol=1e-6)
            tr.compute_returns()
            np.testing.assert_allclose(b.value_preds, d[f"it{it}/value_preds"], rtol=0, atol=1e-5)
            updates, perms = tr.train()
            assert np.array_equal(perms, d[f"it{it}/perms"])
            np.testing.assert_allclose(updates, d[f"it{it}/updates"], rtol=1e-4, atol=1e-6)
            np.testing.assert_allclose(updates[:, 1], 10.0, rtol=1e-6)   # critic_grad_norm: the second clip's norm
            tr.after_update()
            for k, v in tr.pol.items():
                np.testing.assert_allclose(v.detach().numpy(), d[f"it{it}/params/model.{k}"], rtol=1e-4, atol=1e-6, err_msg=k)
    finally:
        torch.set_num_threads(before)


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return gxx_shim(tmp_path_factory, "deepg", "deep_core_gaussian_shim.cpp")


@pytest.mark.parametrize("n", [1, 6, 8])
@pytest.mark.parametrize("d", [1, 17, 64])
def test_gaussian_core_matches_torch_autograd(shim, d, n):
    act = 1
    torch.manual_seed(0)
    cfg = loop.make_cfg(use_share_model=True, activation_id=act)
    params = nets.init_policy_value(cfg, d, "Box", n)
    g = torch.Generator().manual_seed(d * 10 + n)
    for v in params.values():   # non-trivial LayerNorm affine / biases / log-stds
        v.add_(0.1 * torch.randn(v.shape, generator=g))
        v.requires_grad_(True)
    names = list(params)
    assert names[-3:] == ["act.action_out.fc_mean.weight", "act.action_out.fc_mean.bias", "act.action_out.logstd._bias"]
    total = sum(v.numel() for v in params.values())
    assert shim.shim_gauss_param_count(d, n) == total and shim.shim_gauss_logstd_offset(d, n) == total - n
    rows = 37
    X = torch.randn(rows, d, generator=g)
    dv = torch.randn(rows, 1, generator=g)
    acts = torch.randn(rows, n, generator=g)
    w = torch.randn(rows, n, generator=g)
    feat = nets.shared_trunk(params, cfg, X)
    values = torch.nn.functional.linear(feat, params["v_out.weight"], params["v_out.bias"])
    mean = torch.nn.functional.linear(feat, params["act.action_out.fc_mean.weight"], params["act.action_out.fc_mean.bias"])
    mean.retain_grad()
    logstd = params["act.action_out.logstd._bias"].t().expand(rows, n)   # one copy per row: its gradient is the row's
    logstd.retain_grad()
    # a weighted per-dimension Gaussian log-likelihood and entropy, so both mean and logstd carry gradient
    dist = torch.distributions.Normal(mean, logstd.exp())
    loss = (values * dv).sum() + (dist.log_prob(acts) * w).sum() - 0.3 * dist.entropy().sum()
    loss.backward()
    P = np.concatenate([v.detach().numpy().reshape(-1) for v in params.values()]).astype(np.float32)
    W = shim.shim_gauss_tape_width()
    tape = np.zeros((rows, W), np.float32)
    v_out, m_out = np.zeros(rows, np.float32), np.zeros((rows, n), np.float32)
    Xn, dvn = X.numpy().copy(), dv.numpy().reshape(-1).copy()
    dmn, dlsn = mean.grad.numpy().astype(np.float32).copy(), logstd.grad.numpy().astype(np.float32).copy()
    shim.shim_gauss_rows(ptr(P), d, n, act, rows, ptr(Xn), ptr(v_out), ptr(m_out), ptr(dvn), ptr(dmn), ptr(dlsn), ptr(tape))
    np.testing.assert_allclose(v_out, values.detach().numpy().reshape(-1), rtol=1e-5, atol=5e-6)
    np.testing.assert_allclose(m_out, mean.detach().numpy(), rtol=1e-5, atol=5e-6)
    t64 = tape.astype(np.float64)
    got = grads_from_tape(t64, d, n)
    got["act.action_out.fc_mean.weight"] = got.pop("act.action_out.linear.weight")
    got["act.action_out.fc_mean.bias"] = got.pop("act.action_out.linear.bias")
    dls = shim.shim_gauss_dls_field()
    assert (t64[:, dls + n:dls + 8] == 0).all()
    got["act.action_out.logstd._bias"] = t64[:, dls:dls + n].sum(0)
    assert set(got) == set(params)
    for k, p in params.items():
        want = p.grad.numpy()
        np.testing.assert_allclose(got[k].reshape(want.shape), want, rtol=2e-4, atol=2e-5 * max(1.0, float(np.abs(want).max())), err_msg=k)
