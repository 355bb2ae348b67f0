"""The sequential recurrent-network core shared by the CUDA GRU kernels (openrl_b200/csrc/orl_rnn_core.h)
compiled with g++ and checked on the CPU against the torch oracle (oracle/nets.py: MLPBase -> RNNLayer ->
head; reference mlp.py / rnn.py): forward step, chunked BPTT (L steps with masked hidden-state carry) and
every parameter gradient obtained from the per-row tape as dW = sum_rows P^T Q."""
import numpy as np
import pytest
import torch

from helpers import gxx_shim, ptr
from oracle import loop, nets


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return gxx_shim(tmp_path_factory, "rnn", "rnn_core_shim.cpp")


def _flat(params):
    return np.concatenate([v.detach().numpy().reshape(-1) for v in params.values()]).astype(np.float32)


@pytest.mark.parametrize("kind,d,n,act", [("policy", 18, 5, 1), ("critic", 54, 1, 1), ("policy", 7, 3, 0), ("policy", 4, 2, 3)])
def test_chunk_forward_backward_matches_torch(shim, kind, d, n, act):
    torch.manual_seed(0)
    cfg = loop.make_cfg(use_recurrent_policy=True, activation_id=act)
    params = nets.init_policy(cfg, d, "Discrete", n) if kind == "policy" else nets.init_critic(cfg, d)
    g = torch.Generator().manual_seed(1)
    for v in params.values():   # make LayerNorm affine / biases non-trivial
        v.add_(0.1 * torch.randn(v.shape, generator=g))
        v.requires_grad_(True)
    order = list(params.keys())
    assert shim.shim_param_count(d, n) == sum(v.numel() for v in params.values())
    L, C = 3, 5
    X = torch.randn(L * C, d, generator=g)
    H0 = torch.randn(C, 1, 64, generator=g) * 0.5
    masks = (torch.rand(L * C, 1, generator=g) > 0.3).float()
    dlog = torch.randn(L * C, n, generator=g)
    # torch reference
    feat = nets.mlp_base(params, "base", X, cfg.layer_N, cfg.activation_id)
    feat, _ = nets.rnn_layer(params, "rnn", feat, H0, masks)
    if kind == "policy":
        out = torch.nn.functional.linear(feat, params["act.action_out.linear.weight"], params["act.action_out.linear.bias"])
    else:
        out = torch.nn.functional.linear(feat, params["v_out.weight"], params["v_out.bias"])
    (out * dlog).sum().backward()
    # C core
    P = _flat(params)
    T = shim.shim_tape_width()
    tape = np.zeros((L * C, T), np.float32)
    Out = np.zeros((L * C, n), np.float32)
    Xn, H0n, mn, dn = (np.ascontiguousarray(a.numpy(), dtype=np.float32) for a in (X, H0.reshape(C, 64), masks.reshape(-1), dlog))
    shim.shim_chunk_fwdbwd(ptr(P), d, n, act, L, C, ptr(Xn), ptr(H0n), ptr(mn), ptr(dn), ptr(Out), ptr(tape))
    np.testing.assert_allclose(Out, out.detach().numpy(), rtol=1e-4, atol=2e-5)
    t = tape.astype(np.float64)
    dz1, dz3, dgi, dgh, dlg = t[:, 0:64], t[:, 64:128], t[:, 128:320], t[:, 320:512], t[:, 512:512 + n]
    x, y1, y3, hm, o = t[:, 520:520 + d], t[:, 584:648], t[:, 648:712], t[:, 712:776], t[:, 776:840]
    got = {
        "base.mlp.fc1.0.weight": dz1.T @ x, "base.mlp.fc1.0.bias": dz1.sum(0),
        "base.mlp.fc1.2.weight": t[:, 840:904].sum(0), "base.mlp.fc1.2.bias": t[:, 904:968].sum(0),
        "base.mlp.fc3.0.weight": dz3.T @ y1, "base.mlp.fc3.0.bias": dz3.sum(0),
        "base.mlp.fc3.1.weight": t[:, 968:1032].sum(0), "base.mlp.fc3.1.bias": t[:, 1032:1096].sum(0),
        "rnn.rnn.weight_ih_l0": dgi.T @ y3, "rnn.rnn.weight_hh_l0": dgh.T @ hm,
        "rnn.rnn.bias_ih_l0": dgi.sum(0), "rnn.rnn.bias_hh_l0": dgh.sum(0),
        "rnn.norm.weight": t[:, 1096:1160].sum(0), "rnn.norm.bias": t[:, 1160:1224].sum(0),
    }
    head = "act.action_out.linear" if kind == "policy" else "v_out"
    got[head + ".weight"] = dlg.T @ o
    got[head + ".bias"] = dlg.sum(0)
    assert list(got.keys()) == order   # the flat layout IS the reference's state_dict order
    for k in order:
        want = params[k].grad.numpy()
        np.testing.assert_allclose(got[k].reshape(want.shape), want, rtol=2e-3, atol=2e-5 * max(1.0, np.abs(want).max()), err_msg=k)


def test_single_step_matches_torch(shim):
    torch.manual_seed(3)
    cfg = loop.make_cfg(use_recurrent_policy=True)
    params = nets.init_policy(cfg, 18, "Discrete", 5)
    rows = 9
    X, Hin = torch.randn(rows, 18), torch.randn(rows, 1, 64)
    masks = torch.tensor([[1.0], [0.0], [1.0]] * 3)
    with torch.no_grad():
        feat = nets.mlp_base(params, "base", X, 1, 1)
        feat, hout = nets.rnn_layer(params, "rnn", feat, Hin, masks)
        out = torch.nn.functional.linear(feat, params["act.action_out.linear.weight"], params["act.action_out.linear.bias"])
    P = _flat(params)
    Hout, Out = np.zeros((rows, 64), np.float32), np.zeros((rows, 5), np.float32)
    Xn, Hn, mn = (np.ascontiguousarray(a.numpy(), dtype=np.float32) for a in (X, Hin.reshape(rows, 64), masks.reshape(-1)))
    shim.shim_forward_rows(ptr(P), 18, 5, 1, rows, ptr(Xn), ptr(Hn), ptr(mn), ptr(Hout), ptr(Out))
    np.testing.assert_allclose(Out, out.numpy(), rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(Hout, hout.numpy().reshape(rows, 64), rtol=1e-4, atol=1e-6)
