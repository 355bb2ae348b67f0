"""The high-precision recurrent update reference (tests/rnn_ref64.py) against the unmodified reference's traces.

Iteration 0 of the simple_spread GRU trace (chunks of 2, one minibatch), the JRPO trace with two minibatches of
4-step v3 chunks and the CartPole GRU trace (episodes ending inside chunks of 4, two minibatches) is replayed update
by update with the recorded permutations, in float64.  Every update's six logged scalars must match at the bar of
tests/test_gru_cuda.py (2e-4 relative), and so must the parameters and the ValueNorm state after the iteration: the
reference the scale tests (tests/test_rnn_scale_cuda.py) hold the kernels to is itself held to the executed
reference here."""
import os

import numpy as np
import pytest
import torch

import rnn_ref64
from conftest import GOLDEN
from oracle import loop


def _trace_state(d):
    flat = {}
    for mk, key in (("policy", "pol"), ("critic", "cri")):
        names = [k[len(f"init/{mk}."):] for k in d.files if k.startswith(f"init/{mk}.") and "value_normalizer" not in k]
        flat[key] = torch.from_numpy(np.concatenate([d[f"init/{mk}.{k}"].reshape(-1) for k in names])).double()
    return flat, names


@pytest.mark.parametrize("tag", ["mpe_gru", "mpe_jrpo_mb", "cartpole_gru"])
def test_rnn_ref64_reproduces_reference_trace(tag):
    d = np.load(os.path.join(GOLDEN, f"trace_{tag}.npz"), allow_pickle=True)
    flags = str(d["meta/flags"])
    cfg = loop.cfg_from_flags(flags)
    cfg.vn_beta = 0.99999
    joint = "--use_joint_action_loss true" in flags
    T, N, A = d["it0/actions"].shape[:3]
    L = cfg.data_chunk_length
    buf = {k: torch.from_numpy(d[f"it0/{k}"]).double() for k in
           ("policy_obs", "critic_obs", "rnn_states", "rnn_states_critic", "masks", "active_masks", "actions",
            "action_log_probs", "value_preds", "returns")}
    vn0 = torch.from_numpy(d["it0/vn_before_update"]).double()
    vp = buf["value_preds"][:T]
    if cfg.use_valuenorm:   # the buffer's advantages: returns - denormalised value predictions (orl_gae)
        m = vn0[0] / vn0[2].clamp(min=1e-5)
        var = (vn0[1] / vn0[2].clamp(min=1e-5) - m * m).clamp(min=1e-2)
        vp = vp * var.sqrt() + m
    buf["advantages"] = buf["returns"][:T] - vp

    flat, _ = _trace_state(d)
    state = dict(pol=flat["pol"], cri=flat["cri"], pol_m=torch.zeros_like(flat["pol"]), pol_v=torch.zeros_like(flat["pol"]),
                 cri_m=torch.zeros_like(flat["cri"]), cri_v=torch.zeros_like(flat["cri"]), steps=(0, 0), vn=vn0)
    dims = (d["it0/policy_obs"].shape[-1], d["it0/action_masks"].shape[-1], d["it0/critic_obs"].shape[-1])
    perms = d["it0/perms"]
    mbc = perms.shape[1] // cfg.num_mini_batch
    groups = mbc * L
    want = d["it0/updates"]
    k = 0
    for perm in perms:
        for i in range(cfg.num_mini_batch):
            ids = torch.from_numpy(perm[i * mbc:(i + 1) * mbc].copy())
            out = rnn_ref64.update(cfg, buf, state, ids, L, dims, joint=joint)
            ls = out["losses"]
            got = [ls[3], out["norms"][1], ls[0], ls[1], out["norms"][0], ls[2] / groups]
            np.testing.assert_allclose([float(x) for x in got], want[k], rtol=2e-4, atol=2e-6, err_msg=f"{tag} update {k}")
            state = dict(pol=out["pol"], cri=out["cri"], pol_m=out["pol_m"], pol_v=out["pol_v"], cri_m=out["cri_m"],
                         cri_v=out["cri_v"], steps=(out["pol_step"], out["cri_step"]), vn=out["vn"])
            k += 1
    assert k == len(want)
    for mk, key, dd, nn, critic in (("policy", "pol", dims[0], dims[1], False), ("critic", "cri", dims[2], 1, True)):
        for name, s in rnn_ref64.blocks(dd, nn, critic).items():
            np.testing.assert_allclose(state[key][s].numpy(), d[f"it0/params/{mk}.{name}"].reshape(-1), rtol=2e-4, atol=2e-6,
                                       err_msg=f"{tag} {mk}.{name}")
    if cfg.use_valuenorm:
        np.testing.assert_allclose(state["vn"].numpy(), d["it0/vn_after_update"], rtol=2e-4, atol=1e-9)
