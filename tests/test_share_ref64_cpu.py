"""The high-precision shared-model update reference (tests/share_ref64.py) against the reference's traces, and its
deliberate mistakes against the correct reference, on the CPU.

- Iteration 0 of trace_share_model (CartPole, Categorical head) and trace_share_gaussian (IdentityEnvcontinuous,
  DiagGaussian head, 2 epochs x 2 minibatches each) is replayed update by update with the recorded permutations, in
  float32.  Every update's six logged scalars must match at 2e-4 relative, and so must the parameters and the ValueNorm
  state after the iteration: the reference tests/test_share_scale_cuda.py holds the kernels to is itself held to the
  executed reference here.
- Every mutant of share_ref64.MUTANTS moves the quantity it is meant to be caught by far beyond a float32 rounding of
  that quantity (no mutant is a no-op)."""
import os
import types

import numpy as np
import pytest
import torch

import share_ref64 as ref
from conftest import GOLDEN
from oracle import loop


@pytest.mark.parametrize("tag,head", [("share_model", "categorical"), ("share_gaussian", "gaussian")])
def test_share_ref64_reproduces_reference_trace(tag, head):
    d = np.load(os.path.join(GOLDEN, f"trace_{tag}.npz"), allow_pickle=True)
    cfg = loop.cfg_from_flags(str(d["meta/flags"]))
    assert cfg.use_share_model
    T, N = d["it0/actions"].shape[:2]
    rows = lambda key, slots=T: torch.from_numpy(d[f"it0/{key}"][:slots].reshape(slots * N, -1).copy())   # noqa: E731
    obs_dim = d["it0/policy_obs"].shape[-1]
    n = d["it0/actions"].shape[-1] if head == "gaussian" else d["it0/action_masks"].shape[-1]
    dims = (obs_dim, n)
    vn0 = torch.from_numpy(d["it0/vn_before_update"]).double()
    vp = rows("value_preds").double()
    if cfg.use_valuenorm:   # the buffer's advantages: returns - denormalised value predictions (orl_gae)
        m = vn0[0] / vn0[2].clamp(min=1e-5)
        vp = vp * (vn0[1] / vn0[2].clamp(min=1e-5) - m * m).clamp(min=1e-2).sqrt() + m
    buf = dict(obs=rows("policy_obs"), actions=rows("actions"), action_log_probs=rows("action_log_probs"),
               value_preds=rows("value_preds"), returns=rows("returns"), active_masks=rows("active_masks"),
               advantages=(rows("returns").double() - vp).float())
    if head == "categorical":
        buf["action_masks"] = rows("action_masks")
    names = [name for name, _ in ref.param_shapes(*dims, head)]
    assert {k[len("init/model."):] for k in d.files if k.startswith("init/model.") and "value_normalizer" not in k
            and "critic_obs_prep" not in k} == set(names)
    p0 = torch.from_numpy(np.concatenate([d[f"init/model.{k}"].reshape(-1) for k in names]))
    state = dict(p=p0, m=torch.zeros_like(p0), v=torch.zeros_like(p0), step=0, vn=vn0.float())
    perms, want = d["it0/perms"], d["it0/updates"]
    mb = perms.shape[1] // cfg.num_mini_batch
    rcfg = types.SimpleNamespace(**vars(cfg))
    k = 0
    for perm in perms:
        for i in range(cfg.num_mini_batch):
            idx = torch.from_numpy(perm[i * mb:(i + 1) * mb].copy())
            out = ref.update(rcfg, buf, state, idx, dims, head, torch.float32)
            ls = out["losses"]
            got = [ls[3], out["norms"][1], ls[0], ls[1], out["norms"][0], out["ratio_mean"]]
            np.testing.assert_allclose([float(x) for x in got], want[k], rtol=2e-4, atol=2e-6, err_msg=f"{tag} update {k}")
            state = dict(p=out["p"], m=out["m"], v=out["v"], step=out["step"], vn=out["vn"])
            k += 1
    assert k == len(want) == 4 and state["step"] == 4
    for name, s in ref.blocks(*dims, head).items():
        np.testing.assert_allclose(state["p"][s].numpy(), d[f"it0/params/model.{name}"].reshape(-1), rtol=2e-4, atol=2e-6,
                                   err_msg=f"{tag} {name}")
    np.testing.assert_allclose(state["vn"].numpy(), d["it0/vn_after_update"], rtol=2e-4, atol=1e-9)


CFG = dict(use_huber_loss=True, use_clipped_value_loss=True, use_value_active_masks=True, use_policy_active_masks=True,
           use_valuenorm=True, use_adv_normalize=False, use_max_grad_norm=True, dual_clip_ppo=False, a2c=False, activation_id=1,
           clip_param=0.2, entropy_coef=0.01, value_loss_coef=0.5, huber_delta=1.0, max_grad_norm=10.0, dual_clip_coeff=3.0,
           lr=5e-4, critic_lr=5e-4, opti_eps=1e-5, weight_decay=0.0)
D, N_ACT, R = 5, 4, 2 * 1024 + 300


def _case(head, seed):
    """A buffer of R rows (three tape row blocks over the minibatch) and a mid-run state.  The old log-probs sit near
    the current ones, so ratios are near 1 and the clip leaves most rows' gradients in place."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)   # noqa: E731
    n = N_ACT
    parts = []
    for name, shp in ref.param_shapes(D, n, head):
        x = r(*shp)
        parts.append((x / shp[1] ** 0.5 if len(shp) == 2 and shp[1] > 1 else 0.1 * x).reshape(-1))
    p = torch.cat(parts)
    state = dict(p=p, m=1e-3 * r(p.numel()), v=1e-6 * torch.rand(p.numel(), generator=g, dtype=torch.float64), step=2,
                 vn=torch.zeros(3, dtype=torch.float64))   # a fresh ValueNorm, as at a run's first update
    obs = r(R, D)
    buf = dict(obs=obs, advantages=r(R, 1), value_preds=r(R, 1), returns=2 * r(R, 1) + 1,
               active_masks=(torch.rand(R, 1, generator=g) > 0.1).double())
    cfg = types.SimpleNamespace(**CFG)
    pd = ref.unflatten(p, D, n, head)
    ncfg = ref.ffma_ref64.oracle_cfg(cfg)
    with torch.no_grad():
        if head == "gaussian":
            mean, std = ref.nets.gaussian_params(pd, ref.nets.policy_features(pd, ncfg, obs)[0])
            buf["actions"] = mean + std * r(R, n)
            logp, _ = ref.nets.policy_eval_gaussian(pd, ncfg, obs, buf["actions"])
        else:
            am = (torch.rand(R, n, generator=g) > 0.3).double()
            act = torch.randint(0, n, (R,), generator=g)
            am[torch.arange(R), act] = 1.0
            buf["actions"], buf["action_masks"] = act.double()[:, None], am
            logp, _ = ref.nets.policy_eval(pd, ncfg, obs, buf["actions"], am)
    buf["action_log_probs"] = logp + 0.05 * r(*logp.shape)
    return buf, state, torch.randperm(R, generator=g)[:R - 40]


@pytest.mark.parametrize("mutant", list(ref.MUTANTS))
def test_every_mutant_changes_its_quantity(mutant):
    desc, what, opts, on = ref.MUTANTS[mutant]
    head = "gaussian" if on == "gaussian" else "categorical"
    buf, state, rows = _case(head, seed=len(mutant))
    if on == "categorical":
        del buf["action_masks"]
    cfg = types.SimpleNamespace(**{**CFG, **opts})
    dims = (D, N_ACT)
    clean64 = ref.update(cfg, buf, state, rows, dims, head)
    clean32 = ref.update(cfg, buf, state, rows, dims, head, torch.float32)
    bad = ref.update(cfg, buf, state, rows, dims, head, mutant=mutant)
    a, a32, b = (ref.target(x, what, dims, head) for x in (clean64, clean32, bad))
    rel = float((a - b).norm() / a.norm())
    e32 = float((a32.double() - a).norm() / a.norm())
    print(f"\n  {mutant}: {what} moves by {rel:.3e} (relative L2); float32 is {e32:.1e} off")
    assert rel > max(1e3 * e32, 1e-4), (mutant, rel, e32)
    if mutant == "critic-norm-unclipped":   # the case where the two logged norms differ: the first clip acts
        assert float(clean64["norms"][0]) > cfg.max_grad_norm


@pytest.mark.parametrize("activation_id", [1, 2])
def test_teacher_forced_branches_act_on_ties_only(activation_id):
    """The kernel's ReLU / LeakyReLU branches replace the reference's only where |z| < BRANCH_TIE: given the reference's
    own branches, or the opposite ones everywhere, the update on a buffer without ties is the plain one, bit for bit; a
    tie planted on one unit takes the given branch."""
    buf, state, rows = _case("categorical", seed=3)
    cfg = types.SimpleNamespace(**{**CFG, "activation_id": activation_id})
    dims = (D, N_ACT)
    p = ref.unflatten(state["p"], *dims, "categorical")
    x = buf["obs"][rows]
    z1 = x @ p["obs_prep.mlp.fc1.0.weight"].t() + p["obs_prep.mlp.fc1.0.bias"]
    y3 = ref.nets.mlp_base(p, "obs_prep", x, 1, activation_id)
    z5 = y3 @ p["common.fc1.0.weight"].t() + p["common.fc1.0.bias"]
    keep = (z1.abs().min(-1).values > ref.BRANCH_TIE) & (z5.abs().min(-1).values > ref.BRANCH_TIE)   # rows without ties
    rows, z1, z5 = rows[keep], z1[keep], z5[keep]
    assert rows.numel() > 2000
    plain = ref.update(cfg, buf, state, rows, dims, "categorical")
    for own in (True, False):
        br = {"obs_prep": (z1 > 0) == own, "common": (z5 > 0) == own}
        forced = ref.update(cfg, buf, state, rows, dims, "categorical", branches=br)
        assert torch.equal(forced["grad"], plain["grad"]) and torch.equal(forced["p"], plain["p"])
    # a tie: unit 0's bias moved so that the first minibatch row's common pre-activation is +1e-7
    state2 = dict(state)
    b5 = ref.blocks(*dims, "categorical")["common.fc1.0.bias"]
    state2["p"] = state["p"].clone()
    state2["p"][b5.start] -= float(z5[0, 0]) - 1e-7
    br = {"obs_prep": z1 > 0, "common": torch.zeros_like(z5, dtype=torch.bool)}
    on = ref.update(cfg, buf, state2, rows, dims, "categorical")
    off = ref.update(cfg, buf, state2, rows, dims, "categorical", branches=br)
    assert not torch.equal(on["grad"], off["grad"])
