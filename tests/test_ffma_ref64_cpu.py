"""The float64 reference of the feed-forward PPO update (tests/ffma_ref64.py) on a small CPU buffer: its float32 run
stays close to its float64 run, its default ValueNorm matches the reference's float32 one, and every deliberate mistake
of tests/test_ppo_ffma_scale_cuda.py really changes the quantity it is meant to be caught by (no mutant is a no-op)."""
import types

import pytest
import torch

import ffma_ref64 as ref

CFG = dict(use_huber_loss=True, use_clipped_value_loss=True, use_value_active_masks=True, use_policy_active_masks=True,
           use_valuenorm=True, use_adv_normalize=False, use_max_grad_norm=True, dual_clip_ppo=False, a2c=False, activation_id=1,
           clip_param=0.2, entropy_coef=0.01, value_loss_coef=0.5, huber_delta=1.0, max_grad_norm=10.0, dual_clip_coeff=3.0,
           lr=5e-4, critic_lr=5e-4, opti_eps=1e-5, weight_decay=0.0)
DIMS, R = (5, 6, 7), 300


def _case(seed=0):
    d, n, dc = DIMS
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)   # noqa: E731
    buf = dict(policy_obs=r(R, d), critic_obs=r(R, dc), actions=r(R, n), action_log_probs=-1.4 + 0.2 * r(R, n),
               advantages=r(R, 1), value_preds=r(R, 1), returns=2 * r(R, 1), active_masks=(torch.rand(R, 1, generator=g) > 0.1).double())
    state = {}
    for key, dd, head in (("pol", d, "gaussian"), ("cri", dc, "critic")):
        parts = []
        for name, shp in ref.param_shapes(dd, n, head):
            x = r(*shp)
            parts.append((x / shp[1] ** 0.5 if len(shp) == 2 and shp[1] > 1 else 0.1 * x).reshape(-1))
        state[key] = torch.cat(parts)
        state[key + "_m"] = 1e-3 * r(state[key].numel())
        state[key + "_v"] = 1e-6 * torch.rand(state[key].numel(), generator=g, dtype=torch.float64)
    state["steps"], state["vn"] = [2, 2], torch.zeros(3, dtype=torch.float64)
    return buf, state, torch.randperm(R, generator=g)[:R - 40]


def test_float32_run_tracks_float64():
    buf, state, rows = _case()
    cfg = types.SimpleNamespace(**CFG)
    r64 = ref.update(cfg, buf, state, rows, DIMS, "gaussian", torch.float64)
    r32 = ref.update(cfg, buf, state, rows, DIMS, "gaussian", torch.float32)
    for k in ("grad_pol", "grad_cri", "pol", "cri", "pol_v", "cri_v"):
        assert float((r32[k].double() - r64[k]).norm() / r64[k].norm()) < 1e-4, k
    assert (r64["pol_step"], r64["cri_step"]) == (3, 3)
    assert float(r64["ratio_mean"]) > 0 and r64["vn"].dtype == torch.float64


def test_value_norm_default_dtype_is_float32():
    from oracle.ppo import ValueNormState

    vn = ValueNormState([0.1, 0.2, 0.3])
    assert vn.running_mean.dtype == torch.float32 and vn.state().dtype.name == "float32"
    vn64 = ValueNormState([0.1, 0.2, 0.3], dtype=torch.float64)
    assert vn64.debiasing_term.dtype == torch.float64 and vn64.state()[2] == 0.3


def _target(out, what):
    """The quantity a check line of the GPU test names: 'grad pol.<param>' / 'grad cri.<param>'."""
    net, name = what.split(" ")[1].split(".", 1)
    head = "gaussian" if net == "pol" else "critic"
    d, n, dc = DIMS
    return out["grad_" + net][ref.blocks(d if net == "pol" else dc, n, head)[name]]


@pytest.mark.parametrize("mutant", list(ref.MUTANTS))
def test_every_mutant_changes_its_quantity(mutant):
    _, what, opts, _ = ref.MUTANTS[mutant]
    buf, state, rows = _case(seed=1)
    cfg = types.SimpleNamespace(**{**CFG, **opts})
    dropped = rows[:37] if mutant == "cta-last-tile-dropped" else None
    clean = ref.update(cfg, buf, state, rows, DIMS, "gaussian")
    bad = ref.update(cfg, buf, state, rows, DIMS, "gaussian", mutant=mutant, dropped_rows=dropped)
    a, b = _target(clean, what), _target(bad, what)
    rel = float((a - b).norm() / a.norm())
    print(f"\n  {mutant}: {what} moves by {rel:.3e} (relative L2)")
    assert rel > 1e-2, (mutant, rel)
