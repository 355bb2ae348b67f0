"""The absolute-term scales of tests/tc_ref64.py on a small CPU buffer: the captured per-row terms of every parameter
block sum, without absolute values, to the reference gradient; their absolute sums bound it; and every deliberate mistake
of TC_MUTANTS really changes the block it is meant to be caught in."""
import types

import pytest
import torch

import ffma_ref64
import tc_ref64 as ref

CFG = dict(use_huber_loss=True, use_clipped_value_loss=True, use_value_active_masks=True, use_policy_active_masks=True,
           use_valuenorm=True, use_adv_normalize=True, use_max_grad_norm=True, dual_clip_ppo=False, a2c=False, activation_id=1,
           clip_param=0.2, entropy_coef=0.01, value_loss_coef=0.5, huber_delta=1.0, max_grad_norm=10.0, dual_clip_coeff=3.0,
           lr=5e-4, critic_lr=5e-4, opti_eps=1e-5, weight_decay=0.0)
DIMS, R = (4, 5, 6), 600


def _case(seed=0, activation_id=1):
    d, n, dc = DIMS
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)   # noqa: E731
    am = (torch.rand(R, n, generator=g) < 0.7).double()
    act = torch.randint(0, n, (R,), generator=g)
    am[torch.arange(R), act] = 1.0
    buf = dict(policy_obs=r(R, d), critic_obs=r(R, dc), actions=act.double()[:, None], action_log_probs=-1.4 + 0.3 * r(R, 1),
               advantages=r(R, 1), value_preds=r(R, 1), returns=2 * r(R, 1), action_masks=am,
               active_masks=(torch.rand(R, 1, generator=g) > 0.1).double())
    state = {}
    for key, dd, head in (("pol", d, "categorical"), ("cri", dc, "critic")):
        parts = []
        for name, shp in ffma_ref64.param_shapes(dd, n, head):
            x = r(*shp)
            parts.append((x / shp[1] ** 0.5 if len(shp) == 2 else (1.0 + 0.2 * x if name.endswith("weight") else 0.1 * x)).reshape(-1))
        state[key] = torch.cat(parts)
        state[key + "_m"] = 1e-3 * r(state[key].numel())
        state[key + "_v"] = 1e-6 * torch.rand(state[key].numel(), generator=g, dtype=torch.float64)
    state["steps"], state["vn"] = [2, 2], torch.tensor([0.1, 0.5, 0.3], dtype=torch.float64)
    cfg = types.SimpleNamespace(**{**CFG, "activation_id": activation_id})
    return cfg, buf, state, torch.randperm(R, generator=g)[:R - 100]


@pytest.mark.parametrize("activation_id", [0, 1, 2, 3], ids=["tanh", "relu", "leaky_relu", "elu"])
def test_row_terms_sum_to_the_gradient(activation_id):
    cfg, buf, state, rows = _case(activation_id=activation_id)
    out = ref.update(cfg, buf, state, rows, DIMS)
    for net in ("pol", "cri"):
        terms = out["terms_" + net]
        blocks = ref.blocks(DIMS, net)
        assert set(terms) == set(blocks), net
        for name, s in blocks.items():
            signed, absum = terms[name]
            scale = absum.norm()
            want = out["grad_" + net][s]
            err = float((signed - want).norm())
            assert bool((absum >= want.abs() * (1 - 1e-12)).all()), (net, name)
            assert err <= 1e-12 * float(scale), (net, name, err, float(scale))
            assert float(scale) >= float(want.norm()) * (1 - 1e-12) and float(scale) > 0, (net, name)
    # with advantages of both signs the policy terms cancel: their absolute sum is well above the gradient
    sig, sc = out["terms_pol"]["base.mlp.fc1.0.weight"]
    assert float(sc.norm()) > 2 * float(sig.norm())
    for net in ("pol", "cri"):
        assert all(v > 0 for v in out["peaks"][net].values()), out["peaks"]


def test_capture_leaves_the_reference_unchanged():
    cfg, buf, state, rows = _case(seed=2)
    a = ref.update(cfg, buf, state, rows, DIMS)
    b = ffma_ref64.update(cfg, buf, state, rows, DIMS, "categorical")
    for k in ("grad_pol", "grad_cri", "pol", "cri", "pol_m", "cri_v", "losses", "vn"):
        assert torch.equal(a[k], b[k]), k


def test_operand_scales_follow_the_kernel_formula():
    w = torch.full((2, 64), 0.01)
    sz, su = ref.operand_scales(524288, w, torch.ones(64))
    assert su == 2.0 ** 22 and sz == 2.0 ** (22 + 7)   # floor(log2 0.01) = -7
    sz, su = ref.operand_scales(37, w, torch.ones(64))
    assert su == 2.0 ** 9 and sz == 2.0 ** 16


@pytest.mark.parametrize("mutant", list(ref.TC_MUTANTS))
def test_every_mutant_changes_its_block(mutant):
    cfg, buf, state, rows = _case(seed=1)
    clean = ref.update(cfg, buf, state, rows, DIMS)
    kw = {}
    if mutant == "cta-last-tile-dropped":
        kw = dict(remove_rows=rows[-37:])
    elif mutant == "stale-staged-tile":
        kw = dict(remove_rows=rows[128:256], add_rows=rows[:128])
    elif mutant == "partial-tail-counted":
        kw = dict(add_rows=torch.tensor([i for i in range(R) if i not in set(rows.tolist())][:40]))
    else:
        kw = dict(clamp_dz3={"pol": 0.25 * clean["peaks"]["pol"]["dz3"]})
    bad = ref.mutant_grad_pol(mutant, cfg, buf, state, rows, DIMS, clean, **kw)
    name = ref.TC_MUTANTS[mutant][1].split(".", 1)[1]
    s = ref.blocks(DIMS, "pol")[name]
    rel = float((bad[s] - clean["grad_pol"][s]).norm() / clean["terms_pol"][name][1].norm())
    print(f"\n  {mutant}: {name} moves by {rel:.3e} of its absolute-term scale")
    assert rel > 1e-3, (mutant, rel)
