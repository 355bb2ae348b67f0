"""High-precision reference of one feed-forward PPO minibatch update (`orl_ppo_fwdbwd` + `orl_ppo_reduce` +
`orl_ppo_apply`, the FFMA kernel of orl_ppo.cu), and deliberate mistakes ("mutants") of it.

TEST INFRASTRUCTURE.  A thin layer over the oracle (oracle/nets.py, oracle/ppo.py `ppo_update`), which is
dtype-agnostic: the same code runs in float64 (the reference) and in float32 (the yardstick for how far a correct float32
implementation may drift from it).  Inputs are the update kernel's row layout: every buffer array viewed as (rows, width),
row r of every array belonging together; a minibatch is a LongTensor of rows.  The loss coefficients and Adam constants
are rounded to float32 first, as the kernel receives them (OrlPpoArgs).

`update` returns the true (pre-clip) gradients of both nets flattened in the kernel's parameter order (net_offsets: W1,
b1, LN1 gain / bias, W3, b3, LN3 gain / bias, head W, head b[, logstd]), the loss sums in the order of the kernel's loss
slots (policy loss, entropy, ratio sum, value loss) with the weighted sum of the absolute terms of each, both gradient
norms, the reported ratio mean, and the parameters, Adam moments, step counts and ValueNorm state after the clip and the
Adam step.
"""
import contextlib
import types
from unittest import mock

import numpy as np
import torch

import param_layout as layout
import rnn_ref64
from oracle import nets, ppo as oppo

H = layout.H


def param_shapes(d, n, head):
    """(state_dict name, shape) in the order of the flat parameter buffer; head: "gaussian", "categorical" or "critic"."""
    return layout.mlp_trunk(d) + layout.head(n, head)


def blocks(d, n, head):
    """{name: slice of the flat buffer} in flat order."""
    return layout.blocks(param_shapes(d, n, head))


def unflatten(flat, d, n, head):
    return layout.unflatten(flat, param_shapes(d, n, head))


def f32(x):
    return float(np.float32(x))


def oracle_cfg(cfg):
    """The oracle's option names, coefficients as the float32 values the kernel receives."""
    return types.SimpleNamespace(
        layer_N=1, activation_id=cfg.activation_id, use_recurrent_policy=False, use_naive_recurrent_policy=False,
        use_policy_active_masks=cfg.use_policy_active_masks, use_value_active_masks=cfg.use_value_active_masks,
        use_huber_loss=cfg.use_huber_loss, huber_delta=f32(cfg.huber_delta), use_clipped_value_loss=cfg.use_clipped_value_loss,
        clip_param=f32(cfg.clip_param), entropy_coef=f32(cfg.entropy_coef), value_loss_coef=f32(cfg.value_loss_coef),
        use_max_grad_norm=cfg.use_max_grad_norm, max_grad_norm=f32(cfg.max_grad_norm), lr=f32(cfg.lr),
        critic_lr=f32(cfg.critic_lr), opti_eps=f32(cfg.opti_eps), weight_decay=f32(cfg.weight_decay),
        a2c=bool(getattr(cfg, "a2c", False)), dual_clip_ppo=bool(getattr(cfg, "dual_clip_ppo", False)),
        dual_clip_coeff=f32(getattr(cfg, "dual_clip_coeff", 3.0)))


def _seed_adam(opt, params, m, v, step):
    """Start torch's Adam from a kernel's state: moments, step count and the float32 betas of OrlPpoArgs."""
    opt.param_groups[0]["betas"] = (f32(0.9), f32(0.999))
    for p, mm, vv in zip(params, m.values(), v.values()):
        opt.state[p] = {"step": torch.tensor(float(step)), "exp_avg": mm.clone(), "exp_avg_sq": vv.clone()}


class _StaleTargetValueNorm(oppo.ValueNormState):
    """Mutant: normalises the value targets with the ValueNorm state from before this minibatch's update."""

    def update(self, x):
        self.before = (self.running_mean.clone(), self.running_mean_sq.clone(), self.debiasing_term.clone())
        super().update(x)

    def normalize(self, x):
        after = (self.running_mean, self.running_mean_sq, self.debiasing_term)
        self.running_mean, self.running_mean_sq, self.debiasing_term = self.before
        try:
            return super().normalize(x)
        finally:
            self.running_mean, self.running_mean_sq, self.debiasing_term = after


# name: (what it changes, the compared quantity that must catch it, options it needs, whether it needs ratios away from 1)
MUTANTS = {
    "entropy-weight-1/rows": ("entropy weight 1/rows instead of 1/(rows n) without policy active masks",
                              "grad pol.act.action_out.logstd._bias", dict(use_policy_active_masks=False), False),
    "one-ratio-per-row": ("one ratio per row (log-probs summed over the dimensions) instead of one per dimension",
                          "grad pol.act.action_out.fc_mean.weight", {}, True),
    "logstd-grad-without-entropy": ("dL/dlogstd without its entropy term", "grad pol.act.action_out.logstd._bias", {}, False),
    "head-rows-4-7-dropped": ("head-gradient rows 4..7 dropped (one head row-block for n > 4)",
                              "grad pol.act.action_out.fc_mean.weight", {}, False),
    "cta-last-tile-dropped": ("the rows of one CTA's last tile left out", "grad pol.base.mlp.fc1.0.weight", {}, False),
    "vn-target-before-update": ("ValueNorm target from the state before this minibatch's update", "grad cri.v_out.weight",
                                {}, False),
}


def _mutant_eval(kind):
    orig = nets.policy_eval_gaussian

    def f(p, cfg, obs, actions, active_masks=None):
        logp, ent = orig(p, cfg, obs, actions, active_masks)
        if kind == "entropy-weight-1/rows" and not cfg.use_policy_active_masks:
            ent = ent * logp.shape[-1]          # sum / rows instead of sum / (rows n)
        elif kind == "one-ratio-per-row":
            logp = logp.sum(-1, keepdim=True)
        elif kind == "logstd-grad-without-entropy":
            ent = ent.detach()                  # the entropy depends on logstd alone
        return logp, ent
    return f


def update(cfg, buf, state, rows, dims, head, dtype=torch.float64, vn_beta=0.99999, mutant=None, dropped_rows=None,
           functional=None):
    """One minibatch update in `dtype` on the buffer rows `rows`.

    cfg: the project's option names (clip_param, entropy_coef, ..., use_valuenorm, use_adv_normalize, a2c).
    buf: (rows, width) arrays policy_obs, critic_obs, actions, action_log_probs, advantages, value_preds, returns,
      active_masks[, action_masks]; the advantages are normalised over every row of buf["advantages"] (the GAE moments).
    state: flat parameters pol / cri, Adam moments pol_m, pol_v, cri_m, cri_v, step counts steps = (pol, cri), ValueNorm
      state vn (3,).  dims: (d, n, dc); head: "gaussian" or "categorical".
    mutant: a key of MUTANTS; "cta-last-tile-dropped" leaves out `dropped_rows` (a subset of `rows`) while keeping
      the minibatch's loss weights.
    functional: None, or functional(pol, cri) -> the stand-in for torch.nn.functional that oracle/nets.py runs the
      update under, given the two nets' parameter dicts (tests/tc_ref64.py records the layer calls with it)."""
    d, n, dc = dims
    dev = rows.device
    cast = lambda x: torch.as_tensor(x).to(device=dev, dtype=dtype)   # noqa: E731
    ocfg = oracle_cfg(cfg)
    pol = unflatten(cast(state["pol"]), d, n, head)
    cri = unflatten(cast(state["cri"]), dc, 1, "critic")
    opt_p, opt_c = oppo.make_optimizers(ocfg, pol, cri)
    _seed_adam(opt_p, pol.values(), unflatten(cast(state["pol_m"]), d, n, head), unflatten(cast(state["pol_v"]), d, n, head),
               state["steps"][0])
    _seed_adam(opt_c, cri.values(), unflatten(cast(state["cri_m"]), dc, 1, "critic"),
               unflatten(cast(state["cri_v"]), dc, 1, "critic"), state["steps"][1])
    vn = None
    if cfg.use_valuenorm:
        vn_cls = _StaleTargetValueNorm if mutant == "vn-target-before-update" else oppo.ValueNormState
        vn = vn_cls([float(x) for x in state["vn"]], beta=vn_beta, dtype=dtype, device=dev)

    R = buf["advantages"].shape[0]
    active_all = buf["active_masks"][:R].to(dtype)
    adv = rnn_ref64.normalized_advantages(buf["advantages"].to(dtype), active_all, cfg.use_adv_normalize)
    g = lambda key: buf[key].to(dtype)[rows]   # noqa: E731
    batch = dict(policy_obs=g("policy_obs"), critic_obs=g("critic_obs"), actions=g("actions"), old_logp=g("action_log_probs"),
                 value_preds=g("value_preds"), returns=g("returns"), active_masks=g("active_masks"), adv=adv[rows])
    if "action_masks" in buf:
        batch["action_masks"] = g("action_masks")
    rec = {}
    with contextlib.ExitStack() as patches:
        if mutant in ("entropy-weight-1/rows", "one-ratio-per-row", "logstd-grad-without-entropy"):
            patches.enter_context(mock.patch.object(nets, "policy_eval_gaussian", _mutant_eval(mutant)))
            if mutant == "one-ratio-per-row":
                batch["old_logp"] = batch["old_logp"].sum(-1, keepdim=True)
        if functional is not None:
            patches.enter_context(mock.patch.object(nets, "F", functional(pol, cri)))
        oppo.ppo_update(ocfg, pol, cri, opt_p, opt_c, vn, batch, record=rec)

    gp = torch.cat([x.reshape(-1) for x in rec["grads_policy"].values()])
    gc = torch.cat([x.reshape(-1) for x in rec["grads_critic"].values()])
    act = batch["active_masks"]
    wsum = (lambda x: (x * act).sum() / act.sum()) if ocfg.use_policy_active_masks else (lambda x: x.mean())   # noqa: E731
    ratio = rec["ratio"].to(device=dev, dtype=dtype)
    ratio_sum = ratio.mean(-1).sum() if not ocfg.a2c else torch.zeros((), dtype=dtype, device=dev)
    sums = torch.stack([rec["policy_loss"], rec["entropy"], ratio_sum, rec["value_loss"]])
    scales = torch.stack([wsum(rec["surr"].abs().sum(-1, keepdim=True)), rec["entropy"].abs(), ratio_sum, rec["value_loss"]])
    out = dict(grad_pol=gp, grad_cri=gc, losses=sums, loss_scales=scales, norms=(gp.norm(), gc.norm()),
               ratio_mean=ratio_sum / rows.numel(), ratio_spread=(ratio - 1).abs().max() if not ocfg.a2c else None, vn=None if vn is None else torch.as_tensor(vn.state()).to(dev))
    for key, opt, params in (("pol", opt_p, pol), ("cri", opt_c, cri)):
        st = [opt.state[p] for p in params.values()]
        out[key] = torch.cat([p.detach().reshape(-1) for p in params.values()])
        out[key + "_m"] = torch.cat([s["exp_avg"].reshape(-1) for s in st])
        out[key + "_v"] = torch.cat([s["exp_avg_sq"].reshape(-1) for s in st])
        out[key + "_step"] = int(st[0]["step"])

    if mutant == "head-rows-4-7-dropped":
        hw = blocks(d, n, head)["act.action_out.fc_mean.weight" if head == "gaussian" else "act.action_out.linear.weight"]
        out["grad_pol"] = out["grad_pol"].clone()
        out["grad_pol"][hw.start + 4 * H:hw.stop] = 0.0
    elif mutant == "cta-last-tile-dropped":
        # the policy loss is a weighted sum of per-row terms: remove the dropped rows' share at the minibatch's weights
        part = update(cfg, buf, state, dropped_rows, dims, head, dtype, vn_beta)
        a_rows = buf["active_masks"][:].to(dtype)
        share = (a_rows[dropped_rows].sum() / a_rows[rows].sum() if ocfg.use_policy_active_masks
                 else torch.tensor(dropped_rows.numel() / rows.numel(), dtype=dtype))
        out["grad_pol"] = out["grad_pol"] - share.to(dev) * part["grad_pol"]
    return out
