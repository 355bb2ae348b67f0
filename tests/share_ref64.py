"""High-precision reference of one shared policy-value minibatch update (cfg.use_share_model: `orl_share_fwdbwd` +
`orl_share_apply`, orl_share.cu), and deliberate mistakes ("mutants") of it.

TEST INFRASTRUCTURE.  A thin layer over the oracle (oracle/nets.py, oracle/ppo.py `ppo_update` with one parameter dict
for both roles: `make_optimizers(cfg, p, p)` builds the one Adam with lr = cfg.lr), as tests/ffma_ref64.py is for the
two-net update.  The same code runs in float64 (the reference) and in float32 (the yardstick for how far a correct
float32 implementation may drift from it); tests/test_share_ref64_cpu.py pins it to the reference's traces.  Inputs
are the update kernel's row layout: every buffer array viewed as (rows, width); a minibatch is a LongTensor of rows in
the kernel's tape order.  Loss coefficients and Adam constants are rounded to float32 first, as the kernel receives them.

`update` returns, in the flat order of `deep_offsets` (orl_deep_core.h: the named_parameters order of
PolicyValueNetwork, logstd last):
- the true (pre-clip) gradient;
- the loss sums in the order of the kernel's loss slots (policy loss, entropy, ratio sum, value loss) and the weighted
  sum of the absolute terms of each;
- `actor_grad_norm` (the norm the first clip_grad_norm_ measures) and `critic_grad_norm` (the second one's, over the
  already clipped gradient), and the reported ratio mean;
- the parameters, exp_avg, exp_avg_sq and step count after the clip-twice-then-Adam step, and the ValueNorm state.
"""
import contextlib
from unittest import mock

import torch
import torch.nn.functional as F

import ffma_ref64
import param_layout as layout
import rnn_ref64
from oracle import nets, ppo as oppo

H = layout.H
TAPE_ROW_BLOCK = 1024   # rows per partial sum of the tape reduction (orl_tape.cu)


def param_shapes(d, n, head):
    """(state_dict name, shape) in the order of the flat parameter buffer; head: "gaussian" or "categorical"."""
    return layout.mlp_trunk(d, "obs_prep.mlp.") + layout.mlp_trunk(H, "common.") + layout.head(1, "critic") + layout.head(n, head)


def blocks(d, n, head):
    """{state_dict name: slice of the flat buffer} in flat order."""
    return layout.blocks(param_shapes(d, n, head))


def unflatten(flat, d, n, head):
    return layout.unflatten(flat, param_shapes(d, n, head))


class _BatchReturnsValueNorm(oppo.ValueNormState):
    """ValueNorm updated with a fixed minibatch's returns whatever rows the loss sees (the dropped rows of a mutant)."""

    def __init__(self, *args, batch_returns, **kw):
        super().__init__(*args, **kw)
        self.batch_returns = batch_returns

    def update(self, x):
        super().update(self.batch_returns)


# Pre-activations closer to the ReLU / LeakyReLU kink than this are ties: a float32 dot product of 64 terms of order
# one is ~5e-7 off, so its rounding can take either branch.  On a real buffer a handful of the 33.5 million (row, unit)
# pairs of C2 fall there (|z| <= 6.3e-7 measured); each one moves the gradient by a whole row's term.
BRANCH_TIE = 1e-5


def _act_teacher_forced(z, activation_id, on):
    """nets.activation, except that where |z| < BRANCH_TIE the branch is the one in `on` (a kernel's own choice)."""
    if on is None or activation_id not in (1, 2):
        return nets.activation(z, activation_id)
    pos = torch.where(z.detach().abs() < BRANCH_TIE, on, z.detach() > 0)
    return torch.where(pos, z, z * (0.0 if activation_id == 1 else 0.01))


def _trunk_teacher_forced(branches):
    """nets.shared_trunk (layer_N = 1) with the two activations' tie branches taken from `branches`
    {"obs_prep": on (rows, 64), "common": on (rows, 64)}, in minibatch row order."""
    def trunk(p, cfg, obs):
        h = F.linear(obs, p["obs_prep.mlp.fc1.0.weight"], p["obs_prep.mlp.fc1.0.bias"])
        h = _act_teacher_forced(h, cfg.activation_id, branches["obs_prep"])
        h = F.layer_norm(h, h.shape[-1:], p["obs_prep.mlp.fc1.2.weight"], p["obs_prep.mlp.fc1.2.bias"])
        h = F.linear(h, p["obs_prep.mlp.fc3.0.weight"], p["obs_prep.mlp.fc3.0.bias"])
        h = F.layer_norm(h, h.shape[-1:], p["obs_prep.mlp.fc3.1.weight"], p["obs_prep.mlp.fc3.1.bias"])
        h = _act_teacher_forced(F.linear(h, p["common.fc1.0.weight"], p["common.fc1.0.bias"]), cfg.activation_id,
                                branches["common"])
        h = F.layer_norm(h, h.shape[-1:], p["common.fc1.2.weight"], p["common.fc1.2.bias"])
        h = F.linear(h, p["common.fc3.0.weight"], p["common.fc3.0.bias"])
        return F.layer_norm(h, h.shape[-1:], p["common.fc3.1.weight"], p["common.fc3.1.bias"])
    return trunk


def _critic_forward_detached(p, cfg, obs, rnn_states=None, masks=None):
    """Mutant: the value head reads the shared trunk's feature as a constant."""
    f = nets.shared_trunk(p, cfg, obs).detach()
    return F.linear(f, p["v_out.weight"], p["v_out.bias"]), rnn_states


# name: (what it changes, the compared quantity that must catch it, cfg options it needs, the head it runs on)
# The quantity is "grad <block>", "param <block>" or "train_info critic grad norm".
MUTANTS = {
    "last-row-block-dropped": ("the rows of the last 1024-row tape block left out, the minibatch's loss weights kept",
                               "grad v_out.bias", {}, "categorical"),
    "value-grad-stops-at-head": ("the value loss does not back-propagate into common / obs_prep",
                                 "grad obs_prep.mlp.fc1.0.weight", {}, "categorical"),
    "adam-with-critic-lr": ("the shared Adam steps with critic_lr instead of lr", "param common.fc1.0.weight",
                            dict(critic_lr=2e-3), "categorical"),
    "critic-norm-unclipped": ("critic_grad_norm reported as the norm before the first clip", "train_info critic grad norm",
                              dict(max_grad_norm=0.05), "categorical"),
    "vn-target-before-update": ("ValueNorm target from the state before this minibatch's update", "grad v_out.weight", {},
                                "categorical"),
    "entropy-weight-1/rows": ("entropy weight 1/rows instead of 1/(rows n) without policy active masks",
                              "grad act.action_out.logstd._bias", dict(use_policy_active_masks=False), "gaussian"),
    "action-mask-ignored-in-update": ("the update evaluates the masked Categorical without its action masks",
                                      "grad act.action_out.linear.weight", {}, "categorical-masked"),
}


def target(out, what, dims, head):
    """The compared quantity a MUTANTS entry names, from an `update` result."""
    if what == "train_info critic grad norm":
        return out["norms"][1].reshape(1)
    kind, name = what.split(" ", 1)
    return out["grad" if kind == "grad" else "p"][blocks(*dims, head)[name]]


def adam_from(cfg, state, grad, dims, head, dtype=torch.float64):
    """The optimiser step alone (both clip_grad_norm_ calls, one Adam step with lr = cfg.lr) from a given gradient:
    the parameters, exp_avg, exp_avg_sq and step count after it."""
    cast = lambda x: torch.as_tensor(x).to(device=grad.device, dtype=dtype)   # noqa: E731
    ocfg = ffma_ref64.oracle_cfg(cfg)
    p = unflatten(cast(state["p"]), *dims, head)
    opt, _ = oppo.make_optimizers(ocfg, p, p)
    ffma_ref64._seed_adam(opt, p.values(), unflatten(cast(state["m"]), *dims, head), unflatten(cast(state["v"]), *dims, head),
                          state["step"])
    for q, g in zip(p.values(), unflatten(cast(grad), *dims, head).values()):
        q.grad = g
    if ocfg.use_max_grad_norm:
        for _ in range(2):
            torch.nn.utils.clip_grad_norm_(list(p.values()), ocfg.max_grad_norm)
    opt.step()
    st = [opt.state[q] for q in p.values()]
    return dict(p=torch.cat([q.detach().reshape(-1) for q in p.values()]), m=torch.cat([s["exp_avg"].reshape(-1) for s in st]),
                v=torch.cat([s["exp_avg_sq"].reshape(-1) for s in st]), step=int(st[0]["step"]))


def update(cfg, buf, state, rows, dims, head, dtype=torch.float64, vn_beta=0.99999, mutant=None, branches=None):
    """One minibatch update of the shared model in `dtype` on the buffer rows `rows`.

    cfg: the project's option names (clip_param, entropy_coef, ..., lr, critic_lr, use_valuenorm, use_adv_normalize, a2c).
    buf: (rows, width) arrays obs, actions, action_log_probs, advantages, value_preds, returns, active_masks
      [, action_masks]; the advantages are normalised over every row of buf["advantages"] (the GAE moments).
    state: flat parameters p, Adam moments m, v, step count step, ValueNorm state vn (3,).  dims: (d, n).
    head: "gaussian" or "categorical".  mutant: a key of MUTANTS.
    branches: None, or a kernel's own ReLU / LeakyReLU branches {"obs_prep": on, "common": on} ((rows, 64) bool, in
      minibatch order), which the reference takes at the pre-activations within BRANCH_TIE of the kink (teacher
      forcing, as a rollout is teacher-forced on the kernel's actions)."""
    d, n = dims
    dev = rows.device
    cast = lambda x: torch.as_tensor(x).to(device=dev, dtype=dtype)   # noqa: E731
    ocfg = ffma_ref64.oracle_cfg(cfg)
    p = unflatten(cast(state["p"]), d, n, head)
    opt, _ = oppo.make_optimizers(ocfg, p, p)
    ffma_ref64._seed_adam(opt, p.values(), unflatten(cast(state["m"]), d, n, head), unflatten(cast(state["v"]), d, n, head),
                          state["step"])
    if mutant == "adam-with-critic-lr":
        opt.param_groups[0]["lr"] = ocfg.critic_lr
    vn = None
    if cfg.use_valuenorm:
        vn_cls = ffma_ref64._StaleTargetValueNorm if mutant == "vn-target-before-update" else oppo.ValueNormState
        vn = vn_cls([float(x) for x in state["vn"]], beta=vn_beta, dtype=dtype, device=dev)

    R = buf["advantages"].shape[0]
    adv = rnn_ref64.normalized_advantages(buf["advantages"].to(dtype), buf["active_masks"][:R].to(dtype), cfg.use_adv_normalize)

    def batch_of(idx):
        g = lambda key: buf[key].to(device=dev, dtype=dtype)[idx]   # noqa: E731
        obs = g("obs")
        b = dict(policy_obs=obs, critic_obs=obs, actions=g("actions"), old_logp=g("action_log_probs"), value_preds=g("value_preds"),
                 returns=g("returns"), active_masks=g("active_masks"), adv=adv[idx])
        if "action_masks" in buf and mutant != "action-mask-ignored-in-update":
            b["action_masks"] = g("action_masks")
        return b

    def patches(positions):
        """The oracle with the tie branches of the minibatch positions `positions` and the mutant's change."""
        stack = contextlib.ExitStack()
        if branches is not None:
            stack.enter_context(mock.patch.object(nets, "shared_trunk", _trunk_teacher_forced(
                {k: v[positions] for k, v in branches.items()})))
        if mutant == "entropy-weight-1/rows":
            stack.enter_context(mock.patch.object(nets, "policy_eval_gaussian", ffma_ref64._mutant_eval(mutant)))
        elif mutant == "value-grad-stops-at-head":
            stack.enter_context(mock.patch.object(nets, "critic_forward", _critic_forward_detached))
        return stack

    batch = batch_of(rows)
    rec = {}
    with patches(slice(None)):
        vl, cgn, pl, ent, agn, _ = oppo.ppo_update(ocfg, p, p, opt, opt, vn, batch, record=rec)

    grad = torch.cat([x.reshape(-1) for x in rec["grads_policy"].values()])
    act = batch["active_masks"]
    wsum = (lambda x: (x * act).sum() / act.sum()) if ocfg.use_policy_active_masks else (lambda x: x.mean())   # noqa: E731
    ratio = rec["ratio"].to(device=dev, dtype=dtype)
    ratio_sum = ratio.mean(-1).sum() if not ocfg.a2c else torch.zeros((), dtype=dtype, device=dev)
    sums = torch.stack([rec["policy_loss"], rec["entropy"], ratio_sum, rec["value_loss"]])
    scales = torch.stack([wsum(rec["surr"].abs().sum(-1, keepdim=True)), rec["entropy"].abs(), ratio_sum, rec["value_loss"]])
    norms = torch.tensor([agn, agn if mutant == "critic-norm-unclipped" else cgn], dtype=dtype, device=dev)
    st = [opt.state[q] for q in p.values()]
    out = dict(grad=grad, losses=sums, loss_scales=scales, norms=norms, ratio_mean=ratio_sum / rows.numel(),
               ratio_spread=(ratio - 1).abs().max() if not ocfg.a2c else None,
               vn=None if vn is None else torch.as_tensor(vn.state()).to(dev),
               p=torch.cat([q.detach().reshape(-1) for q in p.values()]), m=torch.cat([s["exp_avg"].reshape(-1) for s in st]),
               v=torch.cat([s["exp_avg_sq"].reshape(-1) for s in st]), step=int(st[0]["step"]))

    if mutant == "last-row-block-dropped":
        # the loss is a weighted sum of per-row terms: remove the dropped rows' share at the minibatch's weights (and with
        # the minibatch's ValueNorm update); both loss terms weight rows alike when both active-mask options agree
        assert ocfg.use_policy_active_masks == ocfg.use_value_active_masks
        first = (rows.numel() - 1) // TAPE_ROW_BLOCK * TAPE_ROW_BLOCK
        drop = rows[first:]
        pd = unflatten(cast(state["p"]), d, n, head)
        opt_d, _ = oppo.make_optimizers(ocfg, pd, pd)
        vn_d = None
        if cfg.use_valuenorm:
            vn_d = _BatchReturnsValueNorm([float(x) for x in state["vn"]], beta=vn_beta, dtype=dtype, device=dev,
                                          batch_returns=batch["returns"])
        rec_d = {}
        with patches(slice(first, None)):
            oppo.ppo_update(ocfg, pd, pd, opt_d, opt_d, vn_d, batch_of(drop), record=rec_d)
        a_all = buf["active_masks"].to(device=dev, dtype=dtype)
        share = (a_all[drop].sum() / a_all[rows].sum() if ocfg.use_policy_active_masks
                 else torch.tensor(drop.numel() / rows.numel(), dtype=dtype, device=dev))
        out["grad"] = grad - share * torch.cat([x.reshape(-1) for x in rec_d["grads_policy"].values()])
    return out
