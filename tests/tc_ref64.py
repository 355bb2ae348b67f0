"""The float64 reference of one PPO minibatch update (tests/ffma_ref64.py) with, per parameter block, the magnitude of
the terms a kernel adds up to that block's gradient, and the deliberate mistakes of the tensor-core update kernel
(`ppo_fwdbwd_tc_kernel`, orl_ppo_tc.cu) that the bars of tests/test_ppo_tc_scale_cuda.py must catch.

TEST INFRASTRUCTURE.  A gradient block is a sum over the minibatch rows of one term c_r per row.  With advantages of
both signs these terms cancel: the block's norm can be orders of magnitude below the terms', and a correct float32
kernel is then far off in relative L2 while each of its roundings is tiny against what it adds.  So the bar of a block is
set against S_block = || sum_r |c_r| ||_2 (element-wise absolute values), which the oracle's float64 graph already holds:
every layer is one `F.linear` or `F.layer_norm` call (oracle/nets.py), whose input x and output gradient dL/dy give

    linear weight   c_r = dy_r^T x_r         linear bias   c_r = dy_r
    LayerNorm gain  c_r = dy_r * xhat_r      LayerNorm bias c_r = dy_r       (xhat: the normalised input)

`update` also returns the signed sums of the same terms (tests/test_tc_ref64_cpu.py pins them to the reference gradient)
and, per net, the peaks of the backward operands the kernel converts to split fp16 (dZ3 = dL/d fc3 output, dZ1 = dL/d
fc1 output, U = dL/dhead * rstd3) before its per-minibatch power-of-two scales are applied (`operand_scales`).
"""
import math

import torch
import torch.nn.functional as F

import ffma_ref64 as ref

H = ref.H
FP16_MAX = 65504.0   # the largest finite fp16: split conversions saturate here (cvt.rn.satfinite)

# name: (what it changes, the gradient block that must catch it)
TC_MUTANTS = {
    "cta-last-tile-dropped": ("the rows of one CTA's last tile left out", "grad pol.base.mlp.fc1.0.weight"),
    "stale-staged-tile": ("one CTA's k-th tile computed on the rows of its (k-1)-th tile (a staging parity slip)",
                          "grad pol.base.mlp.fc1.0.weight"),
    "partial-tail-counted": ("the rows past the end of the partial last tile weighted like minibatch rows",
                             "grad pol.base.mlp.fc1.0.weight"),
    "dZ3-saturated": ("the scaled dZ3 of the policy net clamped at +-65504 (a saturating split conversion)",
                      "grad pol.base.mlp.fc3.0.weight"),
}


class _Capture:
    """Stands in for torch.nn.functional inside oracle/nets.py: records every linear / LayerNorm call on parameters of
    `params` with its input, its normalised input and its output (whose gradient is retained)."""

    def __init__(self, params, clamp_dz3=None):
        self.names = {id(v): k for k, v in params.items()}
        self.calls, self.clamp_dz3 = [], clamp_dz3

    def __getattr__(self, name):
        return getattr(F, name)

    def linear(self, x, w, b=None):
        y = F.linear(x, w, b)
        name = self.names.get(id(w))
        if name is not None:
            if self.clamp_dz3 is not None and name.endswith("fc3.0.weight") and name in self.clamp_dz3:
                lim = self.clamp_dz3[name]
                y.register_hook(lambda g: g.clamp(-lim, lim))
            y.retain_grad()
            self.calls.append(("linear", name, self.names.get(id(b)), x.detach(), y))
        return y

    def layer_norm(self, x, shape, w=None, b=None, eps=1e-5):
        y = F.layer_norm(x, shape, w, b, eps)
        name = self.names.get(id(w))
        if name is not None:
            y.retain_grad()
            var = x.detach().var(-1, unbiased=False, keepdim=True)
            xhat = F.layer_norm(x.detach(), shape, None, None, eps)
            self.calls.append(("layer_norm", name, self.names.get(id(b)), (xhat, torch.rsqrt(var + eps)), y))
        return y


def _block_terms(calls):
    """{parameter name: (signed sum of the row terms, sum of their absolute values)} from the recorded calls."""
    out = {}
    for kind, wname, bname, x, y in calls:
        dy = y.grad
        if kind == "linear":
            dy2, x2 = dy.reshape(-1, dy.shape[-1]), x.reshape(-1, x.shape[-1])
            out[wname] = (dy2.t() @ x2, dy2.abs().t() @ x2.abs())
        else:
            xhat = x[0]
            out[wname] = ((dy * xhat).reshape(-1, dy.shape[-1]).sum(0), (dy * xhat).abs().reshape(-1, dy.shape[-1]).sum(0))
        if bname is not None:
            dy2 = dy.reshape(-1, dy.shape[-1])
            out[bname] = (dy2.sum(0), dy2.abs().sum(0))
    return out


def _peaks(calls):
    """Peaks of the backward operands before scaling: max |dZ3|, max |dZ1| and max_r,j |dL/dhead_rj| rstd3_r."""
    by = {name: (x, y) for _, name, _, x, y in calls}
    fc1 = next(k for k in by if k.endswith("fc1.0.weight"))
    fc3 = next(k for k in by if k.endswith("fc3.0.weight"))
    ln3 = next(k for k in by if k.endswith("fc3.1.weight"))
    head = next(k for k in by if k.startswith(("act.", "v_out")))
    rstd3 = by[ln3][0][1]
    return dict(dz3=float(by[fc3][1].grad.abs().max()), dz1=float(by[fc1][1].grad.abs().max()),
                u=float((by[head][1].grad.abs() * rstd3).max()), rstd3=float(rstd3.max()))


def operand_scales(rows, head_w, ln3_gain):
    """(S_z, S_u) of the kernel for a net: powers of two from the rows the row weights divide by (sum(active) under the
    net's active-mask option, else the row count) and max |Whf| (tc_net_pass)."""
    whf = (head_w.double() * ln3_gain.double()[None, :]).float()
    wmax = float(whf.abs().max())
    e_rows = math.ceil(math.log2(max(float(rows), 1.0)))
    e_u = min(e_rows + 3, 60)
    e_z = min(max(e_rows + 3 - math.floor(math.log2(max(wmax, 1e-12))), 0), 60)
    return 2.0 ** e_z, 2.0 ** e_u


def net_operand_scales(state, dims, head, rows):
    """{"pol" | "cri": (S_z, S_u)}; rows: one count for both nets, or {"pol": .., "cri": ..}."""
    d, n, dc = dims
    rows = rows if isinstance(rows, dict) else {"pol": rows, "cri": rows}
    out = {}
    for net, dd, nn, hd in (("pol", d, n, head), ("cri", dc, 1, "critic")):
        p = ref.unflatten(state[net].double().cpu(), dd, nn, hd)
        hw = p["v_out.weight" if hd == "critic" else "act.action_out.linear.weight"]
        out[net] = operand_scales(rows[net], hw, p["base.mlp.fc3.1.weight"])
    return out


def update(cfg, buf, state, rows, dims, dtype=torch.float64, vn_beta=0.99999, clamp_dz3=None):
    """ffma_ref64.update with a Categorical head, plus `terms_pol` / `terms_cri` ({block: (signed row-term sum, sum of the
    absolute row terms)}, both flattened in the kernel's order; S_block is the norm of the second)
    and `peaks` ({"pol" | "cri": operand peaks}).  clamp_dz3: {"pol" | "cri": limit} clamps dL/d fc3-output of that net."""
    captures = []

    def functional(pol, cri):
        names = {**pol, **{"cri." + k: v for k, v in cri.items()}}
        lim = {("cri." if k == "cri" else "") + "base.mlp.fc3.0.weight": v for k, v in (clamp_dz3 or {}).items()}
        captures.append(_Capture(names, lim))
        return captures[-1]

    out = ref.update(cfg, buf, state, rows, dims, "categorical", dtype, vn_beta=vn_beta, functional=functional)
    calls = captures[0].calls
    pol_calls = [c for c in calls if not c[1].startswith("cri.")]
    cri_calls = [(k, w[4:], b[4:] if b else b, x, y) for k, w, b, x, y in calls if w.startswith("cri.")]
    for net, c in (("pol", pol_calls), ("cri", cri_calls)):
        out["terms_" + net] = {k: (a.reshape(-1), b.reshape(-1)) for k, (a, b) in _block_terms(c).items()}
    out["peaks"] = dict(pol=_peaks(pol_calls), cri=_peaks(cri_calls))
    return out


def _share(cfg, buf, part_rows, rows):
    a = buf["active_masks"][:, 0].double()
    if cfg.use_policy_active_masks:
        return float(a[part_rows].sum() / a[rows].sum())
    return part_rows.numel() / rows.numel()


def _policy_grad(cfg, buf, state, rows, dims, vn_beta):
    return ref.update(cfg, buf, state, rows, dims, "categorical", torch.float64, vn_beta=vn_beta)["grad_pol"]


def mutant_grad_pol(mutant, cfg, buf, state, rows, dims, clean, vn_beta=0.99999, add_rows=None, remove_rows=None,
                    clamp_dz3=None):
    """The policy gradient of the float64 reference with one mistake of TC_MUTANTS.  The policy loss and entropy are
    weighted means of per-row terms, so rows left out, doubled or swapped change the clean gradient by their weighted
    share: remove_rows are rows the mistake loses, add_rows rows it adds at the minibatch's row weights."""
    if mutant == "dZ3-saturated":
        return update(cfg, buf, state, rows, dims, vn_beta=vn_beta, clamp_dz3=clamp_dz3)["grad_pol"]
    g = clean["grad_pol"].clone()
    for part, sign in ((remove_rows, -1.0), (add_rows, 1.0)):
        if part is not None:
            g += sign * _share(cfg, buf, part, rows) * _policy_grad(cfg, buf, state, part, dims, vn_beta)
    return g


def blocks(dims, net):
    d, n, dc = dims
    return ref.blocks(d, n, "categorical") if net == "pol" else ref.blocks(dc, 1, "critic")
