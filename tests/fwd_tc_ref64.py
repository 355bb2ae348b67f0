"""Float64 reference of the tensor-core forward passes (orl_fwd_tc.cu: `critic_values_tc_kernel`, `rollout_tc_kernel`,
`rollout_cartpole_rows_kernel`), the per-row error scale their bars are measured against, and deliberate mistakes
("mutants") of them.

TEST INFRASTRUCTURE.  The forward is the oracle's (oracle/nets.py `mlp_base`, `categorical_logits`, `critic_forward`)
over the flat parameter vector (tests/ffma_ref64.py `unflatten`), for the 64-wide trunk with one fc1 and one fc3 layer.
The kernels run it with the LayerNorm affines folded into the next linear layer (orl_mlp.cuh `folded_w3` ...
`folded_bh`):
    W3f = W3 diag(g1),  b3f = b3 + W3 be1,  whf = Wh diag(g3),  bhf = bh + Wh be3,
and fc3 as three fp16 tensor-core passes over split operands (x = hi + lo, hi = fp16(x), lo = fp16(x - hi)):
    n1 . W3f^T  ~=  Al.Bh + Ah.Bl + Ah.Bh   (A = n1, B = W3f).
`folded` restates that forward in float64, exactly or with the split emulated, and with each mutant's mistake.

Per-row error scale.  For row r and output j,
    S_rj = sum_k |whf_jk| (|x3_rk| + rstd3_r A3_rk) + |bhf_j|,   A3_rk = sum_i |n1_ri| |W3f_ki| + |b3f_k|,
where x3 is the LayerNorm-3 output, rstd3 its 1 / sqrt(var + eps), and the weights are the folded ones in float64.  It is
the first-order bound of a forward whose fc3 products and head sums are each rounded at a relative size e: |error_rj| <=
e S_rj.  An error of n1 (LayerNorm-1) enters through A3.

Subnormal floor.  A split half below 2^-14, fp16's smallest normal, is rounded on the fixed subnormal grid of 2^-24: an
absolute error of up to 2^-25, whatever the element's size, where the split's relative model allows 2^-22 |x|.  For the
weights that excess is a fixed property of the net, proportional to |n1|, and TAU carries it.  For n1 it is not: a row
whose LayerNorm-1 variance is far below eps (an initial net, b1 = 0, and an observation near 0) has n1 elements far below
2^-14, and its error relative to S grows without bound as the observation shrinks.  The floor carries n1's excess through
fc3 and the head:
    D_rj = sum_k |whf_jk| rstd3_r F3_rk,   F3_rk = sum_i |W3f_ki| max(0, 2^-25 - 2^-22 |n1_ri|),
and the bars are TAU S + D.  It is zero for n1 elements of 2^-3 and more, and small against TAU S on ordinary rows."""
import types

import torch

import ffma_ref64
from oracle import nets

H = 64
LN_EPS = 1e-5
SUBNORMAL = 2.0 ** -25   # half the spacing of fp16's subnormals

# name: what the mutant changes (`folded(mutant=...)` for the first four; the last two act on kernel outputs / inputs)
MUTANTS = {
    "fc3-hi-only": "fc3 from Ah.Bh alone",
    "fc3-no-Al": "fc3 without the Al.Bh pass",
    "ln-eps-dropped": "both LayerNorms without eps",
    "ln1-bias-fold-dropped": "b3f without its W3.be1 term (invisible on initial nets, whose be1 is 0)",
    "stale-tile": "critic pass: one CTA's k-th tile gets the values of its (k-1)-th tile's rows",
    "noise-row-shifted": "rollout: the noise q of row e + 1 instead of row e",
}
FORWARD_MUTANTS = ("fc3-hi-only", "fc3-no-Al", "ln-eps-dropped", "ln1-bias-fold-dropped")


def _head_names(head):
    return ("v_out.weight", "v_out.bias") if head == "critic" else ("act.action_out.linear.weight", "act.action_out.linear.bias")


def params(flat, d, n, head):
    """{state_dict name: float64 tensor} of a flat parameter vector; head: "categorical" or "critic"."""
    return ffma_ref64.unflatten(flat.double(), d, n, head)


def forward(flat, d, n, head, obs, activation_id):
    """The oracle's float64 forward of (rows, d) observations: values (rows, 1) for a critic, raw logits (rows, n) for a
    Categorical head (nets.categorical_logits is their log-softmax)."""
    p = params(flat, d, n, head)
    cfg = _net_cfg(activation_id)
    x = obs.double()
    if head == "critic":
        return nets.critic_forward(p, cfg, x)[0]
    wn, bn = _head_names(head)
    return torch.nn.functional.linear(nets.mlp_base(p, "base", x, 1, activation_id), p[wn], p[bn])


def _net_cfg(activation_id):
    return types.SimpleNamespace(layer_N=1, activation_id=activation_id, use_recurrent_policy=False,
                                 use_naive_recurrent_policy=False)


def fold(p, head, drop_ln1_bias=False):
    """The kernels' folded weights in float64: W1, b1, W3f, b3f, whf, bhf."""
    wn, bn = _head_names(head)
    W3, g1, be1 = p["base.mlp.fc3.0.weight"], p["base.mlp.fc1.2.weight"], p["base.mlp.fc1.2.bias"]
    Wh, g3, be3 = p[wn], p["base.mlp.fc3.1.weight"], p["base.mlp.fc3.1.bias"]
    b3f = p["base.mlp.fc3.0.bias"] + (0.0 if drop_ln1_bias else W3 @ be1)
    return dict(W1=p["base.mlp.fc1.0.weight"], b1=p["base.mlp.fc1.0.bias"], W3f=W3 * g1[None, :], b3f=b3f,
                whf=Wh * g3[None, :], bhf=p[bn] + Wh @ be3)


def split16(x):
    """(hi, lo) of the kernels' split-fp16 operands, as float64: hi = fp16(x), lo = fp16(x - hi)."""
    hi = x.to(torch.float16).double()
    return hi, (x - hi).to(torch.float16).double()


def fc3_split(n1, W3f, passes=("lh", "hl", "hh")):
    """n1 . W3f^T from the split operands: "lh" = Al.Bh, "hl" = Ah.Bl, "hh" = Ah.Bh, each product exact in float64."""
    (ah, al), (bh, bl) = split16(n1), split16(W3f)
    ops = {"lh": (al, bh), "hl": (ah, bl), "hh": (ah, bh)}
    return sum(a @ b.t() for a, b in (ops[k] for k in passes))


def _ln(x, eps):
    mu = x.mean(-1, keepdim=True)
    var = x.var(-1, unbiased=False, keepdim=True)
    rstd = (var + eps).rsqrt()
    return (x - mu) * rstd, rstd, mu.abs()[:, 0] / var.sqrt()[:, 0]


def folded(flat, d, n, head, obs, activation_id, mutant=None, split=False):
    """The folded float64 forward: out (rows, n), the error scale S and the subnormal floor D (rows, n), and the |mu| /
    sigma of the LayerNorm-1 and LayerNorm-3 inputs per row (mu_sigma1, mu_sigma3).  split: fc3 through the split-fp16 emulation; mutant: one of
    FORWARD_MUTANTS."""
    assert mutant in (None,) + FORWARD_MUTANTS, mutant
    f = fold(params(flat, d, n, head), head, drop_ln1_bias=mutant == "ln1-bias-fold-dropped")
    eps = 0.0 if mutant == "ln-eps-dropped" else LN_EPS
    x = obs.double()
    n1, _, ms1 = _ln(nets.activation(x @ f["W1"].t() + f["b1"], activation_id), eps)
    if mutant == "fc3-hi-only":
        z3 = fc3_split(n1, f["W3f"], ("hh",))
    elif mutant == "fc3-no-Al":
        z3 = fc3_split(n1, f["W3f"], ("hl", "hh"))
    elif split:
        z3 = fc3_split(n1, f["W3f"])
    else:
        z3 = n1 @ f["W3f"].t()
    z3 = z3 + f["b3f"]
    x3, rstd3, ms3 = _ln(z3, eps)
    out = x3 @ f["whf"].t() + f["bhf"]
    A3 = n1.abs() @ f["W3f"].abs().t() + f["b3f"].abs()
    S = (x3.abs() + rstd3 * A3) @ f["whf"].abs().t() + f["bhf"].abs()
    F3 = (SUBNORMAL - 2.0 ** -22 * n1.abs()).clamp(min=0) @ f["W3f"].abs().t()
    D = (rstd3 * F3) @ f["whf"].abs().t()
    return dict(out=out, S=S, D=D, A3=A3, mu_sigma1=ms1, mu_sigma3=ms3)


def reference(flat, d, n, head, obs, activation_id):
    """What the GPU tests compare against: the oracle's out, the folded forward's S, D and |mu| / sigma."""
    r = folded(flat, d, n, head, obs, activation_id)
    r["out"] = forward(flat, d, n, head, obs, activation_id)
    return r


def stale_tile(values, rows, grid, cta, k, tile_rows=128):
    """Mutant "stale-tile" of a critic pass over `rows` rows on `grid` CTAs: CTA `cta`'s k-th tile (k >= 1) carries the
    values of the rows of its (k-1)-th tile.  Returns the mutated copy and the rows that changed."""
    assert k >= 1
    t_now, t_prev = cta + k * grid, cta + (k - 1) * grid
    lo, hi = t_now * tile_rows, min((t_now + 1) * tile_rows, rows)
    assert lo < rows, "the CTA has no k-th tile"
    out = values.clone()
    out[lo:hi] = values[t_prev * tile_rows:t_prev * tile_rows + (hi - lo)]
    return out, torch.arange(lo, hi, device=values.device)


def noise_row_shifted(q):
    """Mutant "noise-row-shifted" of a (T, rows, n) noise table: row e draws with the q of row e + 1 (the last row keeps
    its own)."""
    out = q.clone()
    out[:, :-1] = q[:, 1:]
    return out
