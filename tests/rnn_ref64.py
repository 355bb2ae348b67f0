"""High-precision reference of the recurrent MAPPO update: one minibatch of `orl_rnn_fwdbwd` + `orl_rnn_apply`.

TEST INFRASTRUCTURE.  Built on the dtype-agnostic oracle networks (oracle/nets.py `rnn_layer`, `policy_eval`,
`critic_forward`), so the same code runs in float64 (the reference) and in float32 (the yardstick for how far a
correct fp32 implementation may drift from it); pinned to the unmodified reference's traces by
tests/test_rnn_ref64_cpu.py.

Inputs are the device buffer layout: every array is (slots, N, A, ...) or (slots, B, ...), so row t*B + b of
`rows(x)` is (step t, agent row b).  Chunks follow the kernels' gathers:
- ordinary recurrent chunks (`chunk_row_indices`): sample f = b*T + t, chunk c covers f in [c*L, c*L + L);
- JRPO chunks (`v3_row_indices`): sample f = n*T + t carries the A agent rows n*A + a.
A chunk starts from the hidden state stored at its first step; `rnn_layer` applies `h * mask_t` before every step.

`update` returns the true (pre-clip) gradients of both nets flattened in state_dict order, the four loss sums in
`loss_acc` order (policy loss, entropy, ratio sum, value loss), the gradient norms, and the parameters, Adam moments,
Adam step counts and ValueNorm state after the global-norm clip and Adam.
"""
import math
import types

import torch

import param_layout as layout
from oracle import nets

H = layout.H


def param_shapes(d, n, critic):
    """(state_dict name, shape) of a recurrent policy (head width n) or critic net on d-wide observations, in the
    order of the flat parameter buffer (orl_rnn_core.h rnn_offsets)."""
    return (layout.mlp_trunk(d) + [("rnn.rnn.weight_ih_l0", (3 * H, H)), ("rnn.rnn.weight_hh_l0", (3 * H, H)),
                                   ("rnn.rnn.bias_ih_l0", (3 * H,)), ("rnn.rnn.bias_hh_l0", (3 * H,)),
                                   ("rnn.norm.weight", (H,)), ("rnn.norm.bias", (H,))]
            + layout.head(n, "critic" if critic else "categorical"))


def blocks(d, n, critic):
    """{name: slice of the flat buffer} in flat order."""
    return layout.blocks(param_shapes(d, n, critic))


def unflatten(flat, d, n, critic):
    """Leaf tensors (requires_grad) viewing copies of the flat buffer, keyed by state_dict name."""
    return {name: x.requires_grad_(True) for name, x in layout.unflatten(flat, param_shapes(d, n, critic)).items()}


def rows(x):
    """(slots, ..., w) -> (slots * B, w): row t*B + b."""
    return x.reshape(-1, x.shape[-1])


def net_cfg(activation_id, use_policy_active_masks):
    return types.SimpleNamespace(layer_N=1, activation_id=activation_id, use_recurrent_policy=True,
                                 use_naive_recurrent_policy=False, use_policy_active_masks=use_policy_active_masks)


def normalized_advantages(adv, active, use_adv_normalize):
    """ppo.py:384-409 on the buffer's raw advantages (T*B rows): optional normalisation over every row, then the
    normalisation over the active rows; population standard deviations."""
    if use_adv_normalize:
        adv = (adv - adv.mean()) / (adv.std(unbiased=False) + 1e-5)
    sel = adv[active != 0]
    return (adv - sel.mean()) / (sel.std(unbiased=False) + 1e-5)


def vn_update(vn, ret, beta):
    """ValueNorm.update (valuenorm.py:59-76) with this minibatch's returns, in the working dtype."""
    w = beta
    return torch.stack([vn[0] * w + ret.mean() * (1 - w), vn[1] * w + (ret ** 2).mean() * (1 - w), vn[2] * w + (1 - w)])


def vn_normalize(vn, x):
    m = vn[0] / vn[2].clamp(min=1e-5)
    msq = vn[1] / vn[2].clamp(min=1e-5)
    return (x - m) / (msq - m * m).clamp(min=1e-2).sqrt()


def huber(e, d):
    a = (e.abs() <= d).to(e.dtype)
    return a * e ** 2 / 2 + (1 - a) * d * (e.abs() - d / 2)


def gather(T, B, A, L, ids, joint):
    """Buffer rows of a minibatch of chunks, time-major: policy rows (L, m) and critic rows (L, n)."""
    lane = torch.arange(L, device=ids.device)
    f = (ids[None, :] * L + lane[:, None])                              # (L, n)
    if not joint:
        r = (f % T) * B + f // T
        return r, r
    r0 = (f % T) * B + (f // T) * A                                     # agent 0 of every sample
    return (r0[:, :, None] + torch.arange(A, device=ids.device)).reshape(L, -1), r0


def forward(cfg, buf, pol, cri, ids, L, joint, dtype):
    """Chunk forward of both nets: policy rows rp (L, m), critic rows rc (L, n), log-probs of the recorded actions
    and entropy (policy rows, time-major), values (critic rows, time-major)."""
    T = buf["actions"].shape[0]
    B = rows(buf["actions"]).shape[0] // T
    A = buf["actions"].shape[2] if joint else 1
    rp, rc = gather(T, B, A, L, ids, joint)
    g = lambda key, r: rows(buf[key]).to(dtype)[r.reshape(-1)]   # noqa: E731
    ncfg = net_cfg(cfg.activation_id, cfg.use_policy_active_masks)
    # policy: every row of the chunks (every agent row of the JRPO samples)
    logp, ent = nets.policy_eval(pol, ncfg, g("policy_obs", rp), g("actions", rp), None, g("active_masks", rp),
                                 g("rnn_states", rp[0]).unsqueeze(1), g("masks", rp))
    # critic: the chunk rows (agent 0's row of every JRPO sample)
    values, _ = nets.critic_forward(cri, ncfg, g("critic_obs", rc), g("rnn_states_critic", rc[0]).unsqueeze(1), g("masks", rc))
    return rp, rc, logp, ent, values


def losses(cfg, buf, pol, cri, ids, L, joint, dtype, vn=None):
    """Forward of one minibatch: (policy loss, entropy, value loss, loss sums, loss scales, ValueNorm state after the
    update).  The scale of a loss is the same weighted sum over absolute terms: the magnitude its rounding error is
    relative to (the policy loss of a whole buffer at ratio 1 is a sum of normalised advantages, ~0).
    cfg carries the reference's option names (clip_param, use_huber_loss, ...)."""
    T = buf["actions"].shape[0]
    B = rows(buf["actions"]).shape[0] // T
    A = buf["actions"].shape[2] if joint else 1
    rp, rc, logp, ent, values = forward(cfg, buf, pol, cri, ids, L, joint, dtype)
    g = lambda key, r: rows(buf[key]).to(dtype)[r.reshape(-1)]   # noqa: E731
    act_all = rows(buf["active_masks"]).to(dtype)
    adv_all = normalized_advantages(rows(buf["advantages"]).to(dtype), act_all[:T * B], cfg.use_adv_normalize)
    old = g("action_log_probs", rp)
    if joint:   # ratio of the joint action of the A agents of a sample; agent 0's advantage and active mask
        logp, old = logp.view(-1, A).sum(-1, keepdim=True), old.view(-1, A).sum(-1, keepdim=True)
    adv, act = adv_all[rc.reshape(-1)], g("active_masks", rc)
    ratio = torch.exp(logp - old)
    if getattr(cfg, "dual_clip_ppo", False):
        ratio = torch.minimum(ratio, torch.tensor(cfg.dual_clip_coeff, dtype=dtype, device=ratio.device))
    surr = torch.min(ratio * adv, torch.clamp(ratio, 1.0 - cfg.clip_param, 1.0 + cfg.clip_param) * adv)
    wmean = (lambda x: (x * act).sum() / act.sum()) if cfg.use_policy_active_masks else (lambda x: x.mean())   # noqa: E731
    policy_loss, policy_scale = wmean(-surr), wmean(surr.detach().abs())

    vp, ret = g("value_preds", rc), g("returns", rc)
    clipped = vp + (values - vp).clamp(-cfg.clip_param, cfg.clip_param)
    vn_after = None
    target = ret
    if vn is not None:
        vn_after = vn_update(vn.to(dtype), ret, cfg.vn_beta)
        target = vn_normalize(vn_after, ret)
    e_c, e_o = target - clipped, target - values
    if cfg.use_huber_loss:
        l_c, l_o = huber(e_c, cfg.huber_delta), huber(e_o, cfg.huber_delta)
    else:
        l_c, l_o = e_c ** 2 / 2, e_o ** 2 / 2
    vl = torch.max(l_o, l_c) if cfg.use_clipped_value_loss else l_o
    value_loss = (vl * act).sum() / act.sum() if cfg.use_value_active_masks else vl.mean()
    sums = torch.stack([policy_loss.detach(), ent.detach(), ratio.detach().sum(), value_loss.detach()])
    scales = torch.stack([policy_scale, ent.detach(), ratio.detach().sum(), value_loss.detach()])
    return policy_loss, ent, value_loss, sums, scales, vn_after


def adam_step(flat, g, m, v, step, lr, cfg):
    """clip_grad_norm_ (already applied to g) + weight decay + torch.optim.Adam, one step.  The betas are the float32
    values the kernels receive (OrlRnnArgs.adam_beta1/2): with beta2 = 0.999f, 1 - beta2 is 1.3e-5 smaller than
    torch's 1 - 0.999, which moves exp_avg_sq by that relative amount."""
    b1, b2 = (float(torch.tensor(b, dtype=torch.float32)) for b in getattr(cfg, "adam_betas", (0.9, 0.999)))
    if cfg.weight_decay:
        g = g + cfg.weight_decay * flat
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    step = step + 1
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    return flat - (lr / bc1) * m / (v.sqrt() / math.sqrt(bc2) + cfg.opti_eps), m, v, step


def update(cfg, buf, state, ids, L, dims, joint=False, dtype=torch.float64):
    """One minibatch of the recurrent update in `dtype`.

    cfg: the reference's option names (clip_param, entropy_coef, value_loss_coef, huber_delta, max_grad_norm,
      use_max_grad_norm, use_huber_loss, use_clipped_value_loss, use_value_active_masks, use_policy_active_masks,
      use_adv_normalize, dual_clip_ppo, dual_clip_coeff, activation_id, lr, critic_lr, opti_eps, weight_decay,
      vn_beta; use_valuenorm decides whether state["vn"] is used).
    buf: device-layout arrays policy_obs, critic_obs, rnn_states, rnn_states_critic, masks, active_masks (T+1 slots),
      actions, action_log_probs, advantages (T slots), value_preds, returns (T or T+1 slots).
    state: flat parameters pol / cri, Adam moments pol_m, pol_v, cri_m, cri_v, step counts steps = (pol, cri),
      ValueNorm state vn (3,).
    dims: (d, n, dc).  ids: chunk ids of the minibatch."""
    d, n, dc = dims
    dev = ids.device
    cast = lambda x: torch.as_tensor(x).to(device=dev, dtype=dtype)   # noqa: E731
    pol = unflatten(cast(state["pol"]), d, n, False)
    cri = unflatten(cast(state["cri"]), dc, 1, True)
    vn = cast(state["vn"]) if cfg.use_valuenorm else None
    policy_loss, ent, value_loss, sums, scales, vn_after = losses(cfg, buf, pol, cri, ids, L, joint, dtype, vn)
    gp = torch.cat([x.reshape(-1) for x in torch.autograd.grad(policy_loss - ent * cfg.entropy_coef, list(pol.values()))])
    gc = torch.cat([x.reshape(-1) for x in torch.autograd.grad(value_loss * cfg.value_loss_coef, list(cri.values()))])
    out = dict(grad_pol=gp, grad_cri=gc, losses=sums, loss_scales=scales, norms=(gp.norm(), gc.norm()),
               vn=vn_after if vn_after is not None else (cast(state["vn"]) if "vn" in state else None))
    for key, g, lr, k in (("pol", gp, cfg.lr, 0), ("cri", gc, cfg.critic_lr, 1)):
        norm = g.norm()
        if cfg.use_max_grad_norm:
            g = g * torch.clamp(cfg.max_grad_norm / (norm + 1e-6), max=1.0)
        p, m, v, s = adam_step(cast(state[key]), g, cast(state[key + "_m"]), cast(state[key + "_v"]), int(state["steps"][k]), lr, cfg)
        out[key], out[key + "_m"], out[key + "_v"], out[key + "_step"] = p, m, v, s
    return out
