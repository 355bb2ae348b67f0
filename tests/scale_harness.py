"""What the float64 scale tests of the update kernels share: the self-calibrated bar, the options, random nets and
synthetic buffers kept off every branch point of the loss, the hand-built kernel arguments, and the save / restore of a
live trainer's state (tests/test_rnn_scale_cuda.py, test_ppo_ffma_scale_cuda.py, test_ppo_tc_scale_cuda.py,
test_share_scale_cuda.py).

TEST INFRASTRUCTURE.  The bar of a quantity is self-calibrating: the reference runs once in float64 and once in float32
(TF32 off for matmul and cuDNN), and the kernel's error against float64 may be at most RATIO x the float32 reference's
error against float64, never less than the floor of the kernel under test and never more than CEIL (relative L2 norm
per block; relative error per scalar against the sum of its absolute terms)."""
import types

import pytest
import torch

import ffma_ref64
import rnn_ref64

RATIO, CEIL = 4.0, 1e-3
ATOL = 2e-5   # element-wise bar of rollout and critic quantities (tests/test_gru_cuda.py)
KINK = 5e-3   # synthetic rows keep at least this distance from every branch point of the loss
ACT_KINK = 1e-4   # synthetic fc1 pre-activations keep at least this distance from 0
# The floor of the recurrent kernels: the C3 entropy sum (153 600 terms added per lane, per CTA and by float atomics) is
# 1.1e-6 off float64, where torch's pairwise float32 sum is 1.6e-9 off: a long float32 sum in a fixed kernel order
# legitimately reaches ~1e-6.
RNN_FLOOR = 2e-6
# The floor of the two-net PPO update kernels (FFMA and tensor-core), 2.5x RNN_FLOOR, measured on an H100 SXM (132 SMs,
# 66 CTAs per net): an FFMA kernel thread adds its rows' weight-gradient terms in one fixed-order float32 chain (512
# terms per thread for the 64 x 54 critic fc1 gradient at 4 tiles per CTA, MG = 1) and a single-element block has no
# other elements to average over (the n = 1 head bias, 25k rows with cancellation); those reached 2.5e-6 and 3.2e-6
# against float64, where torch's pairwise float32 sums are 3e-7 off.  Every mutant of ffma_ref64 moves its block by 1e-2
# or more.
PPO_FLOOR = 5e-6


@pytest.fixture
def no_tf32():
    before = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = before


def rel(x, ref, scale=None):
    den = float(ref.double().norm()) if scale is None else float(scale)
    num = float((x.double() - ref.double()).norm())
    return num / den if den > 0 else num


class Checker:
    """Collects kernel-vs-float64 errors against the self-calibrated bar; fails with every violation listed."""

    def __init__(self, case, floor):
        self.case, self.bad, self.worst, self.floor = case, [], (0.0, ""), floor

    def bar(self, e32):
        return min(max(RATIO * e32, self.floor), CEIL)

    def __call__(self, what, got, r64, r32, scale=None):
        ek, e32 = rel(got, r64, scale), rel(r32, r64, scale)
        bar = self.bar(e32)
        ratio = ek / e32 if e32 > 0 else (0.0 if ek == 0 else float("inf"))
        if ratio > self.worst[0]:
            self.worst = (ratio, what)
        print(f"  {self.case:48s} {what:44s} kernel {ek:9.2e}  fp32 {e32:9.2e}  ratio {ratio:7.2f}")
        if not ek <= bar:
            self.bad.append(f"{what}: kernel {ek:.3e} > bar {bar:.3e} (fp32 {e32:.3e})")

    def done(self):
        print(f"  {self.case}: worst kernel/fp32 error ratio {self.worst[0]:.2f} ({self.worst[1]})")
        assert not self.bad, f"{self.case}:\n" + "\n".join(self.bad)


# ---------------------------------------------------------------- device helpers --------------------------------------

def lib():
    from openrl_b200 import lib
    return lib, lib.load()


def mb_stats(rows_idx, buf_returns, buf_active):
    """orl_minibatch_stats of the rows rows_idx: sum and sum of squares of the returns, sum of the active masks."""
    lb, L = lib()
    out = torch.zeros(3, dtype=torch.float64, device="cuda")
    lb.check(L.orl_minibatch_stats(lb.ptr(rows_idx), int(rows_idx.numel()), lb.ptr(buf_returns), lb.ptr(buf_active),
                                   lb.ptr(out), lb.current_stream()), "orl_minibatch_stats")
    return out


def gae_stats(buf):
    """The GAE moments of a synthetic buffer of (rows, 1) arrays advantages, active_masks and returns."""
    adv = buf["advantages"].double()[:, 0]
    act = buf["active_masks"].double()[:adv.numel(), 0] != 0
    ret = buf["returns"].double()[:adv.numel(), 0]
    return torch.stack([adv.sum(), (adv * adv).sum(), torch.tensor(float(adv.numel()), device="cuda", dtype=torch.float64),
                        adv[act].sum(), (adv[act] ** 2).sum(), ret.sum(), (ret * ret).sum(), act.double().sum()])


def loss_sums(folded, stride):
    """The four loss sums (policy loss, entropy, ratio sum, value loss) from the folded partials of the PPO update."""
    return torch.stack([folded[0, stride - 8], folded[0, stride - 7], folded[0, stride - 6], folded[1, stride - 8]]).clone()


# ---------------------------------------------------------------- options ---------------------------------------------

BASE = dict(use_huber_loss=True, use_clipped_value_loss=True, use_value_active_masks=True, use_policy_active_masks=True,
            use_valuenorm=True, use_adv_normalize=False, use_max_grad_norm=True, dual_clip_ppo=False, a2c=False, activation_id=1,
            clip_param=0.2, entropy_coef=0.01, value_loss_coef=0.5, huber_delta=1.0, max_grad_norm=1e3, dual_clip_coeff=3.0,
            lr=7e-4, critic_lr=5e-4, opti_eps=1e-5, weight_decay=0.0, vn_beta=0.99999)

# the option sets of tests/test_ppo_flags_cuda.py's flag matrix ("A2C" sets a2c), which the scale tests sweep too
CASES = [
    [],
    ["--use_huber_loss", "false"],
    ["--use_clipped_value_loss", "false"],
    ["--use_valuenorm", "false"],
    ["--use_value_active_masks", "false", "--use_policy_active_masks", "false"],
    ["--use_adv_normalize", "true"],
    ["--use_max_grad_norm", "false"],
    ["--weight_decay", "0.01", "--lr", "1e-3", "--critic_lr", "2e-3"],
    ["--activation_id", "0"],
    ["--activation_id", "2"],
    ["--activation_id", "3"],
    ["--clip_param", "0.05", "--entropy_coef", "0.05", "--value_loss_coef", "1.0", "--huber_delta", "0.5"],
    ["--max_grad_norm", "0.5"],
    ["--use_proper_time_limits", "true"],
    ["--use_gae", "false"],
    ["--dual_clip_ppo", "true", "--dual_clip_coeff", "1.05"],
    ["A2C"],
]


def ppo_flags(cfg):
    """The PPO_* option bits of a config."""
    lb, _ = lib()
    return ((lb.PPO_HUBER if cfg.use_huber_loss else 0) | (lb.PPO_CLIP_VALUE if cfg.use_clipped_value_loss else 0)
            | (lb.PPO_VALUE_ACTIVE_MASKS if cfg.use_value_active_masks else 0)
            | (lb.PPO_POLICY_ACTIVE_MASKS if cfg.use_policy_active_masks else 0) | (lb.PPO_VALUENORM if cfg.use_valuenorm else 0)
            | (lb.PPO_ADV_NORMALIZE if cfg.use_adv_normalize else 0) | (lb.PPO_MAX_GRAD_NORM if cfg.use_max_grad_norm else 0)
            | (lb.PPO_DUAL_CLIP if cfg.dual_clip_ppo else 0) | (lb.PPO_A2C if getattr(cfg, "a2c", False) else 0))


def flag_cfg(flags):
    """The parsed config of a CASES entry ("A2C" sets a2c), with the ValueNorm beta of BASE."""
    from openrl_b200.configs.config import create_config_parser

    a2c = "A2C" in flags
    cfg = create_config_parser().parse_args(["--seed", "3"] + [f for f in flags if f != "A2C"])
    return types.SimpleNamespace(**{**vars(cfg), "a2c": a2c, "vn_beta": 0.99999})


# ---------------------------------------------------------------- synthetic buffers -----------------------------------

def random_net(g, shapes):
    """A flat parameter vector with random weights over a reference's param_shapes list: std ~ 0.74 for a Gaussian
    head's logstd, weights at 1 / sqrt(fan-in) (0.3 of that in the heads), LayerNorm gains around 1, small biases."""
    parts = []
    for name, shp in shapes:
        x = torch.randn(shp, generator=g, device="cuda")
        if name.endswith("logstd._bias"):   # std ~ 0.74: policy gradients large enough for the 0.5 clip to act
            x = 0.2 * x - 0.3
        elif len(shp) == 2:
            x *= (0.3 if name.startswith(("act.", "v_out")) else 1.0) / shp[1] ** 0.5
        elif name.endswith("weight"):   # LayerNorm gains
            x = 1.0 + 0.2 * x
        else:
            x *= 0.1
        parts.append(x.reshape(-1))
    return torch.cat(parts)


def _redraw(bad, draw, x):
    return torch.where(bad, draw(x.shape), x)


def redraw_off_act_kink(g, obs, rows_idx, preacts):
    """Redraws the observations of the minibatch rows rows_idx (N(0, 1), in place) until no fc1 pre-activation lies
    within ACT_KINK of 0, where float32 rounding could take the other branch of a ReLU / LeakyReLU derivative.
    preacts(x): the pre-activations of the float64 rows x, one (rows, 64) tensor per checked layer."""
    for _ in range(50):
        x = obs[rows_idx].double()
        bad = torch.stack([(z.abs() < ACT_KINK).any(-1) for z in preacts(x)]).any(0)
        if not bool(bad.any()):
            break
        obs[rows_idx[bad]] = torch.randn(int(bad.sum()), x.shape[1], generator=g, device="cuda")
    assert not bool(bad.any()), "observations kept landing on an activation kink"


def draw_kink_free(g, cfg, vn, logp, v, old_logp, lp_idx, value_preds, returns, v_idx, ratio_spread=0.15,
                   returns_draw=(3.0, 2.0), both_clip_sides=True, huber_branches=False):
    """Old log-probs, value predictions and returns of the minibatch drawn from the float64 forward (logp at the rows
    lp_idx of old_logp, values v at the rows v_idx of value_preds and returns; written in place) so that ratios spread
    as exp(ratio_spread N(0, 1)) (10 % far above, in [2.5, 4]), value predictions 0.4 N(0, 1) off, returns
    returns_draw[0] N(0, 1) + returns_draw[1], and no row lies within KINK of a branch point of the loss: the ratio clip
    edges and the dual-clip coefficient, the value clip, the Huber threshold and the tie of the clipped and unclipped
    value losses.  vn: the ValueNorm state the update starts from.  both_clip_sides: check that ratios and value
    predictions land on both sides of their clips; huber_branches: that the value errors reach both Huber branches."""
    kinks = torch.tensor([1 - cfg.clip_param, 1 + cfg.clip_param, cfg.dual_clip_coeff], device="cuda", dtype=torch.float64)

    def draw_ratio(shape):
        near = torch.exp(ratio_spread * torch.randn(shape, generator=g, device="cuda", dtype=torch.float64))
        far = 2.5 + 1.5 * torch.rand(shape, generator=g, device="cuda", dtype=torch.float64)
        return torch.where(torch.rand(shape, generator=g, device="cuda", dtype=torch.float64) < 0.1, far, near)
    ratio = draw_ratio(logp.shape)
    for _ in range(50):
        bad = ((ratio[..., None] - kinks).abs() < KINK).any(-1)
        if not bool(bad.any()):
            break
        ratio = _redraw(bad, draw_ratio, ratio)
    old_logp[lp_idx] = (logp - ratio.log()).float()
    got = (logp - old_logp[lp_idx].double()).exp()
    assert bool(((got[..., None] - kinks).abs() >= KINK / 2).all())
    if both_clip_sides:
        assert bool((got < 1 - cfg.clip_param).any()) and bool((got > 1 + cfg.clip_param).any())

    draw_delta = lambda shape: 0.4 * torch.randn(shape, generator=g, device="cuda", dtype=torch.float64)   # noqa: E731
    delta = draw_delta(v.shape)
    for _ in range(50):
        bad = (delta.abs() - cfg.clip_param).abs() < KINK
        if not bool(bad.any()):
            break
        delta = _redraw(bad, draw_delta, delta)
    value_preds[v_idx] = (v - delta).float()
    vp = value_preds[v_idx].double()
    if both_clip_sides:
        assert bool((v - vp > cfg.clip_param).any()) and bool((v - vp < -cfg.clip_param).any())
    scale, shift = returns_draw
    draw_ret = lambda shape: scale * torch.randn(shape, generator=g, device="cuda", dtype=torch.float64) + shift   # noqa: E731
    ret = draw_ret(v.shape)
    for _ in range(100):
        r32 = ret.float().double()
        target = r32
        if cfg.use_valuenorm:
            target = rnn_ref64.vn_normalize(rnn_ref64.vn_update(vn.double(), r32, cfg.vn_beta), r32)
        clipped = vp + (v - vp).clamp(-cfg.clip_param, cfg.clip_param)
        e_o, e_c = (target - v).abs(), (target - clipped).abs()
        outside = (v - vp).abs() > cfg.clip_param
        bad = (((e_o - cfg.huber_delta).abs() < KINK) | ((e_c - cfg.huber_delta).abs() < KINK)
               | (outside & ((e_o - e_c).abs() < KINK)))
        if not bool(bad.any()):
            break
        ret = _redraw(bad, draw_ret, ret)
    assert not bool(bad.any()), "returns kept landing on a kink"
    if huber_branches and cfg.use_huber_loss and cfg.huber_delta < 2:
        assert bool((e_o > cfg.huber_delta).any()) and bool((e_o < cfg.huber_delta).any())
    returns[v_idx] = ret.float()


def ppo_synthetic(cfg, dims, head, total, rows_idx, seed, net_edit=None):
    """A buffer of `total` random rows (returns ~ 3 N(0, 1) + 2 and a ValueNorm std of 0.7: value errors with a mean, so
    that the critic gradient is large enough for the 0.5 clip to act) and nets with random weights, Adam moments mid-run, active masks with zeros and,
    for a Categorical head, action masks.  Old log-probs, value predictions and returns of the minibatch rows are drawn
    from the float64 forward so that ratios spread over ~[0.7, 1.4] (with 10 % far above) and no row lies within KINK of
    a branch point of the loss: the ratio clip edges and the dual-clip coefficient, the value clip, the Huber threshold
    and the tie of the clipped and unclipped value losses.  net_edit(head, flat) -> flat edits each random net
    ("critic" for the critic) before the log-probs and values are drawn from it."""
    from oracle import nets

    d, n, dc = dims
    gauss = head == "gaussian"
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, device="cuda")        # noqa: E731
    u = lambda *s: torch.rand(*s, generator=g, device="cuda")         # noqa: E731
    na = n if gauss else 1
    buf = dict(policy_obs=r(total, d), critic_obs=r(total, dc), advantages=r(total, 1), value_preds=r(total, 1),
               returns=3 * r(total, 1) + 2.0, active_masks=(u(total, 1) > 0.1).float(), action_log_probs=torch.zeros(total, na, device="cuda"))
    if gauss:
        buf["actions"] = r(total, n)
    else:
        am = (u(total, n) < 0.6).float()
        act = torch.randint(0, n, (total,), generator=g, device="cuda")
        am[torch.arange(total, device="cuda"), act] = 1.0
        buf["actions"], buf["action_masks"] = act.float()[:, None], am
    edit = net_edit or (lambda hd, flat: flat)
    state = dict(pol=edit(head, random_net(g, ffma_ref64.param_shapes(d, n, head))),
                 cri=edit("critic", random_net(g, ffma_ref64.param_shapes(dc, 1, "critic"))),
                 vn=torch.tensor([0.3, 0.5, 0.8], device="cuda"), steps=[3, 3])
    for k in ("pol", "cri"):
        state[k + "_m"] = 1e-3 * r(state[k].numel())
        state[k + "_v"] = 1e-6 * u(state[k].numel()) + 1e-8

    ncfg = types.SimpleNamespace(layer_N=1, activation_id=cfg.activation_id, use_recurrent_policy=False, use_policy_active_masks=True)
    pol = ffma_ref64.unflatten(state["pol"].double(), d, n, head)
    cri = ffma_ref64.unflatten(state["cri"].double(), dc, 1, "critic")
    for key, p in (("policy_obs", pol), ("critic_obs", cri)):
        redraw_off_act_kink(g, buf[key], rows_idx, lambda x: [x @ p["base.mlp.fc1.0.weight"].t() + p["base.mlp.fc1.0.bias"]])
    x = lambda k: buf[k].double()[rows_idx]   # noqa: E731
    with torch.no_grad():
        if gauss:
            logp, _ = nets.policy_eval_gaussian(pol, ncfg, x("policy_obs"), x("actions"))
        else:
            logp, _ = nets.policy_eval(pol, ncfg, x("policy_obs"), x("actions"), x("action_masks"))
        v, _ = nets.critic_forward(cri, ncfg, x("critic_obs"))
    draw_kink_free(g, cfg, state["vn"], logp, v, buf["action_log_probs"], rows_idx, buf["value_preds"], buf["returns"],
                     rows_idx, huber_branches=True)
    return buf, state


def minibatch(total, batch_rows, contiguous_from, seed):
    """(indices, rows): a shuffled index list of batch_rows of `total` rows, or (None, the contiguous range from
    contiguous_from)."""
    if contiguous_from is None:
        g = torch.Generator(device="cuda").manual_seed(seed + 1)
        idx = torch.randperm(total, device="cuda", generator=g)[:batch_rows].contiguous()
        return idx, idx
    return None, torch.arange(contiguous_from, contiguous_from + batch_rows, device="cuda")


# ---------------------------------------------------------------- kernel arguments ------------------------------------

def fill_coefs(a, cfg):
    """The loss coefficients, Adam constants and ValueNorm beta of OrlPpoArgs / OrlRnnArgs."""
    a.clip_param, a.entropy_coef, a.value_loss_coef = cfg.clip_param, cfg.entropy_coef, cfg.value_loss_coef
    a.huber_delta, a.max_grad_norm, a.dual_clip_coeff = cfg.huber_delta, cfg.max_grad_norm, cfg.dual_clip_coeff
    a.adam_beta1, a.adam_beta2, a.adam_eps, a.weight_decay = 0.9, 0.999, cfg.opti_eps, cfg.weight_decay
    a.vn_beta, a.norm_rows = cfg.vn_beta, 0


def ppo_args(cfg, dims, head_kind, flags, G, buf, batch_rows, total, indices, row_begin, stats, dev, steps, lrs, train_info,
             partials, folded, grads):
    """OrlPpoArgs of one update on a synthetic buffer of (rows, width) arrays (action_masks optional).
    dims: (d, n, dc); stats: (GAE moments, minibatch moments); dev: the device's pol, cri, pol_m, pol_v, cri_m, cri_v
    and vn (a shared model passes its one net as both)."""
    lb, _ = lib()
    d, n, dc = dims
    a = lb.OrlPpoArgs()
    a.obs_dim, a.critic_obs_dim, a.n_actions, a.activation_id = d, dc, n, cfg.activation_id
    a.flags, a.grid_per_net, a.head_kind = flags, G, head_kind
    a.batch_rows, a.row_begin, a.total_rows = batch_rows, row_begin, total
    a.indices = None if indices is None else lb.ptr(indices)
    for k, key in (("policy_obs", "policy_obs"), ("critic_obs", "critic_obs"), ("actions", "actions"),
                   ("old_log_probs", "action_log_probs"), ("advantages", "advantages"), ("value_preds", "value_preds"),
                   ("returns", "returns"), ("active_masks", "active_masks")):
        setattr(a, k, lb.ptr(buf[key]))
    a.action_masks = lb.ptr(buf["action_masks"]) if "action_masks" in buf else None
    a.gae_stats, a.mb_stats, a.vn_state = lb.ptr(stats[0]), lb.ptr(stats[1]), lb.ptr(dev["vn"])
    a.policy_params, a.critic_params = lb.ptr(dev["pol"]), lb.ptr(dev["cri"])
    a.policy_adam_m, a.policy_adam_v = lb.ptr(dev["pol_m"]), lb.ptr(dev["pol_v"])
    a.critic_adam_m, a.critic_adam_v = lb.ptr(dev["cri_m"]), lb.ptr(dev["cri_v"])
    a.adam_steps, a.lrs, a.train_info = lb.ptr(steps), lb.ptr(lrs), lb.ptr(train_info)
    fill_coefs(a, cfg)
    a.partials, a.folded, a.grads = lb.ptr(partials), lb.ptr(folded), lb.ptr(grads)
    return a


def moment_scale(cfg, grad, norm, p, m):
    """Per element, the magnitude of the terms an Adam step combines into exp_avg: beta1 |m| + (1 - beta1) |g|, g the
    clipped gradient plus weight decay.  exp_avg mixes terms of both signs, so its error is measured against them, as a
    loss sum's is against its absolute terms (exp_avg_sq adds positive terms: its own norm is their magnitude).
    grad: the float64 gradient of one net, norm its clip norm; p, m: the net's parameters and exp_avg before the step."""
    g = grad.abs()
    if cfg.use_max_grad_norm:
        g = g * min(1.0, cfg.max_grad_norm / (float(norm) + 1e-6))
    p, m = (x.to(g.device, torch.float64).abs() for x in (p, m))
    return 0.9 * m + 0.1 * (g + cfg.weight_decay * p)


# ---------------------------------------------------------------- a live two-net trainer ------------------------------
# c: a namespace with the trainer tr, its algo module m, the buffer b and `live`, the device tensors pol, cri, pol_m,
# pol_v, cri_m, cri_v and vn

def snapshot(c):
    return {k: v.clone() for k, v in c.live.items()}, c.m.adam_steps.clone()


def restore(c, snap):
    saved, steps = snap
    for k, v in c.live.items():
        v.copy_(saved[k])
    c.m.adam_steps.copy_(steps)
    c.tr.train_info.zero_()


def state(c):
    return dict({k: v.clone() for k, v in c.live.items()}, steps=[int(x) for x in c.m.adam_steps])


def kernel_update(c, idx, stats, rows):
    """One PPOAlgorithm.ppo_update as train_async issues it; what the comparison reads back."""
    tr = c.tr
    tr.train_info.zero_()
    tr.sync_lrs()
    tr.ppo_update(c.b, rows, idx, 0, mb_stats=stats)
    torch.cuda.synchronize()
    np_, nc = int(c.live["pol"].numel()), int(c.live["cri"].numel())
    return dict(grad_pol=tr.grads[0, :np_].clone(), grad_cri=tr.grads[1, :nc].clone(), losses=loss_sums(tr.folded, tr.stride),
                info=tr.train_info.clone(), steps=[int(x) for x in c.m.adam_steps], **{k: v.clone() for k, v in c.live.items()})


# ---------------------------------------------------------------- the recurrent update --------------------------------

def c3_buf(b):
    """The device buffer arrays rnn_ref64.update reads."""
    return {k: getattr(b, k) for k in ("policy_obs", "critic_obs", "rnn_states", "rnn_states_critic", "masks", "active_masks",
                                       "actions", "action_log_probs", "value_preds", "returns", "advantages")}


def drive(a, grads, loss_acc, outs):
    """orl_rnn_fwdbwd (gradients, loss sums), then orl_rnn_apply; `outs` names the device tensors read back after."""
    lb, L = lib()
    s = lb.current_stream()
    lb.check(L.orl_rnn_fwdbwd(a, s), "orl_rnn_fwdbwd")
    g, la = grads.clone(), loss_acc[:4].clone()
    lb.check(L.orl_rnn_apply(a, s), "orl_rnn_apply")
    torch.cuda.synchronize()
    return g, la, {k: v.clone() for k, v in outs.items()}


def rnn_compare(case, dims, k, r64, r32, check_vn):
    """Every quantity of one recurrent update against the bar at RNN_FLOOR: gradients per block, loss sums, parameters,
    Adam moments, ValueNorm state and step counts."""
    d, n, dc = dims
    chk = Checker(case, RNN_FLOOR)
    for net, dd, nn, critic in (("pol", d, n, False), ("cri", dc, 1, True)):
        for name, s in rnn_ref64.blocks(dd, nn, critic).items():
            chk(f"grad {net}.{name}", k["grad_" + net][s], r64["grad_" + net][s], r32["grad_" + net][s])
    for i, name in enumerate(("policy loss", "entropy", "ratio sum", "value loss")):
        chk(f"loss_acc[{i}] {name}", k["losses"][i:i + 1], r64["losses"][i:i + 1], r32["losses"][i:i + 1],
            scale=r64["loss_scales"][i])
    for net, dd, nn, critic in (("pol", d, n, False), ("cri", dc, 1, True)):
        for key in ("", "_m", "_v"):
            for name, s in rnn_ref64.blocks(dd, nn, critic).items():
                chk(f"{net}{key or '_param'} {name}", k[net + key][s], r64[net + key][s], r32[net + key][s])
    if check_vn:
        chk("vn_state", k["vn"], r64["vn"], r32["vn"])
    assert k["steps"] == [r64["pol_step"], r64["cri_step"]]
    chk.done()
