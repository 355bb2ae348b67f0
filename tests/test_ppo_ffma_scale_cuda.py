"""The FFMA PPO update (`ppo_fwdbwd_kernel` + `orl_ppo_reduce` + `orl_ppo_apply`, orl_ppo.cu) at C5 scale against a
float64 reference: DiagGaussian heads, observations wider than 8, every loss option.

The FFMA kernel takes every update the tensor-core kernel does not: DiagGaussian heads, observation widths above 8 and the
MPE-shaped feed-forward MAPPO.  C5 (obs 17, Box(6), 1024 host-stepped envs, T = 128, 4 epochs x 1 minibatch) runs on it
alone.  Here it runs (a) on a real C5 buffer, where every CTA walks 15-16 tiles on the contiguous whole-buffer path and on
a shuffled quarter of it; (b) on synthetic buffers at the edges of its thread mappings: head widths 1 .. 8 (one and two
head row-blocks), observation widths whose weight-gradient mapping leaves threads idle (d = 9, 17, 33), one partial tile,
exactly one tile per CTA, many tiles with a partial last one, a contiguous range that does not start at row 0, and a
masked Categorical head at the MPE shape; (c) under every loss option of tests/test_ppo_flags_cuda.py with a Gaussian
head; (d) against deliberately wrong references, to show that the bars catch a subtle kernel error.

The reference is tests/ffma_ref64.py over the oracle (oracle/ppo.py `ppo_update`).  Bars are those of
tests/test_rnn_scale_cuda.py with a higher FLOOR (see below): per parameter block, the kernel's relative L2 error against
float64 may be at most RATIO x the float32 reference's error against float64, clamped to [FLOOR, CEIL]; loss sums are
relative to the weighted sum of their absolute terms and Adam's exp_avg to the terms it combines.  Every case prints its
kernel / float32 error ratios (`pytest -s`)."""
import types

import numpy as np
import pytest
import torch

import ffma_ref64 as ref
import rnn_ref64
from test_ppo_flags_cuda import CASES
from test_rnn_scale_cuda import ATOL, KINK, Checker, _mb_stats, _rel, no_tf32  # noqa: F401  (no_tf32: pytest fixture)

pytestmark = pytest.mark.gpu

P_M = 128   # rows per tile of the FFMA update kernel
# The floor of the bar, 2.5x that of test_rnn_scale_cuda.py (2e-6), measured on an H100 SXM (132 SMs, 66 CTAs per net):
# a kernel thread adds its rows' weight-gradient terms in one fixed-order float32 chain (512 terms per thread for the
# 64 x 54 critic fc1 gradient at 4 tiles per CTA, MG = 1) and a single-element block has no other elements to average
# over (the n = 1 head bias, 25k rows with cancellation); those reached 2.5e-6 and 3.2e-6 against float64, where torch's
# pairwise float32 sums are 3e-7 off.  Every mutant below moves its block by 1e-2 or more.
FLOOR = 5e-6
ACT_KINK = 1e-4   # synthetic fc1 pre-activations keep at least this distance from 0
C5_FLAGS = ["--seed", "0", "--episode_length", "128", "--ppo_epoch", "4", "--num_mini_batch", "1", "--log_interval", "1",
            "--host_env_groups", "false"]


def _lib():
    from openrl_b200 import lib
    return lib, lib.load()


def _grid():
    """CTAs per net of the FFMA update: half the SMs (PPOAlgorithm.grid_per_net)."""
    return max(1, torch.cuda.get_device_properties(0).multi_processor_count // 2)


def _moment_scales(r64, state, cfg):
    """Per element, the magnitude of the terms an Adam step combines into exp_avg: beta1 |m| + (1 - beta1) |g|, g the
    clipped gradient plus weight decay.  exp_avg mixes terms of both signs, so its error is measured against them, as a
    loss sum's is against its absolute terms (exp_avg_sq adds positive terms: its own norm is their magnitude)."""
    out = {}
    for j, net in enumerate(("pol", "cri")):
        g = r64["grad_" + net].abs()
        if cfg.use_max_grad_norm:
            g = g * min(1.0, cfg.max_grad_norm / (float(r64["norms"][j]) + 1e-6))
        p, m = (state[net + key].to(g.device, torch.float64).abs() for key in ("", "_m"))
        out[net] = 0.9 * m + 0.1 * (g + cfg.weight_decay * p)
    return out


def _compare(case, dims, head, k, r64, r32, state, cfg, check_vn=True):
    d, n, dc = dims
    chk = Checker(case, floor=FLOOR)
    nets = (("pol", d, n, head), ("cri", dc, 1, "critic"))
    for net, dd, nn, hd in nets:
        for name, s in ref.blocks(dd, nn, hd).items():
            chk(f"grad {net}.{name}", k["grad_" + net][s], r64["grad_" + net][s], r32["grad_" + net][s])
    for i, name in enumerate(("policy loss", "entropy", "ratio sum", "value loss")):
        chk(f"loss sum {name}", k["losses"][i:i + 1], r64["losses"][i:i + 1], r32["losses"][i:i + 1], scale=r64["loss_scales"][i])
    for col, name, j in ((4, "actor grad norm", 0), (1, "critic grad norm", 1), (5, "ratio mean", None)):
        pick = lambda r: (r["ratio_mean"] if j is None else r["norms"][j]).reshape(1)   # noqa: E731
        chk(f"train_info {name}", k["info"][col:col + 1], pick(r64), pick(r32))
    mscale = _moment_scales(r64, state, cfg)
    for net, dd, nn, hd in nets:
        for key in ("", "_m", "_v"):
            for name, s in ref.blocks(dd, nn, hd).items():
                chk(f"{net}{key or '_param'} {name}", k[net + key][s], r64[net + key][s], r32[net + key][s],
                    scale=mscale[net][s].norm() if key == "_m" else None)
    if check_vn:
        chk("vn_state", k["vn"], r64["vn"], r32["vn"])
    assert k["steps"] == [r64["pol_step"], r64["cri_step"]]
    chk.done()


def _loss_sums(folded, stride):
    return torch.stack([folded[0, stride - 8], folded[0, stride - 7], folded[0, stride - 6], folded[1, stride - 8]]).clone()


# ---------------------------------------------------------------- the real C5 buffer ----------------------------------

@pytest.fixture(scope="module")
def c5():
    """One rollout of C5 (the HalfCheetah-shaped synthetic host env of test_gaussian_cuda) and its returns."""
    from openrl_b200 import lib
    from openrl_b200.envs.vec_env import HostVecEnv
    from test_gaussian_cuda import _SyntheticHost
    from test_rnn_host_cuda import _agent

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.manual_seed(0)
    cfg, net, agent = _agent(HostVecEnv(_SyntheticHost(1024)), C5_FLAGS)
    drv = agent.driver
    drv.actor_rollout()
    drv.compute_returns()
    torch.cuda.synchronize()
    tr, b = drv.trainer, drv.buffer.data
    T, N = b.episode_length, b.n_rollout_threads
    rows = T * N * b.num_agents
    assert (T, N, b.num_agents, tr.d, tr.n, tr.dc) == (128, 1024, 1, 17, 6, 17)
    assert not tr.use_tensor_cores and tr.head_kind == lib.HEAD_GAUSSIAN and not tr.share
    assert tr.grid_per_net == _grid()
    tiles = rows // P_M
    assert rows % P_M == 0 and tiles // tr.grid_per_net >= 8   # H100 SXM: 1024 tiles over 66 CTAs, 15-16 per CTA
    print(f"\n  C5: {rows} rows, {tiles} tiles, {tr.grid_per_net} CTAs per net, "
          f"{tiles // tr.grid_per_net}-{-(-tiles // tr.grid_per_net)} tiles per CTA")
    m = tr.algo_module
    pol, cri = m.models["policy"], m.models["critic"]
    op, oc = m.optimizers["policy"], m.optimizers["critic"]
    live = dict(pol=pol.flat_params, cri=cri.flat_params, pol_m=op.exp_avg, pol_v=op.exp_avg_sq, cri_m=oc.exp_avg,
                cri_v=oc.exp_avg_sq, vn=cri.value_normalizer.state)
    buf = dict(policy_obs=b.policy_obs.reshape(-1, 17), critic_obs=b.critic_obs.reshape(-1, 17), actions=b.actions.reshape(-1, 6),
               action_log_probs=b.action_log_probs.reshape(-1, 6), advantages=b.advantages.reshape(-1, 1)[:rows],
               value_preds=b.value_preds.reshape(-1, 1), returns=b.returns.reshape(-1, 1), active_masks=b.active_masks.reshape(-1, 1))
    yield types.SimpleNamespace(cfg=cfg, net=net, agent=agent, drv=drv, tr=tr, b=b, rows=rows, m=m, live=live, buf=buf,
                                vn_beta=cri.value_normalizer.beta)
    torch.cuda.empty_cache()


def _snapshot(c):
    return {k: v.clone() for k, v in c.live.items()}, c.m.adam_steps.clone()


def _restore(c, snap):
    saved, steps = snap
    for k, v in c.live.items():
        v.copy_(saved[k])
    c.m.adam_steps.copy_(steps)
    c.tr.train_info.zero_()


def _state(c):
    return dict({k: v.clone() for k, v in c.live.items()}, steps=[int(x) for x in c.m.adam_steps])


def _kernel_update(c, idx, stats, rows):
    """One PPOAlgorithm.ppo_update as train_async issues it; what the comparison reads back."""
    tr = c.tr
    tr.train_info.zero_()
    tr.sync_lrs()
    tr.ppo_update(c.b, rows, idx, 0, mb_stats=stats)
    torch.cuda.synchronize()
    np_, nc = int(c.live["pol"].numel()), int(c.live["cri"].numel())
    return dict(grad_pol=tr.grads[0, :np_].clone(), grad_cri=tr.grads[1, :nc].clone(), losses=_loss_sums(tr.folded, tr.stride),
                info=tr.train_info.clone(), steps=[int(x) for x in c.m.adam_steps], **{k: v.clone() for k, v in c.live.items()})


def _refs(c, state, rows_idx, **kw):
    rcfg = types.SimpleNamespace(**{**vars(c.cfg), **kw.pop("cfg", {})})
    return [ref.update(rcfg, c.buf, state, rows_idx, (17, 6, 17), "gaussian", dt, vn_beta=c.vn_beta, **kw)
            for dt in (torch.float64, torch.float32)]


def test_c5_value_preds_and_log_probs(c5):
    """The FFMA critic pass over all T + 1 slots (value_preds) and the rollout's Gaussian log-probs of the stored actions
    against a float64 forward of the oracle nets, element-wise."""
    from oracle import nets

    ncfg = types.SimpleNamespace(layer_N=1, activation_id=c5.cfg.activation_id, use_recurrent_policy=False)
    pol = ref.unflatten(c5.live["pol"].double(), 17, 6, "gaussian")
    cri = ref.unflatten(c5.live["cri"].double(), 17, 1, "critic")
    with torch.no_grad():
        v, _ = nets.critic_forward(cri, ncfg, c5.buf["critic_obs"].double())
        feat, _ = nets.policy_features(pol, ncfg, c5.buf["policy_obs"].double()[:c5.rows])
        mean, std = nets.gaussian_params(pol, feat)
        lp = torch.distributions.Normal(mean, std).log_prob(c5.buf["actions"].double())
    np.testing.assert_allclose(c5.buf["value_preds"].cpu().numpy(), v.cpu().numpy(), rtol=0, atol=ATOL)
    np.testing.assert_allclose(c5.buf["action_log_probs"].cpu().numpy(), lp.cpu().numpy(), rtol=0, atol=ATOL)
    assert c5.buf["value_preds"].shape[0] == c5.rows + 1024 and float(v.abs().max()) > 0


def test_c5_four_epochs_contiguous(c5, no_tf32):
    """C5's four updates (4 epochs over the whole buffer, indices == NULL, the GAE moments as minibatch moments), each
    teacher-forced: the reference starts from the device's own state before that update.  Epoch 1 has every ratio at 1;
    epochs 2-4 move them away from 1."""
    snap = _snapshot(c5)
    rows = torch.arange(c5.rows, device="cuda")
    try:
        for epoch in range(4):
            state = _state(c5)
            k = _kernel_update(c5, None, c5.b.gae_stats[5:8], c5.rows)
            r64, r32 = _refs(c5, state, rows)
            _compare(f"c5-epoch{epoch + 1}-contiguous-{c5.rows}rows", (17, 6, 17), "gaussian", k, r64, r32, state, c5.cfg)
            spread = float(r64["ratio_spread"])
            assert (spread > 1e-4) if epoch else (spread < 1e-4), spread   # epoch 1: every ratio 1 up to rounding
    finally:
        _restore(c5, snap)


def test_c5_shuffled_quarter(c5, no_tf32):
    """num_mini_batch 4 on the same buffer: a shuffled index list of a quarter of the rows, orl_minibatch_stats."""
    snap = _snapshot(c5)
    g = torch.Generator(device="cuda").manual_seed(4)
    idx = torch.randperm(c5.rows, device="cuda", generator=g)[:c5.rows // 4].contiguous()
    assert idx.numel() == 32768
    try:
        state = _state(c5)
        k = _kernel_update(c5, idx, _mb_stats(idx, c5.b.returns, c5.b.active_masks), idx.numel())
        r64, r32 = _refs(c5, state, idx)
        _compare("c5-mb4-shuffled-32768rows", (17, 6, 17), "gaussian", k, r64, r32, state, c5.cfg)
    finally:
        _restore(c5, snap)


# ---------------------------------------------------------------- deliberate mistakes ---------------------------------

@pytest.mark.parametrize("mutant", list(ref.MUTANTS))
def test_c5_mutants_are_detected(c5, no_tf32, mutant):
    """The real kernel output on the C5 buffer against a float64 reference with one deliberate mistake: the block the
    mistake lands in must violate its bar (and pass it against the correct reference)."""
    from openrl_b200 import lib

    _, what, opts, moved = ref.MUTANTS[mutant]
    snap, flags = _snapshot(c5), c5.tr.flags
    rows = torch.arange(c5.rows, device="cuda")
    try:
        if moved:      # start from the state after one update: ratios away from 1
            _kernel_update(c5, None, c5.b.gae_stats[5:8], c5.rows)
        if opts.get("use_policy_active_masks") is False:
            c5.tr.flags &= ~lib.PPO_POLICY_ACTIVE_MASKS
        state = _state(c5)
        k = _kernel_update(c5, None, c5.b.gae_stats[5:8], c5.rows)
    finally:
        c5.tr.flags = flags
        _restore(c5, snap)
    G, tiles = c5.tr.grid_per_net, c5.rows // P_M
    last = (tiles - 1) // G * G           # CTA 0's last tile
    dropped = torch.arange(last * P_M, last * P_M + P_M, device="cuda")
    r64, r32 = _refs(c5, state, rows, cfg=opts)
    bad, _ = _refs(c5, state, rows, cfg=opts, mutant=mutant, dropped_rows=dropped)
    net, name = what.split(" ")[1].split(".", 1)
    s = ref.blocks(17, 6 if net == "pol" else 1, "gaussian" if net == "pol" else "critic")[name]
    got, want, wrong, r32s = k["grad_" + net][s], r64["grad_" + net][s], bad["grad_" + net][s], r32["grad_" + net][s]
    good = Checker(f"c5-{mutant}", floor=FLOOR)
    good(what, got, want, r32s)
    good.done()
    e_bad, bar = _rel(got, wrong), good.bar(_rel(r32s, want))
    print(f"  c5-{mutant}: kernel against the mutant {e_bad:.2e}, bar {bar:.2e}")
    assert e_bad > bar, f"{mutant}: the mistake ({ref.MUTANTS[mutant][0]}) passed the bar of {what}"


# ---------------------------------------------------------------- synthetic buffers -----------------------------------

BASE = dict(use_huber_loss=True, use_clipped_value_loss=True, use_value_active_masks=True, use_policy_active_masks=True,
            use_valuenorm=True, use_adv_normalize=False, use_max_grad_norm=True, dual_clip_ppo=False, a2c=False, activation_id=1,
            clip_param=0.2, entropy_coef=0.01, value_loss_coef=0.5, huber_delta=1.0, max_grad_norm=1e3, dual_clip_coeff=3.0,
            lr=7e-4, critic_lr=5e-4, opti_eps=1e-5, weight_decay=0.0)


def _flags(c):
    lib, _ = _lib()
    return ((lib.PPO_HUBER if c.use_huber_loss else 0) | (lib.PPO_CLIP_VALUE if c.use_clipped_value_loss else 0)
            | (lib.PPO_VALUE_ACTIVE_MASKS if c.use_value_active_masks else 0)
            | (lib.PPO_POLICY_ACTIVE_MASKS if c.use_policy_active_masks else 0) | (lib.PPO_VALUENORM if c.use_valuenorm else 0)
            | (lib.PPO_ADV_NORMALIZE if c.use_adv_normalize else 0) | (lib.PPO_MAX_GRAD_NORM if c.use_max_grad_norm else 0)
            | (lib.PPO_DUAL_CLIP if c.dual_clip_ppo else 0) | (lib.PPO_A2C if c.a2c else 0))


def _random_net(g, d, n, head):
    parts = []
    for name, shp in ref.param_shapes(d, n, head):
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


def _synthetic(cfg, dims, head, total, rows_idx, seed):
    """A buffer of `total` random rows (returns ~ 3 N(0, 1) + 2 and a ValueNorm std of 0.7: value errors with a mean, so
    that the critic gradient is large enough for the 0.5 clip to act) and nets with random weights, Adam moments mid-run, active masks with zeros and,
    for a Categorical head, action masks.  Old log-probs, value predictions and returns of the minibatch rows are drawn
    from the float64 forward so that ratios spread over ~[0.7, 1.4] (with 10 % far above) and no row lies within KINK of
    a branch point of the loss: the ratio clip edges and the dual-clip coefficient, the value clip, the Huber threshold
    and the tie of the clipped and unclipped value losses."""
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
    state = dict(pol=_random_net(g, d, n, head), cri=_random_net(g, dc, 1, "critic"), vn=torch.tensor([0.3, 0.5, 0.8], device="cuda"),
                 steps=[3, 3])
    for k in ("pol", "cri"):
        state[k + "_m"] = 1e-3 * r(state[k].numel())
        state[k + "_v"] = 1e-6 * u(state[k].numel()) + 1e-8

    ncfg = types.SimpleNamespace(layer_N=1, activation_id=cfg.activation_id, use_recurrent_policy=False, use_policy_active_masks=True)
    pol = ref.unflatten(state["pol"].double(), d, n, head)
    cri = ref.unflatten(state["cri"].double(), dc, 1, "critic")
    # ReLU / LeakyReLU: no fc1 pre-activation of a minibatch row within ACT_KINK of 0, where float32 rounding could
    # take the other branch of the activation's derivative
    for key, p in (("policy_obs", pol), ("critic_obs", cri)):
        for _ in range(50):
            x = buf[key][rows_idx].double()
            z = x @ p["base.mlp.fc1.0.weight"].t() + p["base.mlp.fc1.0.bias"]
            bad = (z.abs() < ACT_KINK).any(-1)
            if not bool(bad.any()):
                break
            buf[key][rows_idx[bad]] = r(int(bad.sum()), x.shape[1])
        assert not bool(bad.any()), "observations kept landing on an activation kink"
    x = lambda k: buf[k].double()[rows_idx]   # noqa: E731
    with torch.no_grad():
        if gauss:
            logp, _ = nets.policy_eval_gaussian(pol, ncfg, x("policy_obs"), x("actions"))
        else:
            logp, _ = nets.policy_eval(pol, ncfg, x("policy_obs"), x("actions"), x("action_masks"))
        v, _ = nets.critic_forward(cri, ncfg, x("critic_obs"))
    kinks = torch.tensor([1 - cfg.clip_param, 1 + cfg.clip_param, cfg.dual_clip_coeff], device="cuda", dtype=torch.float64)

    def draw_ratio(shape):
        near = torch.exp(0.15 * torch.randn(shape, generator=g, device="cuda", dtype=torch.float64))
        far = 2.5 + 1.5 * torch.rand(shape, generator=g, device="cuda", dtype=torch.float64)
        return torch.where(torch.rand(shape, generator=g, device="cuda", dtype=torch.float64) < 0.1, far, near)
    ratio = draw_ratio(logp.shape)
    for _ in range(50):
        bad = ((ratio[..., None] - kinks).abs() < KINK).any(-1)
        if not bool(bad.any()):
            break
        ratio = _redraw(bad, draw_ratio, ratio)
    buf["action_log_probs"][rows_idx] = (logp - ratio.log()).float()
    lp32 = buf["action_log_probs"][rows_idx].double()
    got = (logp - lp32).exp()
    assert bool(((got[..., None] - kinks).abs() >= KINK / 2).all())
    assert bool((got < 1 - cfg.clip_param).any()) and bool((got > 1 + cfg.clip_param).any())   # both clip sides

    draw_delta = lambda shape: 0.4 * torch.randn(shape, generator=g, device="cuda", dtype=torch.float64)   # noqa: E731
    delta = draw_delta(v.shape)
    for _ in range(50):
        bad = (delta.abs() - cfg.clip_param).abs() < KINK
        if not bool(bad.any()):
            break
        delta = _redraw(bad, draw_delta, delta)
    buf["value_preds"][rows_idx] = (v - delta).float()
    vp = buf["value_preds"][rows_idx].double()
    assert bool((v - vp > cfg.clip_param).any()) and bool((v - vp < -cfg.clip_param).any())   # value clip on both sides
    draw_ret = lambda shape: 3 * torch.randn(shape, generator=g, device="cuda", dtype=torch.float64) + 2.0   # noqa: E731
    ret = draw_ret(v.shape)
    for _ in range(100):
        r32 = ret.float().double()
        target = r32
        if cfg.use_valuenorm:
            target = rnn_ref64.vn_normalize(rnn_ref64.vn_update(state["vn"].double(), r32, cfg.vn_beta), r32)
        clipped = vp + (v - vp).clamp(-cfg.clip_param, cfg.clip_param)
        e_o, e_c = (target - v).abs(), (target - clipped).abs()
        outside = (v - vp).abs() > cfg.clip_param
        bad = (((e_o - cfg.huber_delta).abs() < KINK) | ((e_c - cfg.huber_delta).abs() < KINK)
               | (outside & ((e_o - e_c).abs() < KINK)))
        if not bool(bad.any()):
            break
        ret = _redraw(bad, draw_ret, ret)
    assert not bool(bad.any()), "returns kept landing on a kink"
    if cfg.use_huber_loss and cfg.huber_delta < 2:
        assert bool((e_o > cfg.huber_delta).any()) and bool((e_o < cfg.huber_delta).any())   # both Huber branches
    buf["returns"][rows_idx] = ret.float()
    return buf, state


def _gae_stats(buf):
    adv = buf["advantages"].double()[:, 0]
    act = buf["active_masks"].double()[:adv.numel(), 0] != 0
    ret = buf["returns"].double()[:adv.numel(), 0]
    return torch.stack([adv.sum(), (adv * adv).sum(), torch.tensor(float(adv.numel()), device="cuda", dtype=torch.float64),
                        adv[act].sum(), (adv[act] ** 2).sum(), ret.sum(), (ret * ret).sum(), act.double().sum()])


def _run_synthetic(case, cfg, dims, head, batch_rows, contiguous_from=None, total=None, seed=0):
    """OrlPpoArgs built by hand for a synthetic buffer; the kernel against both reference runs."""
    lib, L = _lib()
    d, n, dc = dims
    G = _grid()
    total = total or batch_rows + 301
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    if contiguous_from is None:
        idx = torch.randperm(total, device="cuda", generator=g)[:batch_rows].contiguous()
        rows_idx = idx
    else:
        idx = None
        rows_idx = torch.arange(contiguous_from, contiguous_from + batch_rows, device="cuda")
    buf, state = _synthetic(cfg, dims, head, total, rows_idx, seed)
    gauss = head == "gaussian"
    stride, gstride = L.orl_ppo_stride(d, dc, n), L.orl_ppo_grads_stride(d, dc, n)
    partials = torch.zeros(2 * G, stride, device="cuda")
    folded = torch.zeros(2, stride, device="cuda")
    grads = torch.zeros(2, gstride, device="cuda")
    dev = {k: state[k].clone() for k in ("pol", "cri", "pol_m", "pol_v", "cri_m", "cri_v", "vn")}
    assert dev["pol"].numel() == L.orl_net_param_count(d, n) + (n if gauss else 0)
    steps = torch.tensor(state["steps"], dtype=torch.int32, device="cuda")
    lrs = torch.tensor([cfg.lr, cfg.critic_lr], dtype=torch.float32, device="cuda")
    gae_stats = _gae_stats(buf)
    mb_stats = _mb_stats(rows_idx.contiguous(), buf["returns"], buf["active_masks"])
    train_info = torch.zeros(6, device="cuda")
    a = lib.OrlPpoArgs()
    a.obs_dim, a.critic_obs_dim, a.n_actions, a.activation_id = d, dc, n, cfg.activation_id
    a.flags, a.grid_per_net, a.head_kind = _flags(cfg), G, lib.HEAD_GAUSSIAN if gauss else lib.HEAD_CATEGORICAL
    a.batch_rows, a.row_begin, a.total_rows = batch_rows, contiguous_from or 0, total
    a.indices = None if idx is None else lib.ptr(idx)
    for k, key in (("policy_obs", "policy_obs"), ("critic_obs", "critic_obs"), ("actions", "actions"),
                   ("old_log_probs", "action_log_probs"), ("advantages", "advantages"), ("value_preds", "value_preds"),
                   ("returns", "returns"), ("active_masks", "active_masks")):
        setattr(a, k, lib.ptr(buf[key]))
    a.action_masks = None if gauss else lib.ptr(buf["action_masks"])
    a.gae_stats, a.mb_stats, a.vn_state = lib.ptr(gae_stats), lib.ptr(mb_stats), lib.ptr(dev["vn"])
    a.policy_params, a.critic_params = lib.ptr(dev["pol"]), lib.ptr(dev["cri"])
    a.policy_adam_m, a.policy_adam_v = lib.ptr(dev["pol_m"]), lib.ptr(dev["pol_v"])
    a.critic_adam_m, a.critic_adam_v = lib.ptr(dev["cri_m"]), lib.ptr(dev["cri_v"])
    a.adam_steps, a.lrs, a.train_info = lib.ptr(steps), lib.ptr(lrs), lib.ptr(train_info)
    a.clip_param, a.entropy_coef, a.value_loss_coef = cfg.clip_param, cfg.entropy_coef, cfg.value_loss_coef
    a.huber_delta, a.max_grad_norm, a.dual_clip_coeff = cfg.huber_delta, cfg.max_grad_norm, cfg.dual_clip_coeff
    a.adam_beta1, a.adam_beta2, a.adam_eps, a.weight_decay = 0.9, 0.999, cfg.opti_eps, cfg.weight_decay
    a.vn_beta, a.norm_rows = cfg.vn_beta, 0
    a.partials, a.folded, a.grads = lib.ptr(partials), lib.ptr(folded), lib.ptr(grads)
    s = lib.current_stream()
    lib.check(L.orl_ppo_fwdbwd(a, s), "orl_ppo_fwdbwd")
    lib.check(L.orl_ppo_reduce(a, s), "orl_ppo_reduce")
    lib.check(L.orl_ppo_apply(a, s), "orl_ppo_apply")
    torch.cuda.synchronize()
    k = dict(grad_pol=grads[0, :dev["pol"].numel()], grad_cri=grads[1, :dev["cri"].numel()], losses=_loss_sums(folded, stride),
             info=train_info, steps=[int(x) for x in steps], **dev)
    r64, r32 = (ref.update(cfg, buf, state, rows_idx, dims, head, dt, vn_beta=cfg.vn_beta) for dt in (torch.float64, torch.float32))
    if cfg.use_max_grad_norm and cfg.max_grad_norm < 1:   # the clip case: the clip must really act on both nets
        assert float(r64["norms"][0]) > cfg.max_grad_norm and float(r64["norms"][1]) > cfg.max_grad_norm
    tiles = -(-batch_rows // P_M)
    print(f"\n  {case}: {batch_rows} rows, {tiles} tiles, {G} CTAs per net, up to {-(-tiles // G)} tiles per CTA")
    _compare(case, dims, head, k, r64, r32, state, cfg, check_vn=cfg.use_valuenorm)
    torch.cuda.empty_cache()


def _rows(kind):
    G = _grid()
    return {"37rows(1 partial tile)": 37, "Gx128rows(1 tile per CTA)": G * P_M,
            "3Gx128+37rows(4 tiles per CTA, partial last)": 3 * G * P_M + 37}[kind]


DIMS = [("gauss-d9-n1-dc9(MG5)", (9, 1, 9), "gaussian"), ("gauss-d17-n6-dc17(MG3,JBH2)", (17, 6, 17), "gaussian"),
        ("gauss-d33-n4-dc24(MG1,MG2,JBH1)", (33, 4, 24), "gaussian"), ("gauss-d17-n5-dc64(JBH2)", (17, 5, 64), "gaussian"),
        ("gauss-d64-n8-dc64(MG1)", (64, 8, 64), "gaussian"), ("cat-mpe-d18-n5-dc54-masked", (18, 5, 54), "categorical")]
ROWS = ["37rows(1 partial tile)", "Gx128rows(1 tile per CTA)", "3Gx128+37rows(4 tiles per CTA, partial last)"]
SHAPES = [(f"{name}-{rk}", dims, head, rk) for name, dims, head in DIMS for rk in ROWS]


@pytest.mark.parametrize("case,dims,head,rows_kind", SHAPES, ids=[s[0] for s in SHAPES])
def test_update_synthetic_edges(no_tf32, case, dims, head, rows_kind):
    """Shuffled minibatches (an index list into a larger buffer) at every width / head-row-block edge and row count."""
    cfg = types.SimpleNamespace(**BASE, vn_beta=0.99999)
    _run_synthetic(case, cfg, dims, head, _rows(rows_kind), seed=len(case) * 7 + dims[0])


@pytest.mark.parametrize("dims,head", [((17, 6, 17), "gaussian"), ((18, 5, 54), "categorical")], ids=["gauss-d17-n6", "cat-mpe"])
def test_update_contiguous_range_not_at_row_zero(no_tf32, dims, head):
    """The contiguous gather (indices == NULL) of a range that starts at row 1000 of a larger buffer, many tiles per
    CTA, partial last tile."""
    G = _grid()
    rows = 2 * G * P_M + 77
    cfg = types.SimpleNamespace(**BASE, vn_beta=0.99999)
    _run_synthetic(f"contiguous-from-1000-{head}-{rows}rows", cfg, dims, head, rows, contiguous_from=1000, total=rows + 1500,
                   seed=dims[0])


def _flag_cfg(flags):
    from openrl_b200.configs.config import create_config_parser

    a2c = "A2C" in flags
    cfg = create_config_parser().parse_args(["--seed", "3"] + [f for f in flags if f != "A2C"])
    return types.SimpleNamespace(**{**vars(cfg), "a2c": a2c, "vn_beta": 0.99999})


@pytest.mark.parametrize("flags", CASES, ids=[" ".join(c) or "default" for c in CASES])
def test_update_flag_sweep_gaussian(no_tf32, flags):
    """Every option of tests/test_ppo_flags_cuda.py on a Gaussian (17, 6) buffer, 3 G tiles + 37 rows (4 tiles per
    CTA), through the FFMA kernel: policy active masks on (default) and off, Huber off, value clip off, ValueNorm off,
    dual clip, A2C, weight decay, the activations, other coefficients and a gradient clip that acts on both nets."""
    cfg = _flag_cfg(flags)
    _run_synthetic("flags-" + ("-".join(flags) or "default"), cfg, (17, 6, 17), "gaussian", 3 * _grid() * P_M + 37, seed=77)
