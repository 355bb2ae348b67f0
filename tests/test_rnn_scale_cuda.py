"""The recurrent MAPPO kernels (orl_rnn.cu, orl_rnn_warp.cuh) at C3 scale against a float64 reference.

C3 is simple_spread, 2048 envs x 3 agents, T = 25.  The golden-trace tests cover 4-8 envs, where every tape reduction
is a single 1024-row block.  Here the update runs on a real C3 buffer and on synthetic buffers built to reach the
edges of the kernels: tape reductions over many row blocks with partial last blocks, the odd-chunk tail slot of the
two-chunk warps, persistent warps looping over many chunk groups, chunk lengths 1, 7 and 32 with T = 25 (chunks that
cross trajectory rows), observation width 64 and head width 8, zero masks at chunk starts, mid-chunk and at row
crossings, and active masks with zeros.

The reference is tests/rnn_ref64.py (pinned to the unmodified reference's traces by tests/test_rnn_ref64_cpu.py).

Bars of the update (gradients per parameter block, loss sums per scalar, parameters / Adam moments / ValueNorm state
after the optimizer step) are self-calibrating: the reference runs once in float64 and once in float32 (TF32 off
for matmul and cuDNN), and the kernel's error against float64 may be at most RATIO x the float32 reference's error
against float64, never less than FLOOR and never more than CEIL (relative L2 norm per block; relative error per scalar,
against the sum of the absolute loss terms).  Rollout and critic quantities are compared element-wise at the 2e-5
absolute bar of tests/test_gru_cuda.py, teacher-forced: every float64 step starts from the device's own hidden state.
Every case prints its observed kernel / float32 error ratios (`pytest -s`)."""
import types

import numpy as np
import pytest
import torch

import rnn_ref64

pytestmark = pytest.mark.gpu

# FLOOR: the C3 entropy sum (153 600 terms added per lane, per CTA and by float atomics) is 1.1e-6 off float64, where
# torch's pairwise float32 sum is 1.6e-9 off: a long float32 sum in a fixed kernel order legitimately reaches ~1e-6.
RATIO, FLOOR, CEIL = 4.0, 2e-6, 1e-3
ATOL = 2e-5
T, H = 25, 64
KINK = 5e-3   # synthetic rows keep at least this distance from every branch point of the loss


@pytest.fixture
def no_tf32():
    before = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = before


def _rel(x, ref, scale=None):
    den = float(ref.double().norm()) if scale is None else float(scale)
    num = float((x.double() - ref.double()).norm())
    return num / den if den > 0 else num


class Checker:
    """Collects kernel-vs-float64 errors against the self-calibrated bar; fails with every violation listed."""

    def __init__(self, case, floor=FLOOR):
        self.case, self.bad, self.worst, self.floor = case, [], (0.0, ""), floor

    def bar(self, e32):
        return min(max(RATIO * e32, self.floor), CEIL)

    def __call__(self, what, got, r64, r32, scale=None):
        ek, e32 = _rel(got, r64, scale), _rel(r32, r64, scale)
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


def _compare(case, dims, k, r64, r32, check_vn):
    d, n, dc = dims
    chk = Checker(case)
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


def _lib():
    from openrl_b200 import lib
    return lib, lib.load()


def _drive(a, grads, loss_acc, outs):
    """orl_rnn_fwdbwd (gradients, loss sums), then orl_rnn_apply; `outs` names the device tensors read back after."""
    lib, L = _lib()
    s = lib.current_stream()
    lib.check(L.orl_rnn_fwdbwd(a, s), "orl_rnn_fwdbwd")
    g, la = grads.clone(), loss_acc[:4].clone()
    lib.check(L.orl_rnn_apply(a, s), "orl_rnn_apply")
    torch.cuda.synchronize()
    return g, la, {k: v.clone() for k, v in outs.items()}


def _mb_stats(rows_idx, buf_returns, buf_active):
    lib, L = _lib()
    out = torch.zeros(3, dtype=torch.float64, device="cuda")
    lib.check(L.orl_minibatch_stats(lib.ptr(rows_idx), int(rows_idx.numel()), lib.ptr(buf_returns), lib.ptr(buf_active),
                                    lib.ptr(out), lib.current_stream()), "orl_minibatch_stats")
    return out


def _refs(cfg, buf, state, ids, L, dims, joint):
    r64 = rnn_ref64.update(cfg, buf, state, ids, L, dims, joint=joint, dtype=torch.float64)
    r32 = rnn_ref64.update(cfg, buf, state, ids, L, dims, joint=joint, dtype=torch.float32)
    return r64, r32


# ---------------------------------------------------------------- the real C3 buffer ----------------------------------

C3_FLAGS = ["--episode_length", "25", "--lr", "7e-4", "--critic_lr", "7e-4", "--ppo_epoch", "1", "--use_recurrent_policy", "true",
            "--use_valuenorm", "true", "--use_adv_normalize", "true", "--log_interval", "1"]


@pytest.fixture(scope="module")
def c3():
    """One fast-mode device rollout of C3 (orl_rnn_rollout), its critic pass (orl_rnn_critic) and returns (orl_gae)."""
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.common import make
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.logger import Logger

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.manual_seed(0)
    cfg = create_config_parser().parse_args(C3_FLAGS)
    cfg.quiet = True
    env = make("simple_spread", env_num=2048)
    agent = PPOAgent(PPONet(env, cfg=cfg, device="cuda:0"))
    agent.train(total_time_steps=0, logger=Logger(quiet=True))
    drv = agent.driver
    drv.actor_rollout()
    drv.compute_returns()
    torch.cuda.synchronize()
    tr, b = drv.trainer, drv.buffer.data
    assert (b.n_rollout_threads, b.num_agents, b.episode_length, tr.chunk_length) == (2048, 3, 25, 2)
    yield types.SimpleNamespace(cfg=cfg, agent=agent, drv=drv, tr=tr, b=b)
    tr.tape = None
    torch.cuda.empty_cache()


def _c3_buf(b):
    return {k: getattr(b, k) for k in ("policy_obs", "critic_obs", "rnn_states", "rnn_states_critic", "masks", "active_masks",
                                       "actions", "action_log_probs", "value_preds", "returns", "advantages")}


@pytest.mark.parametrize("mode,mini", [("ordinary", 1), ("ordinary", 7), ("jrpo", 1), ("jrpo", 7)],
                         ids=["L2-76800chunks-153600rows", "L2-mb7-10971chunks(odd)-21942rows(partial block)",
                              "jrpo-25600chunks-153600policyrows", "jrpo-mb7-3657chunks(odd agent0 tail)"])
def test_update_on_c3_buffer(c3, no_tf32, mode, mini):
    from openrl_b200 import lib
    from openrl_b200.buffers.replay_data import chunk_row_indices, v3_row_indices

    tr, b, cfg = c3.tr, c3.b, c3.cfg
    m = tr.algo_module
    pol, cri = m.models["policy"], m.models["critic"]
    op, oc = m.optimizers["policy"], m.optimizers["critic"]
    vn = cri.value_normalizer
    live = dict(pol=pol.flat_params, cri=cri.flat_params, pol_m=op.exp_avg, pol_v=op.exp_avg_sq, cri_m=oc.exp_avg,
                cri_v=oc.exp_avg_sq, vn=vn.state)
    saved = {k: v.clone() for k, v in live.items()}
    saved_steps, saved_info = m.adam_steps.clone(), tr.train_info.clone()
    joint = mode == "jrpo"
    B, A, L = b.n_rollout_threads * b.num_agents, b.num_agents, tr.chunk_length
    total = T * (b.n_rollout_threads if joint else B) // L
    g = torch.Generator(device="cuda").manual_seed(11 + mini + 100 * joint)
    ids = torch.randperm(total, device="cuda", generator=g)[:total // mini].contiguous()
    if joint:
        stats = torch.cat([_mb_stats(v3_row_indices(ids, L, T, A, B, all_agents=ev), b.returns, b.active_masks) for ev in (False, True)])
    elif mini == 1:
        stats = b.gae_stats[5:8]
    else:
        stats = _mb_stats(chunk_row_indices(ids, L, T, B), b.returns, b.active_masks)
    tape_rows = ids.numel() * L * (A if joint else 1)
    tr.tape = torch.empty(int(tr._lib.orl_rnn_workspace_floats(tape_rows, tr.rnn_stride)), dtype=torch.float32, device="cuda")
    tr.sync_lrs()
    state = dict(saved, steps=[int(x) for x in saved_steps])
    rcfg = types.SimpleNamespace(**vars(cfg), vn_beta=vn.beta)
    try:
        a = tr._rnn_args(b, ids, stats)
        if joint:
            a.flags |= lib.PPO_JOINT_ACTION
        grads, la, after = _drive(a, tr.rnn_grads, tr.loss_acc, live)
        steps = [int(x) for x in m.adam_steps]
    finally:
        tr.tape = None
        for k, v in live.items():
            v.copy_(saved[k])
        m.adam_steps.copy_(saved_steps)
        tr.train_info.copy_(saved_info)
    dims = (tr.d, tr.n, tr.dc)
    np_, nc = int(pol.flat_params.numel()), int(cri.flat_params.numel())
    k = dict(grad_pol=grads[0, :np_], grad_cri=grads[1, :nc], losses=la, steps=steps, **after)
    r64, r32 = _refs(rcfg, _c3_buf(b), state, ids, L, dims, joint)
    _compare(f"c3-{mode}-mb{mini}", dims, k, r64, r32, check_vn=True)


def test_critic_pass_at_c3(c3):
    """orl_rnn_critic over all T + 1 slots of the 2048 x 3 buffer, teacher-forced: value_preds[t] and
    rnn_states_critic[t+1] (zero where masks[t+1] == 0) from the device's own rnn_states_critic[t]."""
    from oracle import nets

    lib, Lb = _lib()
    drv, b, cri = c3.drv, c3.b, c3.tr.algo_module.models["critic"]
    lib.check(Lb.orl_rnn_critic(drv._rnn_args(0, T, None), lib.current_stream()), "orl_rnn_critic")
    torch.cuda.synchronize()
    dc = c3.tr.dc
    p = {k: v.detach().double() for k, v in rnn_ref64.unflatten(cri.flat_params.double(), dc, 1, True).items()}
    ncfg = rnn_ref64.net_cfg(c3.cfg.activation_id, True)
    h = rnn_ref64.rows(b.rnn_states_critic).double()
    masks = rnn_ref64.rows(b.masks).double()
    with torch.no_grad():
        v, hn = nets.critic_forward(p, ncfg, rnn_ref64.rows(b.critic_obs).double(), h.unsqueeze(1), masks)
    B = b.n_rollout_threads * b.num_agents
    np.testing.assert_allclose(rnn_ref64.rows(b.value_preds).cpu().numpy(), v.cpu().numpy(), rtol=0, atol=ATOL)
    want = hn[:T * B, 0] * (masks[B:] != 0)
    np.testing.assert_allclose(h[B:].cpu().numpy(), want.cpu().numpy(), rtol=0, atol=ATOL)
    reset = masks[B:, 0] == 0
    assert int(reset.sum()) > 0 and bool((h[B:][reset] == 0).all()) and bool((h[B:][~reset].abs().amax(1) > 0).all())


def test_rollout_at_c3(c3):
    """orl_rnn_rollout on MPE at 2048 envs x 25 steps, teacher-forced: the log-prob of every recorded action and
    rnn_states[t+1] (zeroed where the env finished, masks[t+1] == 0) from the device's own rnn_states[t]."""
    from oracle import nets

    b, pol = c3.b, c3.tr.algo_module.models["policy"]
    B = b.n_rollout_threads * b.num_agents
    p = {k: v.detach().double() for k, v in rnn_ref64.unflatten(pol.flat_params.double(), c3.tr.d, c3.tr.n, False).items()}
    ncfg = rnn_ref64.net_cfg(c3.cfg.activation_id, True)
    h = rnn_ref64.rows(b.rnn_states).double()
    masks = rnn_ref64.rows(b.masks).double()
    with torch.no_grad():
        feat, hn = nets.policy_features(p, ncfg, rnn_ref64.rows(b.policy_obs).double()[:T * B], h[:T * B].unsqueeze(1), masks[:T * B])
        lp = nets.categorical_logits(p, feat).gather(-1, rnn_ref64.rows(b.actions).long())
    np.testing.assert_allclose(rnn_ref64.rows(b.action_log_probs).cpu().numpy(), lp.cpu().numpy(), rtol=0, atol=ATOL)
    want = hn[:, 0] * (masks[B:] != 0)
    np.testing.assert_allclose(h[B:].cpu().numpy(), want.cpu().numpy(), rtol=0, atol=ATOL)
    reset = masks[B:, 0] == 0
    assert int(reset.sum()) > 0 and bool((h[B:][reset] == 0).all())


@pytest.mark.parametrize("mini", [1, 7])
def test_minibatch_stats_at_c3(c3, mini):
    """orl_minibatch_stats over the gathered rows of C3 chunk minibatches (ordinary and v3, agent 0 and all agents)
    against float64 sums of the same rows."""
    from openrl_b200.buffers.replay_data import chunk_row_indices, v3_row_indices

    b, L = c3.b, c3.tr.chunk_length
    B, A, N = b.n_rollout_threads * b.num_agents, b.num_agents, b.n_rollout_threads
    g = torch.Generator(device="cuda").manual_seed(5 + mini)
    ret, act = b.returns.reshape(-1).double(), b.active_masks.reshape(-1).double()
    for idx in (chunk_row_indices(torch.randperm(T * B // L, device="cuda", generator=g)[:T * B // L // mini], L, T, B),
                v3_row_indices(torch.randperm(T * N // L, device="cuda", generator=g)[:T * N // L // mini], L, T, A, B),
                v3_row_indices(torch.randperm(T * N // L, device="cuda", generator=g)[:T * N // L // mini], L, T, A, B, all_agents=True)):
        got = _mb_stats(idx, b.returns, b.active_masks)
        r, a = ret[idx], act[idx]
        want = torch.stack([r.sum(), (r * r).sum(), a.sum()])
        np.testing.assert_allclose(got.cpu().numpy(), want.cpu().numpy(), rtol=1e-12, atol=0)
        assert idx.numel() > 7000


# ---------------------------------------------------------------- synthetic buffers -----------------------------------

BASE = dict(use_huber_loss=True, use_clipped_value_loss=True, use_value_active_masks=True, use_policy_active_masks=True,
            use_valuenorm=True, use_adv_normalize=False, use_max_grad_norm=True, dual_clip_ppo=False, activation_id=1,
            clip_param=0.2, entropy_coef=0.01, value_loss_coef=0.5, huber_delta=1.0, max_grad_norm=1e3, dual_clip_coeff=3.0,
            lr=7e-4, critic_lr=5e-4, opti_eps=1e-5, weight_decay=0.0, vn_beta=0.99999)


def _flags(c):
    from openrl_b200 import lib
    return ((lib.PPO_HUBER if c.use_huber_loss else 0) | (lib.PPO_CLIP_VALUE if c.use_clipped_value_loss else 0)
            | (lib.PPO_VALUE_ACTIVE_MASKS if c.use_value_active_masks else 0)
            | (lib.PPO_POLICY_ACTIVE_MASKS if c.use_policy_active_masks else 0) | (lib.PPO_VALUENORM if c.use_valuenorm else 0)
            | (lib.PPO_ADV_NORMALIZE if c.use_adv_normalize else 0) | (lib.PPO_MAX_GRAD_NORM if c.use_max_grad_norm else 0)
            | (lib.PPO_DUAL_CLIP if c.dual_clip_ppo else 0))


def _random_net(g, d, n, critic):
    parts = []
    for name, shp in rnn_ref64.param_shapes(d, n, critic):
        x = torch.randn(shp, generator=g, device="cuda")
        if len(shp) == 2:
            x *= (0.3 if name.startswith(("act.", "v_out")) else 1.0) / shp[1] ** 0.5
        elif name.endswith("weight"):   # LayerNorm gains
            x = 1.0 + 0.2 * x
        else:
            x *= 0.1
        parts.append(x.reshape(-1))
    return torch.cat(parts)


def _redraw(bad, draw, x):
    return torch.where(bad, draw(x.shape), x)


def _synthetic(cfg, dims, L, B, n_chunks, seed):
    """A (T, B) buffer of random observations / hidden states / masks, nets with random weights, Adam moments mid-run,
    and a chunk minibatch.  Zero masks at the first step of one chunk, mid-chunk of another and at a trajectory-row
    crossing of a third; active masks with zeros.  Old log-probs, value predictions and returns are drawn from the
    float64 forward so that no row lies near a branch point of the loss: the ratio clip edges and the dual-clip
    coefficient, the value clip, the Huber threshold and the tie of the clipped and unclipped value losses."""
    d, n, dc = dims
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, device="cuda")        # noqa: E731
    u = lambda *s: torch.rand(*s, generator=g, device="cuda")         # noqa: E731
    buf = dict(policy_obs=r(T + 1, B, d), critic_obs=r(T + 1, B, dc), rnn_states=torch.tanh(r(T + 1, B, H)),
               rnn_states_critic=torch.tanh(r(T + 1, B, H)), masks=(u(T + 1, B, 1) > 0.1).float(),
               active_masks=(u(T + 1, B, 1) > 0.1).float(), actions=torch.randint(0, n, (T, B, 1), generator=g, device="cuda").float(),
               advantages=r(T, B, 1), action_log_probs=torch.zeros(T, B, 1, device="cuda"),
               value_preds=r(T + 1, B, 1), returns=2 * r(T + 1, B, 1) + 0.5)
    total = T * B // L
    ids = torch.randperm(total, generator=g, device="cuda")[:n_chunks]
    rp, _ = rnn_ref64.gather(T, B, 1, L, ids, False)             # (L, n_chunks), time-major
    f = ids[None, :] * L + torch.arange(L, device="cuda")[:, None]
    m = rnn_ref64.rows(buf["masks"])
    m[rp[0, 0]] = 0.0                                            # chunk start
    if L > 1 and n_chunks > 1:
        m[rp[L // 2, 1]] = 0.0                                   # mid-chunk
    cross = ((f % T == 0) & (torch.arange(L, device="cuda")[:, None] > 0)).nonzero()
    if len(cross):
        m[rp[cross[0, 0], cross[0, 1]]] = 0.0                    # trajectory-row crossing
    assert L == 1 or len(cross) or n_chunks < 3
    state = dict(pol=_random_net(g, d, n, False), cri=_random_net(g, dc, 1, True), vn=torch.tensor([0.3, 1.5, 0.8], device="cuda"),
                 steps=[3, 3])
    for k in ("pol", "cri"):
        state[k + "_m"] = 1e-3 * r(state[k].numel())
        state[k + "_v"] = 1e-6 * u(state[k].numel()) + 1e-8

    pol = rnn_ref64.unflatten(state["pol"].double(), d, n, False)
    cri = rnn_ref64.unflatten(state["cri"].double(), dc, 1, True)
    with torch.no_grad():
        rp, rc, logp, _, v = rnn_ref64.forward(types.SimpleNamespace(**cfg.__dict__), buf, pol, cri, ids, L, False, torch.float64)
    rp, rc = rp.reshape(-1), rc.reshape(-1)
    kinks = torch.tensor([1 - cfg.clip_param, 1 + cfg.clip_param, cfg.dual_clip_coeff], device="cuda", dtype=torch.float64)

    def draw_ratio(shape):
        near = torch.exp(0.25 * torch.randn(shape, generator=g, device="cuda", dtype=torch.float64))
        far = 2.5 + 1.5 * torch.rand(shape, generator=g, device="cuda", dtype=torch.float64)
        return torch.where(torch.rand(shape, generator=g, device="cuda", dtype=torch.float64) < 0.1, far, near)
    ratio = draw_ratio(logp.shape)
    for _ in range(50):
        bad = ((ratio[..., None] - kinks).abs() < KINK).any(-1)
        if not bool(bad.any()):
            break
        ratio = _redraw(bad, draw_ratio, ratio)
    rows = lambda k: rnn_ref64.rows(buf[k])   # noqa: E731
    rows("action_log_probs")[rp] = (logp - ratio.log()).float()
    lp32 = rows("action_log_probs")[rp].double()
    assert bool((((logp - lp32).exp()[..., None] - kinks).abs() >= KINK / 2).all())

    draw_delta = lambda shape: 0.4 * torch.randn(shape, generator=g, device="cuda", dtype=torch.float64)   # noqa: E731
    delta = draw_delta(v.shape)
    for _ in range(50):
        bad = (delta.abs() - cfg.clip_param).abs() < KINK
        if not bool(bad.any()):
            break
        delta = _redraw(bad, draw_delta, delta)
    rows("value_preds")[rc] = (v - delta).float()
    vp = rows("value_preds")[rc].double()
    draw_ret = lambda shape: 2 * torch.randn(shape, generator=g, device="cuda", dtype=torch.float64) + 0.5   # noqa: E731
    ret = draw_ret(v.shape)
    for it in range(100):
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
    rows("returns")[rc] = ret.float()
    return buf, state, ids


def _gae_stats(buf):
    adv = rnn_ref64.rows(buf["advantages"]).double()[:, 0]
    act = rnn_ref64.rows(buf["active_masks"]).double()[:adv.numel(), 0] != 0
    ret = rnn_ref64.rows(buf["returns"]).double()[:adv.numel(), 0]
    return torch.stack([adv.sum(), (adv * adv).sum(), torch.tensor(float(adv.numel()), device="cuda", dtype=torch.float64),
                        adv[act].sum(), (adv[act] ** 2).sum(), ret.sum(), (ret * ret).sum(), act.double().sum()])


def _run_synthetic(case, cfg, dims, L, B, n_chunks, seed):
    """OrlRnnArgs built by hand for a synthetic buffer; kernel against both reference runs."""
    lib, Lb = _lib()
    from openrl_b200.buffers.replay_data import chunk_row_indices

    d, n, dc = dims
    buf, state, ids = _synthetic(cfg, dims, L, B, n_chunks, seed)
    stride = (max(Lb.orl_rnn_param_count(d, n), Lb.orl_rnn_param_count(dc, 1)) + 3) & ~3
    assert state["pol"].numel() == Lb.orl_rnn_param_count(d, n) and state["cri"].numel() == Lb.orl_rnn_param_count(dc, 1)
    bucket = torch.zeros(2 * stride + 8, dtype=torch.float32, device="cuda")
    grads, loss_acc = bucket[:2 * stride].view(2, stride), bucket[2 * stride:]
    dev = {k: state[k].clone() for k in ("pol", "cri", "pol_m", "pol_v", "cri_m", "cri_v", "vn")}
    steps = torch.tensor(state["steps"], dtype=torch.int32, device="cuda")
    lrs = torch.tensor([cfg.lr, cfg.critic_lr], dtype=torch.float32, device="cuda")
    gae_stats = _gae_stats(buf)
    mb_stats = _mb_stats(chunk_row_indices(ids, L, T, B), buf["returns"], buf["active_masks"])
    tape = torch.empty(int(Lb.orl_rnn_workspace_floats(n_chunks * L, stride)), dtype=torch.float32, device="cuda")
    train_info = torch.zeros(6, dtype=torch.float32, device="cuda")
    ids = ids.contiguous()
    a = lib.OrlRnnArgs()
    a.n_envs, a.n_agents, a.episode_length = B, 1, T
    a.obs_dim, a.critic_obs_dim, a.n_actions, a.activation_id = d, dc, n, cfg.activation_id
    a.chunk_length, a.flags, a.n_chunks, a.chunk_ids = L, _flags(cfg), n_chunks, lib.ptr(ids)
    a.policy_params, a.critic_params = lib.ptr(dev["pol"]), lib.ptr(dev["cri"])
    for k in ("policy_obs", "critic_obs", "rnn_states", "rnn_states_critic", "actions", "action_log_probs", "masks", "active_masks",
              "value_preds", "returns", "advantages"):
        setattr(a, k, lib.ptr(buf[k]))
    a.gae_stats, a.mb_stats, a.vn_state = lib.ptr(gae_stats), lib.ptr(mb_stats), lib.ptr(dev["vn"])
    a.tape, a.grads, a.grads_stride, a.loss_acc = lib.ptr(tape), lib.ptr(grads), stride, lib.ptr(loss_acc)
    a.policy_adam_m, a.policy_adam_v = lib.ptr(dev["pol_m"]), lib.ptr(dev["pol_v"])
    a.critic_adam_m, a.critic_adam_v = lib.ptr(dev["cri_m"]), lib.ptr(dev["cri_v"])
    a.adam_steps, a.lrs, a.train_info = lib.ptr(steps), lib.ptr(lrs), lib.ptr(train_info)
    a.clip_param, a.entropy_coef, a.value_loss_coef = cfg.clip_param, cfg.entropy_coef, cfg.value_loss_coef
    a.huber_delta, a.max_grad_norm, a.dual_clip_coeff = cfg.huber_delta, cfg.max_grad_norm, cfg.dual_clip_coeff
    a.adam_beta1, a.adam_beta2, a.adam_eps, a.weight_decay = 0.9, 0.999, cfg.opti_eps, cfg.weight_decay
    a.vn_beta, a.norm_rows = cfg.vn_beta, 0
    g, la, after = _drive(a, grads, loss_acc, dev)
    del tape
    k = dict(grad_pol=g[0, :state["pol"].numel()], grad_cri=g[1, :state["cri"].numel()], losses=la,
             steps=[int(x) for x in steps], **after)
    r64, r32 = _refs(cfg, buf, state, ids, L, dims, False)
    if cfg.use_max_grad_norm and cfg.max_grad_norm < 1:   # the clip case: the clip must really act on both nets
        assert float(r64["norms"][0]) > cfg.max_grad_norm and float(r64["norms"][1]) > cfg.max_grad_norm
    _compare(case, dims, k, r64, r32, check_vn=cfg.use_valuenorm)
    torch.cuda.empty_cache()


# (id, dims (d, n, dc), L, B rows per slot, n_chunks): every edge is in the id
SHAPES = [
    ("L1-5119chunks(>132x16x2,odd)-5119rows(1024k-1)-d4n2", (4, 2, 4), 1, 220, 5119),
    ("L1-2048chunks-2048rows(1024k)-d4n2", (4, 2, 4), 1, 100, 2048),
    ("L7-3chunks(odd)-21rows(<32)-d18n5-critic54", (18, 5, 54), 7, 12, 3),
    ("L7-21chunks(<16x2,odd)-147rows-d18n5-critic54", (18, 5, 54), 7, 40, 21),
    ("L7-439chunks(odd)-3073rows(1024k+1)-d18n5-critic54", (18, 5, 54), 7, 200, 439),
    ("L32(LMAX)-1chunk-32rows-crossing-d64n8", (64, 8, 64), 32, 8, 1),
    ("L32(LMAX)-4225chunks(>132x16x2,odd)-135200rows-d64n8", (64, 8, 64), 32, 5500, 4225),
]


@pytest.mark.parametrize("case,dims,L,B,n_chunks", SHAPES, ids=[s[0] for s in SHAPES])
def test_update_synthetic_edges(no_tf32, case, dims, L, B, n_chunks):
    _run_synthetic(case, types.SimpleNamespace(**BASE), dims, L, B, n_chunks, seed=len(case) * 7 + L)


FLAG_SWEEP = {
    "base": {},
    "valuenorm-off": dict(use_valuenorm=False),
    "adv-normalize": dict(use_adv_normalize=True),
    "active-masks-off": dict(use_policy_active_masks=False, use_value_active_masks=False),
    "no-huber": dict(use_huber_loss=False),
    "no-value-clip": dict(use_clipped_value_loss=False),
    "dual-clip": dict(dual_clip_ppo=True),
    "act0-tanh": dict(activation_id=0),
    "act2-leaky-relu": dict(activation_id=2),
    "act3-elu": dict(activation_id=3),
    "grad-clip-active": dict(max_grad_norm=1e-2),
}


@pytest.mark.parametrize("name", list(FLAG_SWEEP), ids=list(FLAG_SWEEP))
def test_update_flag_sweep(no_tf32, name):
    """One mid-size shape (L = 7, 1001 chunks, 7007 rows, d = 18, n = 5, critic 54) under each loss / optimizer option."""
    cfg = types.SimpleNamespace(**{**BASE, **FLAG_SWEEP[name]})
    _run_synthetic(f"flags-{name}", cfg, (18, 5, 54), 7, 400, 1001, seed=1234)
