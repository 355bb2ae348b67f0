"""The recurrent MAPPO kernels (orl_rnn.cu, orl_rnn_warp.cuh) at C3 scale against a float64 reference.

C3 is simple_spread, 2048 envs x 3 agents, T = 25.  The golden-trace tests cover 4-8 envs, where every tape reduction
is a single 1024-row block.  Here the update runs on a real C3 buffer and on synthetic buffers built to reach the
edges of the kernels: tape reductions over many row blocks with partial last blocks, the odd-chunk tail slot of the
two-chunk warps, persistent warps looping over many chunk groups, chunk lengths 1, 7 and 32 with T = 25 (chunks that
cross trajectory rows), observation width 64 and head width 8, zero masks at chunk starts, mid-chunk and at row
crossings, and active masks with zeros.

The reference is tests/rnn_ref64.py (pinned to the unmodified reference's traces by tests/test_rnn_ref64_cpu.py).

Bars of the update (tests/scale_harness.py; gradients per parameter block, loss sums per scalar, parameters / Adam moments / ValueNorm state
after the optimizer step) are self-calibrating: the reference runs once in float64 and once in float32 (TF32 off
for matmul and cuDNN), and the kernel's error against float64 may be at most RATIO x the float32 reference's error
against float64, never less than RNN_FLOOR and never more than CEIL (relative L2 norm per block; relative error per scalar,
against the sum of the absolute loss terms).  Rollout and critic quantities are compared element-wise at the 2e-5
absolute bar of tests/test_gru_cuda.py, teacher-forced: every float64 step starts from the device's own hidden state.
Every case prints its observed kernel / float32 error ratios (`pytest -s`)."""
import types

import numpy as np
import pytest
import torch

import rnn_ref64
import scale_harness as h
from scale_harness import ATOL, BASE, no_tf32  # noqa: F401  (no_tf32: pytest fixture)

pytestmark = pytest.mark.gpu

T, H = 25, 64


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
    from openrl_b200.envs.common import make
    from helpers import make_agent

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.manual_seed(0)
    cfg, _, agent = make_agent(make("simple_spread", env_num=2048), C3_FLAGS)
    drv = agent.driver
    drv.actor_rollout()
    drv.compute_returns()
    torch.cuda.synchronize()
    tr, b = drv.trainer, drv.buffer.data
    assert (b.n_rollout_threads, b.num_agents, b.episode_length, tr.chunk_length) == (2048, 3, 25, 2)
    yield types.SimpleNamespace(cfg=cfg, agent=agent, drv=drv, tr=tr, b=b)
    tr.tape = None
    torch.cuda.empty_cache()


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
        stats = torch.cat([h.mb_stats(v3_row_indices(ids, L, T, A, B, all_agents=ev), b.returns, b.active_masks) for ev in (False, True)])
    elif mini == 1:
        stats = b.gae_stats[5:8]
    else:
        stats = h.mb_stats(chunk_row_indices(ids, L, T, B), b.returns, b.active_masks)
    tape_rows = ids.numel() * L * (A if joint else 1)
    tr.tape = torch.empty(int(tr._lib.orl_rnn_workspace_floats(tape_rows, tr.rnn_stride)), dtype=torch.float32, device="cuda")
    tr.sync_lrs()
    state = dict(saved, steps=[int(x) for x in saved_steps])
    rcfg = types.SimpleNamespace(**vars(cfg), vn_beta=vn.beta)
    try:
        a = tr._rnn_args(b, ids, stats)
        if joint:
            a.flags |= lib.PPO_JOINT_ACTION
        grads, la, after = h.drive(a, tr.rnn_grads, tr.loss_acc, live)
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
    r64, r32 = _refs(rcfg, h.c3_buf(b), state, ids, L, dims, joint)
    h.rnn_compare(f"c3-{mode}-mb{mini}", dims, k, r64, r32, check_vn=True)


def test_critic_pass_at_c3(c3):
    """orl_rnn_critic over all T + 1 slots of the 2048 x 3 buffer, teacher-forced: value_preds[t] and
    rnn_states_critic[t+1] (zero where masks[t+1] == 0) from the device's own rnn_states_critic[t]."""
    from oracle import nets

    lb, Lb = h.lib()
    drv, b, cri = c3.drv, c3.b, c3.tr.algo_module.models["critic"]
    lb.check(Lb.orl_rnn_critic(drv._rnn_args(0, T, None), lb.current_stream()), "orl_rnn_critic")
    torch.cuda.synchronize()
    dc = c3.tr.dc
    p = {k: v.detach().double() for k, v in rnn_ref64.unflatten(cri.flat_params.double(), dc, 1, True).items()}
    ncfg = rnn_ref64.net_cfg(c3.cfg.activation_id, True)
    hid = rnn_ref64.rows(b.rnn_states_critic).double()
    masks = rnn_ref64.rows(b.masks).double()
    with torch.no_grad():
        v, hn = nets.critic_forward(p, ncfg, rnn_ref64.rows(b.critic_obs).double(), hid.unsqueeze(1), masks)
    B = b.n_rollout_threads * b.num_agents
    np.testing.assert_allclose(rnn_ref64.rows(b.value_preds).cpu().numpy(), v.cpu().numpy(), rtol=0, atol=ATOL)
    want = hn[:T * B, 0] * (masks[B:] != 0)
    np.testing.assert_allclose(hid[B:].cpu().numpy(), want.cpu().numpy(), rtol=0, atol=ATOL)
    reset = masks[B:, 0] == 0
    assert int(reset.sum()) > 0 and bool((hid[B:][reset] == 0).all()) and bool((hid[B:][~reset].abs().amax(1) > 0).all())


def test_rollout_at_c3(c3):
    """orl_rnn_rollout on MPE at 2048 envs x 25 steps, teacher-forced: the log-prob of every recorded action and
    rnn_states[t+1] (zeroed where the env finished, masks[t+1] == 0) from the device's own rnn_states[t]."""
    from oracle import nets

    b, pol = c3.b, c3.tr.algo_module.models["policy"]
    B = b.n_rollout_threads * b.num_agents
    p = {k: v.detach().double() for k, v in rnn_ref64.unflatten(pol.flat_params.double(), c3.tr.d, c3.tr.n, False).items()}
    ncfg = rnn_ref64.net_cfg(c3.cfg.activation_id, True)
    hid = rnn_ref64.rows(b.rnn_states).double()
    masks = rnn_ref64.rows(b.masks).double()
    with torch.no_grad():
        feat, hn = nets.policy_features(p, ncfg, rnn_ref64.rows(b.policy_obs).double()[:T * B], hid[:T * B].unsqueeze(1), masks[:T * B])
        lp = nets.categorical_logits(p, feat).gather(-1, rnn_ref64.rows(b.actions).long())
    np.testing.assert_allclose(rnn_ref64.rows(b.action_log_probs).cpu().numpy(), lp.cpu().numpy(), rtol=0, atol=ATOL)
    want = hn[:, 0] * (masks[B:] != 0)
    np.testing.assert_allclose(hid[B:].cpu().numpy(), want.cpu().numpy(), rtol=0, atol=ATOL)
    reset = masks[B:, 0] == 0
    assert int(reset.sum()) > 0 and bool((hid[B:][reset] == 0).all())


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
        got = h.mb_stats(idx, b.returns, b.active_masks)
        r, a = ret[idx], act[idx]
        want = torch.stack([r.sum(), (r * r).sum(), a.sum()])
        np.testing.assert_allclose(got.cpu().numpy(), want.cpu().numpy(), rtol=1e-12, atol=0)
        assert idx.numel() > 7000


# ---------------------------------------------------------------- synthetic buffers -----------------------------------

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
    state = dict(pol=h.random_net(g, rnn_ref64.param_shapes(d, n, False)), cri=h.random_net(g, rnn_ref64.param_shapes(dc, 1, True)),
                 vn=torch.tensor([0.3, 1.5, 0.8], device="cuda"), steps=[3, 3])
    for k in ("pol", "cri"):
        state[k + "_m"] = 1e-3 * r(state[k].numel())
        state[k + "_v"] = 1e-6 * u(state[k].numel()) + 1e-8

    pol = rnn_ref64.unflatten(state["pol"].double(), d, n, False)
    cri = rnn_ref64.unflatten(state["cri"].double(), dc, 1, True)
    with torch.no_grad():
        rp, rc, logp, _, v = rnn_ref64.forward(types.SimpleNamespace(**cfg.__dict__), buf, pol, cri, ids, L, False, torch.float64)
    rp, rc = rp.reshape(-1), rc.reshape(-1)
    rows = lambda k: rnn_ref64.rows(buf[k])   # noqa: E731
    h.draw_kink_free(g, cfg, state["vn"], logp, v, rows("action_log_probs"), rp, rows("value_preds"), rows("returns"), rc,
                   ratio_spread=0.25, returns_draw=(2.0, 0.5), both_clip_sides=False)
    return buf, state, ids


def _run_synthetic(case, cfg, dims, L, B, n_chunks, seed):
    """OrlRnnArgs built by hand for a synthetic buffer; kernel against both reference runs."""
    lb, Lb = h.lib()
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
    gae = h.gae_stats({k: rnn_ref64.rows(buf[k]) for k in ("advantages", "active_masks", "returns")})
    mb = h.mb_stats(chunk_row_indices(ids, L, T, B), buf["returns"], buf["active_masks"])
    tape = torch.empty(int(Lb.orl_rnn_workspace_floats(n_chunks * L, stride)), dtype=torch.float32, device="cuda")
    train_info = torch.zeros(6, dtype=torch.float32, device="cuda")
    ids = ids.contiguous()
    a = lb.OrlRnnArgs()
    a.n_envs, a.n_agents, a.episode_length = B, 1, T
    a.obs_dim, a.critic_obs_dim, a.n_actions, a.activation_id = d, dc, n, cfg.activation_id
    a.chunk_length, a.flags, a.n_chunks, a.chunk_ids = L, h.ppo_flags(cfg), n_chunks, lb.ptr(ids)
    a.policy_params, a.critic_params = lb.ptr(dev["pol"]), lb.ptr(dev["cri"])
    for k in ("policy_obs", "critic_obs", "rnn_states", "rnn_states_critic", "actions", "action_log_probs", "masks", "active_masks",
              "value_preds", "returns", "advantages"):
        setattr(a, k, lb.ptr(buf[k]))
    a.gae_stats, a.mb_stats, a.vn_state = lb.ptr(gae), lb.ptr(mb), lb.ptr(dev["vn"])
    a.tape, a.grads, a.grads_stride, a.loss_acc = lb.ptr(tape), lb.ptr(grads), stride, lb.ptr(loss_acc)
    a.policy_adam_m, a.policy_adam_v = lb.ptr(dev["pol_m"]), lb.ptr(dev["pol_v"])
    a.critic_adam_m, a.critic_adam_v = lb.ptr(dev["cri_m"]), lb.ptr(dev["cri_v"])
    a.adam_steps, a.lrs, a.train_info = lb.ptr(steps), lb.ptr(lrs), lb.ptr(train_info)
    h.fill_coefs(a, cfg)
    g, la, after = h.drive(a, grads, loss_acc, dev)
    del tape
    k = dict(grad_pol=g[0, :state["pol"].numel()], grad_cri=g[1, :state["cri"].numel()], losses=la,
             steps=[int(x) for x in steps], **after)
    r64, r32 = _refs(cfg, buf, state, ids, L, dims, False)
    if cfg.use_max_grad_norm and cfg.max_grad_norm < 1:   # the clip case: the clip must really act on both nets
        assert float(r64["norms"][0]) > cfg.max_grad_norm and float(r64["norms"][1]) > cfg.max_grad_norm
    h.rnn_compare(case, dims, k, r64, r32, check_vn=cfg.use_valuenorm)
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
