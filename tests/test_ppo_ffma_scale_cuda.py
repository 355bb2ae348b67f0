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
tests/scale_harness.py at its PPO_FLOOR: per parameter block, the kernel's relative L2 error against float64 may be at
most RATIO x the float32 reference's error against float64, clamped to [PPO_FLOOR, CEIL]; loss sums are
relative to the weighted sum of their absolute terms and Adam's exp_avg to the terms it combines.  Every case prints its
kernel / float32 error ratios (`pytest -s`)."""
import types

import numpy as np
import pytest
import torch

import ffma_ref64 as ref
import scale_harness as h
from scale_harness import ATOL, CASES, PPO_FLOOR, Checker, no_tf32  # noqa: F401  (no_tf32: pytest fixture)

pytestmark = pytest.mark.gpu

P_M = 128   # rows per tile of the FFMA update kernel
C5_FLAGS = ["--seed", "0", "--episode_length", "128", "--ppo_epoch", "4", "--num_mini_batch", "1", "--log_interval", "1",
            "--host_env_groups", "false"]


def _grid():
    """CTAs per net of the FFMA update: half the SMs (PPOAlgorithm.grid_per_net)."""
    return max(1, torch.cuda.get_device_properties(0).multi_processor_count // 2)


def _compare(case, dims, head, k, r64, r32, state, cfg, check_vn=True):
    d, n, dc = dims
    chk = Checker(case, PPO_FLOOR)
    nets = (("pol", d, n, head), ("cri", dc, 1, "critic"))
    for net, dd, nn, hd in nets:
        for name, s in ref.blocks(dd, nn, hd).items():
            chk(f"grad {net}.{name}", k["grad_" + net][s], r64["grad_" + net][s], r32["grad_" + net][s])
    for i, name in enumerate(("policy loss", "entropy", "ratio sum", "value loss")):
        chk(f"loss sum {name}", k["losses"][i:i + 1], r64["losses"][i:i + 1], r32["losses"][i:i + 1], scale=r64["loss_scales"][i])
    for col, name, j in ((4, "actor grad norm", 0), (1, "critic grad norm", 1), (5, "ratio mean", None)):
        pick = lambda r: (r["ratio_mean"] if j is None else r["norms"][j]).reshape(1)   # noqa: E731
        chk(f"train_info {name}", k["info"][col:col + 1], pick(r64), pick(r32))
    mscale = {net: h.moment_scale(cfg, r64["grad_" + net], r64["norms"][j], state[net], state[net + "_m"])
              for j, net in enumerate(("pol", "cri"))}
    for net, dd, nn, hd in nets:
        for key in ("", "_m", "_v"):
            for name, s in ref.blocks(dd, nn, hd).items():
                chk(f"{net}{key or '_param'} {name}", k[net + key][s], r64[net + key][s], r32[net + key][s],
                    scale=mscale[net][s].norm() if key == "_m" else None)
    if check_vn:
        chk("vn_state", k["vn"], r64["vn"], r32["vn"])
    assert k["steps"] == [r64["pol_step"], r64["cri_step"]]
    chk.done()


# ---------------------------------------------------------------- the real C5 buffer ----------------------------------

@pytest.fixture(scope="module")
def c5():
    """One rollout of C5 (the HalfCheetah-shaped synthetic host env of test_gaussian_cuda) and its returns."""
    from openrl_b200 import lib
    from openrl_b200.envs.vec_env import HostVecEnv
    from helpers import SyntheticHost, make_agent

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.manual_seed(0)
    cfg, net, agent = make_agent(HostVecEnv(SyntheticHost(1024)), C5_FLAGS)
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
    snap = h.snapshot(c5)
    rows = torch.arange(c5.rows, device="cuda")
    try:
        for epoch in range(4):
            state = h.state(c5)
            k = h.kernel_update(c5, None, c5.b.gae_stats[5:8], c5.rows)
            r64, r32 = _refs(c5, state, rows)
            _compare(f"c5-epoch{epoch + 1}-contiguous-{c5.rows}rows", (17, 6, 17), "gaussian", k, r64, r32, state, c5.cfg)
            spread = float(r64["ratio_spread"])
            assert (spread > 1e-4) if epoch else (spread < 1e-4), spread   # epoch 1: every ratio 1 up to rounding
    finally:
        h.restore(c5, snap)


def test_c5_shuffled_quarter(c5, no_tf32):
    """num_mini_batch 4 on the same buffer: a shuffled index list of a quarter of the rows, orl_minibatch_stats."""
    snap = h.snapshot(c5)
    g = torch.Generator(device="cuda").manual_seed(4)
    idx = torch.randperm(c5.rows, device="cuda", generator=g)[:c5.rows // 4].contiguous()
    assert idx.numel() == 32768
    try:
        state = h.state(c5)
        k = h.kernel_update(c5, idx, h.mb_stats(idx, c5.b.returns, c5.b.active_masks), idx.numel())
        r64, r32 = _refs(c5, state, idx)
        _compare("c5-mb4-shuffled-32768rows", (17, 6, 17), "gaussian", k, r64, r32, state, c5.cfg)
    finally:
        h.restore(c5, snap)


# ---------------------------------------------------------------- deliberate mistakes ---------------------------------

@pytest.mark.parametrize("mutant", list(ref.MUTANTS))
def test_c5_mutants_are_detected(c5, no_tf32, mutant):
    """The real kernel output on the C5 buffer against a float64 reference with one deliberate mistake: the block the
    mistake lands in must violate its bar (and pass it against the correct reference)."""
    from openrl_b200 import lib

    _, what, opts, moved = ref.MUTANTS[mutant]
    snap, flags = h.snapshot(c5), c5.tr.flags
    rows = torch.arange(c5.rows, device="cuda")
    try:
        if moved:      # start from the state after one update: ratios away from 1
            h.kernel_update(c5, None, c5.b.gae_stats[5:8], c5.rows)
        if opts.get("use_policy_active_masks") is False:
            c5.tr.flags &= ~lib.PPO_POLICY_ACTIVE_MASKS
        state = h.state(c5)
        k = h.kernel_update(c5, None, c5.b.gae_stats[5:8], c5.rows)
    finally:
        c5.tr.flags = flags
        h.restore(c5, snap)
    G, tiles = c5.tr.grid_per_net, c5.rows // P_M
    last = (tiles - 1) // G * G           # CTA 0's last tile
    dropped = torch.arange(last * P_M, last * P_M + P_M, device="cuda")
    r64, r32 = _refs(c5, state, rows, cfg=opts)
    bad, _ = _refs(c5, state, rows, cfg=opts, mutant=mutant, dropped_rows=dropped)
    net, name = what.split(" ")[1].split(".", 1)
    s = ref.blocks(17, 6 if net == "pol" else 1, "gaussian" if net == "pol" else "critic")[name]
    got, want, wrong, r32s = k["grad_" + net][s], r64["grad_" + net][s], bad["grad_" + net][s], r32["grad_" + net][s]
    good = Checker(f"c5-{mutant}", PPO_FLOOR)
    good(what, got, want, r32s)
    good.done()
    e_bad, bar = h.rel(got, wrong), good.bar(h.rel(r32s, want))
    print(f"  c5-{mutant}: kernel against the mutant {e_bad:.2e}, bar {bar:.2e}")
    assert e_bad > bar, f"{mutant}: the mistake ({ref.MUTANTS[mutant][0]}) passed the bar of {what}"


# ---------------------------------------------------------------- synthetic buffers -----------------------------------

def _run_synthetic(case, cfg, dims, head, batch_rows, contiguous_from=None, total=None, seed=0):
    """OrlPpoArgs built by hand for a synthetic buffer; the kernel against both reference runs."""
    lb, L = h.lib()
    d, n, dc = dims
    G = _grid()
    total = total or batch_rows + 301
    idx, rows_idx = h.minibatch(total, batch_rows, contiguous_from, seed)
    buf, state = h.ppo_synthetic(cfg, dims, head, total, rows_idx, seed)
    gauss = head == "gaussian"
    stride, gstride = L.orl_ppo_stride(d, dc, n), L.orl_ppo_grads_stride(d, dc, n)
    partials = torch.zeros(2 * G, stride, device="cuda")
    folded = torch.zeros(2, stride, device="cuda")
    grads = torch.zeros(2, gstride, device="cuda")
    dev = {k: state[k].clone() for k in ("pol", "cri", "pol_m", "pol_v", "cri_m", "cri_v", "vn")}
    assert dev["pol"].numel() == L.orl_net_param_count(d, n) + (n if gauss else 0)
    steps = torch.tensor(state["steps"], dtype=torch.int32, device="cuda")
    lrs = torch.tensor([cfg.lr, cfg.critic_lr], dtype=torch.float32, device="cuda")
    stats = h.gae_stats(buf), h.mb_stats(rows_idx.contiguous(), buf["returns"], buf["active_masks"])
    train_info = torch.zeros(6, device="cuda")
    a = h.ppo_args(cfg, dims, lb.HEAD_GAUSSIAN if gauss else lb.HEAD_CATEGORICAL, h.ppo_flags(cfg), G, buf, batch_rows, total,
                   idx, contiguous_from or 0, stats, dev, steps, lrs, train_info, partials, folded, grads)
    s = lb.current_stream()
    lb.check(L.orl_ppo_fwdbwd(a, s), "orl_ppo_fwdbwd")
    lb.check(L.orl_ppo_reduce(a, s), "orl_ppo_reduce")
    lb.check(L.orl_ppo_apply(a, s), "orl_ppo_apply")
    torch.cuda.synchronize()
    k = dict(grad_pol=grads[0, :dev["pol"].numel()], grad_cri=grads[1, :dev["cri"].numel()], losses=h.loss_sums(folded, stride),
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
    cfg = types.SimpleNamespace(**h.BASE)
    _run_synthetic(case, cfg, dims, head, _rows(rows_kind), seed=len(case) * 7 + dims[0])


@pytest.mark.parametrize("dims,head", [((17, 6, 17), "gaussian"), ((18, 5, 54), "categorical")], ids=["gauss-d17-n6", "cat-mpe"])
def test_update_contiguous_range_not_at_row_zero(no_tf32, dims, head):
    """The contiguous gather (indices == NULL) of a range that starts at row 1000 of a larger buffer, many tiles per
    CTA, partial last tile."""
    G = _grid()
    rows = 2 * G * P_M + 77
    cfg = types.SimpleNamespace(**h.BASE)
    _run_synthetic(f"contiguous-from-1000-{head}-{rows}rows", cfg, dims, head, rows, contiguous_from=1000, total=rows + 1500,
                   seed=dims[0])


@pytest.mark.parametrize("flags", CASES, ids=[" ".join(c) or "default" for c in CASES])
def test_update_flag_sweep_gaussian(no_tf32, flags):
    """Every option of tests/test_ppo_flags_cuda.py on a Gaussian (17, 6) buffer, 3 G tiles + 37 rows (4 tiles per
    CTA), through the FFMA kernel: policy active masks on (default) and off, Huber off, value clip off, ValueNorm off,
    dual clip, A2C, weight decay, the activations, other coefficients and a gradient clip that acts on both nets."""
    cfg = h.flag_cfg(flags)
    _run_synthetic("flags-" + ("-".join(flags) or "default"), cfg, (17, 6, 17), "gaussian", 3 * _grid() * P_M + 37, seed=77)
