"""The tensor-core PPO update (`ppo_fwdbwd_tc_kernel`, orl_ppo_tc.cu, + `orl_ppo_reduce` + `orl_ppo_apply`) at C2 scale
against a float64 reference, where every CTA walks 31-32 tiles of 128 rows.

The wgmma kernel is the update of every Categorical net with observation widths up to 8, and the one in the C2 bench line
(CartPole, 4096 envs, T = 128, 4 epochs of one 524 288-row minibatch).  It carries its weight-gradient sums across tiles
in wgmma accumulators, overlaps each tile's weight-gradient MMAs with the next tile's staging, and scales its backward
operands by powers of two chosen per minibatch.  Here it runs (a) on a real C2 buffer, contiguous (TMA staging, GAE
moments) and on a shuffled quarter (gather staging); (b) on synthetic buffers at the edges of its templates and row
loops; (c) through both staging paths on the same rows, which must agree bit for bit; (d) with every buffer row outside
the minibatch poisoned, which must change nothing; (e) at the edges of its operand scales; (f) against deliberately wrong
references, to show that the bars catch subtle mistakes.

Bars.  The reference is tests/tc_ref64.py (the oracle's float64 update with per-row gradient terms).  The tensor-core
kernel adds ~4000 rows per CTA in truncating fp32 accumulators, and a policy-gradient block is a sum of terms of both
signs whose absolute sum can be far above its norm, so its error is bounded against that absolute sum:
    || kernel - float64 ||_2  <=  TAU * S_block,     S_block = || sum_r |c_r| ||_2
for every gradient block and every loss sum (against the weighted sum of its absolute terms).  The relative L2 errors of
the kernel and of a float32 torch run are printed for information (`pytest -s`).  Parameters after the Adam step are
compared in units of lr: an element whose float64 gradient is outside the bar's noise must land within 0.1 lr, one inside
it may move by up to one Adam step, and such elements must be few.  Adam moments are bounded through the same gradient
bar; the ValueNorm state and the ratio mean use the self-calibrated bar of tests/test_rnn_scale_cuda.py."""
import types

import pytest
import torch

import ffma_ref64
import scale_harness as h
import tc_ref64 as ref
from scale_harness import BASE, PPO_FLOOR, Checker, no_tf32  # noqa: F401  (no_tf32: pytest fixture)

pytestmark = pytest.mark.gpu

T_M = 128   # rows per tile of the tensor-core update kernel
# TAU, measured on an H100 SXM (132 SMs, 700 W power limit; grid_per_net 132, 31-32 tiles per CTA at C2): the worst
# kernel err/S of every case here is 2.25e-5, in C2 epoch 1's critic blocks (LayerNorm-1 gain, fc3 weight), whose value
# gradients barely cancel (S ~ 1.1 x the block's norm), so that the accumulators' truncation over ~770 wgmma accumulate
# steps per CTA shows in full; policy blocks stay at 2.7e-6 of S.  TAU is that worst value x 1.8.  The mutants sit at
# 1.2 TAU (127 rows past a partial last tile), 2.3 TAU (a stale tile) and 2.5 TAU (a dropped tile) on C2.
TAU = 4e-5
NOISE = 4.0        # an element is in the noise when |float64 gradient| <= NOISE * TAU * (its sum of absolute row terms)
NOISY_SHARE = 0.02   # at most this share of a block's elements may be in the noise and move by more than 0.1 lr
C2_FLAGS = ["--seed", "0", "--episode_length", "128", "--ppo_epoch", "4", "--num_mini_batch", "1", "--log_interval", "1000000",
            "--log_each_episode", "false"]


@pytest.fixture(autouse=True)
def _needs_cuda(cuda):
    pass


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


class TauChecker:
    """Collects kernel-vs-float64 errors against TAU x the absolute-term scale; fails with every violation listed."""

    def __init__(self, case):
        self.case, self.bad, self.worst = case, [], (0.0, "")

    def __call__(self, what, got, r64, scale, r32=None):
        err = float((got.double() - r64.double()).norm())
        es = err / float(scale) if float(scale) > 0 else (0.0 if err == 0 else float("inf"))
        rk = h.rel(got, r64)
        r32s = f"fp32 {h.rel(r32, r64):9.2e}" if r32 is not None else " " * 14
        if es > self.worst[0]:
            self.worst = (es, what)
        print(f"  {self.case:44s} {what:42s} rel kernel {rk:9.2e} {r32s}  err/S {es:9.2e}  bar {TAU:.1e}")
        if not es <= TAU:
            self.bad.append(f"{what}: err/S {es:.3e} > TAU {TAU:.1e} (relative L2 {rk:.2e})")
        return es

    def done(self):
        print(f"  {self.case}: worst err/S {self.worst[0]:.2e} = {self.worst[0] / TAU:.2f} TAU ({self.worst[1]})")
        assert not self.bad, f"{self.case}:\n" + "\n".join(self.bad)


def _clip(r64, j, cfg):
    return min(1.0, cfg.max_grad_norm / (float(r64["norms"][j]) + 1e-6)) if cfg.use_max_grad_norm else 1.0


def compare(case, dims, k, r64, r32, state, cfg, check_vn=True):
    """Every quantity of one update: gradients and loss sums against TAU x S, train_info, Adam state, ValueNorm."""
    chk, calib = TauChecker(case), Checker(case, PPO_FLOOR)
    s_tot = {}
    for net in ("pol", "cri"):
        tot = 0.0
        for name, s in ref.blocks(dims, net).items():
            absum = r64["terms_" + net][name][1]
            chk(f"grad {net}.{name}", k["grad_" + net][s], r64["grad_" + net][s], absum.norm(), r32["grad_" + net][s])
            tot += float(absum.norm()) ** 2
        s_tot[net] = tot ** 0.5
    for i, name in enumerate(("policy loss", "entropy", "ratio sum", "value loss")):
        chk(f"loss sum {name}", k["losses"][i:i + 1], r64["losses"][i:i + 1], r64["loss_scales"][i], r32["losses"][i:i + 1])
    # train_info: value_loss, critic_grad_norm, policy_loss, dist_entropy, actor_grad_norm, ratio (a norm differs by at
    # most the norm of the gradient's error, so its bar is TAU x the net's total absolute-term scale)
    for col, name, want, scale in ((0, "value loss", r64["losses"][3], r64["loss_scales"][3]),
                                   (2, "policy loss", r64["losses"][0], r64["loss_scales"][0]),
                                   (3, "entropy", r64["losses"][1], r64["loss_scales"][1]),
                                   (1, "critic grad norm", r64["norms"][1], s_tot["cri"]),
                                   (4, "actor grad norm", r64["norms"][0], s_tot["pol"])):
        chk(f"train_info {name}", k["info"][col:col + 1], want.reshape(1), scale)
    calib("train_info ratio mean", k["info"][5:6], r64["ratio_mean"].reshape(1), r32["ratio_mean"].reshape(1))
    lr = {"pol": cfg.lr, "cri": cfg.critic_lr}
    for j, net in enumerate(("pol", "cri")):
        c = _clip(r64, j, cfg)
        for name, s in ref.blocks(dims, net).items():
            absum = r64["terms_" + net][name][1]
            g64 = r64["grad_" + net][s]
            noisy = g64.abs() <= NOISE * TAU * absum
            # exp_avg moves by (1 - beta1) x the clipped gradient's error; exp_avg_sq by (1 - beta2) x 2 |g| x that error
            em = float((k[net + "_m"][s].double() - r64[net + "_m"][s]).norm())
            bm = 0.1 * c * TAU * float(absum.norm()) + 1e-6 * float(r64[net + "_m"][s].norm()) + 1e-30
            ev = float((k[net + "_v"][s].double() - r64[net + "_v"][s]).norm())
            bv = 0.002 * c * c * float(g64.abs().max()) * TAU * float(absum.norm()) + 1e-6 * float(r64[net + "_v"][s].norm()) + 1e-30
            dp = (k[net][s].double() - r64[net][s]).abs() / lr[net]
            far = dp > 0.1
            n_noisy_far = int((far & noisy).sum())
            print(f"  {case:44s} {net}_param {name:32s} max |dp| {float(dp.max()):.2e} lr, {n_noisy_far} noisy elements "
                  f"moved > 0.1 lr; exp_avg {em / bm:.2f} of bar, exp_avg_sq {ev / bv:.2f} of bar")
            if bool((far & ~noisy).any()) or float(dp.max()) > 1.0 + 1e-3 or n_noisy_far > NOISY_SHARE * dp.numel() + 1:
                chk.bad.append(f"{net}_param {name}: max |dp| {float(dp.max()):.2e} lr, {int((far & ~noisy).sum())} elements "
                               f"outside the noise and {n_noisy_far} inside it moved by > 0.1 lr")
            if em > bm or ev > bv:
                chk.bad.append(f"{net} Adam moments {name}: exp_avg {em:.3e} (bar {bm:.3e}), exp_avg_sq {ev:.3e} (bar {bv:.3e})")
    if check_vn:
        calib("vn_state", k["vn"], r64["vn"], r32["vn"])
    assert k["steps"] == [r64["pol_step"], r64["cri_step"]]
    chk.done()
    calib.done()
    return chk.worst[0]


# ---------------------------------------------------------------- the real C2 buffer ----------------------------------

@pytest.fixture(scope="module")
def c2():
    """The bench's C2 agent (CartPole-v1, 4096 device envs), one rollout and its returns."""
    from openrl_b200.envs.common import make
    from helpers import make_agent

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.manual_seed(0)
    cfg, net, agent = make_agent(make("CartPole-v1", env_num=4096), C2_FLAGS)
    drv = agent.driver
    drv.actor_rollout()
    drv.compute_returns()
    torch.cuda.synchronize()
    tr, b = drv.trainer, drv.buffer.data
    T, N = b.episode_length, b.n_rollout_threads
    rows = T * N * b.num_agents
    assert (T, N, b.num_agents, tr.d, tr.n, tr.dc) == (128, 4096, 1, 4, 2, 4)
    assert tr.use_tensor_cores and tr.grid_per_net == _sms() and not tr.share
    tiles = rows // T_M
    assert rows % T_M == 0 and tiles // tr.grid_per_net >= 8   # H100 SXM: 4096 tiles over 132 CTAs, 31-32 per CTA
    print(f"\n  C2: {rows} rows, {tiles} tiles, {tr.grid_per_net} CTAs per net, "
          f"{tiles // tr.grid_per_net}-{-(-tiles // tr.grid_per_net)} tiles per CTA")
    m = tr.algo_module
    pol, cri = m.models["policy"], m.models["critic"]
    op, oc = m.optimizers["policy"], m.optimizers["critic"]
    live = dict(pol=pol.flat_params, cri=cri.flat_params, pol_m=op.exp_avg, pol_v=op.exp_avg_sq, cri_m=oc.exp_avg,
                cri_v=oc.exp_avg_sq, vn=cri.value_normalizer.state)
    assert b.action_masks_trivial
    buf = dict(policy_obs=b.policy_obs.reshape(-1, 4), critic_obs=b.critic_obs.reshape(-1, 4), actions=b.actions.reshape(-1, 1),
               action_log_probs=b.action_log_probs.reshape(-1, 1), advantages=b.advantages.reshape(-1, 1)[:rows],
               value_preds=b.value_preds.reshape(-1, 1), returns=b.returns.reshape(-1, 1), active_masks=b.active_masks.reshape(-1, 1))
    yield types.SimpleNamespace(cfg=cfg, tr=tr, b=b, rows=rows, m=m, live=live, buf=buf, vn_beta=cri.value_normalizer.beta)
    torch.cuda.empty_cache()


def _refs(c, state, rows_idx):
    r64 = ref.update(c.cfg, c.buf, state, rows_idx, (4, 2, 4), vn_beta=c.vn_beta)
    r32 = ffma_ref64.update(c.cfg, c.buf, state, rows_idx, (4, 2, 4), "categorical", torch.float32, vn_beta=c.vn_beta)
    return r64, r32


def test_c2_four_epochs_contiguous(c2, no_tf32):
    """C2's four updates (4 epochs over the whole buffer, indices == NULL: TMA staging, the GAE moments as minibatch
    moments), each teacher-forced from the device's own state before it.  Epoch 1 has every ratio at 1."""
    snap = h.snapshot(c2)
    rows = torch.arange(c2.rows, device="cuda")
    try:
        for epoch in range(4):
            state = h.state(c2)
            k = h.kernel_update(c2, None, c2.b.gae_stats[5:8], c2.rows)
            r64, r32 = _refs(c2, state, rows)
            compare(f"c2-epoch{epoch + 1}-contiguous-{c2.rows}rows", (4, 2, 4), k, r64, r32, state, c2.cfg)
            spread = float(r64["ratio_spread"])
            assert (spread > 1e-4) if epoch else (spread < 1e-4), spread
    finally:
        h.restore(c2, snap)


def test_c2_shuffled_quarter(c2, no_tf32):
    """num_mini_batch 4 on the same buffer: a shuffled quarter (gather staging, two tiles ahead), orl_minibatch_stats."""
    snap = h.snapshot(c2)
    g = torch.Generator(device="cuda").manual_seed(4)
    idx = torch.randperm(c2.rows, device="cuda", generator=g)[:c2.rows // 4].contiguous()
    assert idx.numel() // T_M // c2.tr.grid_per_net >= 7
    try:
        state = h.state(c2)
        k = h.kernel_update(c2, idx, h.mb_stats(idx, c2.b.returns, c2.b.active_masks), idx.numel())
        r64, r32 = _refs(c2, state, idx)
        compare(f"c2-mb4-shuffled-{idx.numel()}rows", (4, 2, 4), k, r64, r32, state, c2.cfg)
    finally:
        h.restore(c2, snap)


# ---------------------------------------------------------------- deliberate mistakes ---------------------------------

def _cta_tiles(tiles, G, cta=0):
    return list(range(cta, tiles, G))


def _tile_rows(t, limit):
    return torch.arange(t * T_M, min(t * T_M + T_M, limit), device="cuda")


@pytest.mark.parametrize("mutant", [m for m in ref.TC_MUTANTS if m != "dZ3-saturated"])   # dZ3-saturated: below
def test_c2_mutants_are_detected(c2, no_tf32, mutant):
    """The real kernel output on the C2 buffer against a float64 reference with one deliberate mistake: the block the
    mistake lands in must violate TAU x S (and pass it against the correct reference).  partial-tail-counted runs on the
    buffer's first rows - 127 rows, so that the last tile holds one minibatch row and 127 rows past the minibatch."""
    what, block = ref.TC_MUTANTS[mutant]
    rows_n = c2.rows - 127 if mutant == "partial-tail-counted" else c2.rows
    rows = torch.arange(rows_n, device="cuda")
    snap = h.snapshot(c2)
    try:
        state = h.state(c2)
        stats = c2.b.gae_stats[5:8] if rows_n == c2.rows else h.mb_stats(rows, c2.b.returns, c2.b.active_masks)
        k = h.kernel_update(c2, None, stats, rows_n)
    finally:
        h.restore(c2, snap)
    G, tiles = c2.tr.grid_per_net, -(-rows_n // T_M)
    mine = _cta_tiles(tiles, G)
    kw = {}
    if mutant == "cta-last-tile-dropped":
        kw = dict(remove_rows=_tile_rows(mine[-1], rows_n))
    elif mutant == "stale-staged-tile":
        kw = dict(remove_rows=_tile_rows(mine[-1], rows_n), add_rows=_tile_rows(mine[-2], rows_n))
    else:
        kw = dict(add_rows=torch.arange(rows_n, tiles * T_M, device="cuda"))
    r64 = ref.update(c2.cfg, c2.buf, state, rows, (4, 2, 4), vn_beta=c2.vn_beta)
    bad = ref.mutant_grad_pol(mutant, c2.cfg, c2.buf, state, rows, (4, 2, 4), r64, vn_beta=c2.vn_beta, **kw)
    name = block.split(".", 1)[1]
    s = ref.blocks((4, 2, 4), "pol")[name]
    S = float(r64["terms_pol"][name][1].norm())
    got = k["grad_pol"][s].double()
    e_good = float((got - r64["grad_pol"][s]).norm()) / S
    e_bad = float((got - bad[s]).norm()) / S
    print(f"\n  c2-{mutant} ({what}): {block} err/S against the reference {e_good:.2e}, against the mutant {e_bad:.2e} "
          f"= {e_bad / TAU:.1f} TAU")
    assert e_good <= TAU, f"{mutant}: the kernel fails the bar of {block} against the correct reference ({e_good:.3e})"
    assert e_bad > TAU, f"{mutant}: the mistake ({what}) passed the bar of {block}"


# ---------------------------------------------------------------- synthetic buffers -----------------------------------

def _launch(cfg, dims, buf, state, batch_rows, idx, row_begin, total, gae_stats, mb_stats, G=None):
    """OrlPpoArgs built by hand with ORL_PPO_TENSORCORE: fwdbwd, reduce, apply; what the comparison reads back."""
    lb, L = h.lib()
    d, n, dc = dims
    G = G or _sms()
    stride, gstride = L.orl_ppo_stride(d, dc, n), L.orl_ppo_grads_stride(d, dc, n)
    partials = torch.zeros(2 * G, stride, device="cuda")
    folded = torch.zeros(2, stride, device="cuda")
    grads = torch.zeros(2, gstride, device="cuda")
    dev = {k: state[k].clone() for k in ("pol", "cri", "pol_m", "pol_v", "cri_m", "cri_v", "vn")}
    steps = torch.tensor(state["steps"], dtype=torch.int32, device="cuda")
    lrs = torch.tensor([cfg.lr, cfg.critic_lr], dtype=torch.float32, device="cuda")
    train_info = torch.zeros(6, device="cuda")
    a = h.ppo_args(cfg, dims, lb.HEAD_CATEGORICAL, h.ppo_flags(cfg) | lb.PPO_TENSORCORE, G, buf, batch_rows, total, idx, row_begin,
                   (gae_stats, mb_stats), dev, steps, lrs, train_info, partials, folded, grads)
    s = lb.current_stream()
    lb.check(L.orl_ppo_fwdbwd(a, s), "orl_ppo_fwdbwd")
    lb.check(L.orl_ppo_reduce(a, s), "orl_ppo_reduce")
    lb.check(L.orl_ppo_apply(a, s), "orl_ppo_apply")
    torch.cuda.synchronize()
    return dict(grad_pol=grads[0, :dev["pol"].numel()], grad_cri=grads[1, :dev["cri"].numel()], losses=h.loss_sums(folded, stride),
                folded_losses=folded[:, stride - 8:].clone(), info=train_info, steps=[int(x) for x in steps], **dev)


def _setup(cfg, dims, batch_rows, contiguous_from=None, total=None, seed=0, net_edit=None):
    """A synthetic buffer (scale_harness.ppo_synthetic, Categorical head with action masks and active masks with zeros)
    and the minibatch: a shuffled index list, or a contiguous range from `contiguous_from`.
    net_edit(head, flat) edits the random nets before the buffer's log-probs and values are drawn from them."""
    total = total or batch_rows + 301
    idx, rows_idx = h.minibatch(total, batch_rows, contiguous_from, seed)
    buf, state = h.ppo_synthetic(cfg, dims, "categorical", total, rows_idx, seed, net_edit)
    return buf, state, idx, rows_idx, total


def _run(case, cfg, dims, batch_rows, contiguous_from=None, total=None, seed=0, net_edit=None, buf_edit=None):
    buf, state, idx, rows_idx, total = _setup(cfg, dims, batch_rows, contiguous_from, total, seed, net_edit)
    if buf_edit:
        buf_edit(buf, rows_idx)
    G = _sms()
    k = _launch(cfg, dims, buf, state, batch_rows, idx, contiguous_from or 0, total, h.gae_stats(buf),
                h.mb_stats(rows_idx.contiguous(), buf["returns"], buf["active_masks"]))
    r64 = ref.update(cfg, buf, state, rows_idx, dims, vn_beta=cfg.vn_beta)
    r32 = ffma_ref64.update(cfg, buf, state, rows_idx, dims, "categorical", torch.float32, vn_beta=cfg.vn_beta)
    tiles = -(-batch_rows // T_M)
    print(f"\n  {case}: {batch_rows} rows, {tiles} tiles, {G} CTAs per net, up to {-(-tiles // G)} tiles per CTA, "
          f"{'TMA-eligible contiguous range' if idx is None else 'index list'}")
    worst = compare(case, dims, k, r64, r32, state, cfg, check_vn=cfg.use_valuenorm)
    torch.cuda.empty_cache()
    return buf, state, rows_idx, k, r64, worst


def _rows(kind):
    G = _sms()
    return {"37": 37, "G": G * T_M, "3G+37": 3 * G * T_M + 37, "30G+37": 30 * G * T_M + 37}[kind]


# (name, dims (d, n, dc), activation_id, row counts): the NOUT templates 2, 5 and 8 (runtime n = 3, 8); ReLU (ACT = 1)
# and tanh / leaky ReLU / ELU (ACT = -1); d = 4 (float4 loads), 6 and 7 (scalar loads), 8; critic widths != policy widths
SYN = [("n2-relu-d4-dc4", (4, 2, 4), 1, ["37", "G", "3G+37", "30G+37"]),
       ("n5-tanh-d6-dc7", (6, 5, 7), 0, ["3G+37"]),
       ("n3-leaky-d7-dc6", (7, 3, 6), 2, ["3G+37"]),
       ("n8-elu-d8-dc4", (8, 8, 4), 3, ["G", "30G+37"])]
SYN_CASES = [(f"{name}-{rk}rows", dims, act, rk) for name, dims, act, rks in SYN for rk in rks]


@pytest.mark.parametrize("case,dims,act,rows_kind", SYN_CASES, ids=[c[0] for c in SYN_CASES])
def test_update_synthetic_edges(no_tf32, case, dims, act, rows_kind):
    """Shuffled minibatches (an index list into a larger buffer: gather staging) at every template and row-count edge."""
    cfg = types.SimpleNamespace(**{**BASE, "activation_id": act})
    _run(case, cfg, dims, _rows(rows_kind), seed=len(case) * 7 + dims[0])


@pytest.mark.parametrize("dims,act", [((4, 2, 4), 1), ((8, 5, 4), 0), ((7, 3, 6), 1)], ids=["d4-n2-tma", "d8-n5-tma", "d7-n3-scalar"])
def test_update_contiguous_range_not_at_row_zero(no_tf32, dims, act):
    """A contiguous range (indices == NULL) starting at row 1000 of a larger buffer, 3 G tiles + 37 rows: the TMA path
    for d % 4 == 0, the contiguous gather for d = 7."""
    rows = 3 * _sms() * T_M + 37
    cfg = types.SimpleNamespace(**{**BASE, "activation_id": act})
    _run(f"contiguous-from-1000-d{dims[0]}-n{dims[1]}-{rows}rows", cfg, dims, rows, contiguous_from=1000, total=rows + 1500,
         seed=dims[0])


# ---------------------------------------------------------------- staging paths and rows outside the minibatch --------

BUF_KEYS = ("policy_obs", "critic_obs", "actions", "action_log_probs", "advantages", "value_preds", "returns",
            "active_masks", "action_masks")


def _exact(case, dims, cfg, buf, state, rows, row_begin, total, gae, mb, idx):
    k = _launch(cfg, dims, buf, state, rows, idx, row_begin if idx is None else 0, total, gae, mb)
    return {key: (v.clone() if torch.is_tensor(v) else v) for key, v in k.items()}


def _same(a, b):
    return [key for key in a if not (torch.equal(a[key], b[key]) if torch.is_tensor(a[key]) else a[key] == b[key])]


def _staging_setup(dims):
    G = _sms()
    rows = 30 * G * T_M + 37
    begin, total = 1000, rows + 1500
    cfg = types.SimpleNamespace(**{**BASE, "activation_id": 1})
    buf, state, _, rows_idx, _ = _setup(cfg, dims, rows, contiguous_from=begin, total=total, seed=11 + dims[0])
    gae, mb = h.gae_stats(buf), h.mb_stats(rows_idx.contiguous(), buf["returns"], buf["active_masks"])
    return cfg, buf, state, rows, begin, total, gae, mb, rows_idx.contiguous()


STAGING_DIMS = [(4, 2, 4), (8, 5, 8)]


@pytest.mark.parametrize("dims", STAGING_DIMS, ids=["d4-n2", "d8-n5"])
def test_staging_paths_are_bit_identical(dims):
    """The same contiguous rows through the TMA path (indices == NULL) and through the gather path (indices = arange):
    the same tiles on the same CTAs with the same per-tile arithmetic, so gradients, loss slots, train_info and the
    updated state must be identical; so must two runs of the same call."""
    cfg, buf, state, rows, begin, total, gae, mb, ar = _staging_setup(dims)
    assert (rows // T_M) // _sms() >= 30 and rows % T_M
    tma = _exact("tma", dims, cfg, buf, state, rows, begin, total, gae, mb, None)
    tma2 = _exact("tma", dims, cfg, buf, state, rows, begin, total, gae, mb, None)
    gat = _exact("gather", dims, cfg, buf, state, rows, begin, total, gae, mb, ar)
    gat2 = _exact("gather", dims, cfg, buf, state, rows, begin, total, gae, mb, ar)
    print(f"\n  staging d={dims[0]}: TMA vs gather differ in {_same(tma, gat)}; reruns {_same(tma, tma2)} / {_same(gat, gat2)}")
    assert not _same(tma, tma2) and not _same(gat, gat2), "a rerun of the same update is not bit-identical"
    assert not _same(tma, gat), f"TMA and gather staging differ in {_same(tma, gat)}"


@pytest.mark.parametrize("poison", ["nan", "1e30"])
@pytest.mark.parametrize("dims", STAGING_DIMS, ids=["d4-n2", "d8-n5"])
def test_rows_outside_the_minibatch_never_matter(dims, poison):
    """Every buffer row outside the minibatch overwritten with NaN, or with +-1e30: both staging paths must give results
    bit-identical to the clean run (the minibatch moments are those of the clean buffer)."""
    cfg, buf, state, rows, begin, total, gae, mb, ar = _staging_setup(dims)
    clean = {p: _exact(p, dims, cfg, buf, state, rows, begin, total, gae, mb, i) for p, i in (("tma", None), ("gather", ar))}
    outside = torch.ones(total, dtype=torch.bool, device="cuda")
    outside[begin:begin + rows] = False
    for key in BUF_KEYS:
        if key in buf:
            x = buf[key]
            v = torch.full_like(x[:x.shape[0]], float("nan")) if poison == "nan" else \
                1e30 * torch.where(torch.rand_like(x) < 0.5, -1.0, 1.0)
            m = torch.zeros(x.shape[0], dtype=torch.bool, device="cuda")
            m[:min(total, x.shape[0])] = outside[:x.shape[0]]
            x[m] = v[m]
    bad = []
    for p, i in (("tma", None), ("gather", ar)):
        got = _exact(p, dims, cfg, buf, state, rows, begin, total, gae, mb, i)
        diff = _same(clean[p], got)
        print(f"\n  poison {poison} d={dims[0]} {p}: differs in {diff}; finite gradients: {bool(torch.isfinite(got['grad_pol']).all())}")
        if diff:
            bad.append(f"{p}: {diff}")
    assert not bad, f"rows outside the minibatch changed the update ({poison}): {bad}"


# ---------------------------------------------------------------- operand-scale edges ---------------------------------

def _few_active(share):
    def edit(buf, rows_idx):
        a = torch.zeros(rows_idx.numel(), 1, device="cuda")
        a[::share] = 1.0
        buf["active_masks"][rows_idx] = a
    return edit


def _big_adv(scale):
    def edit(buf, rows_idx):
        buf["advantages"].mul_(scale)
    return edit


def _fc3_scaled(factor, dims):
    """net_edit: the policy's fc3 weight and bias x factor, so that LayerNorm-3 sees a spread 1 / factor smaller."""
    def edit(head, flat):
        if head == "critic":
            return flat
        d, n, _ = dims
        bl = ffma_ref64.blocks(d, n, head)
        flat = flat.clone()
        for name in ("base.mlp.fc3.0.weight", "base.mlp.fc3.0.bias"):
            flat[bl[name]] *= factor
        return flat
    return edit


def _combine(*edits):
    def edit(buf, rows_idx):
        for e in edits:
            e(buf, rows_idx)
    return edit


SCALE_DIMS = (4, 2, 4)
SCALE_CASES = {
    "active-1/512": dict(buf_edit=_few_active(512)),
    "adv-1e3-unnormalised": dict(buf_edit=_big_adv(1e3)),
    "rstd3-1e2": dict(net_edit=_fc3_scaled(1e-2, SCALE_DIMS)),
    "combined": dict(buf_edit=_combine(_few_active(512), _big_adv(1e3)), net_edit=_fc3_scaled(1e-2, SCALE_DIMS)),
}


def _scaled_peaks(r64, state, live):
    sc = ref.net_operand_scales(state, SCALE_DIMS, "categorical", live)
    out = {}
    for net in ("pol", "cri"):
        sz, su = sc[net]
        p = r64["peaks"][net]
        out[net] = dict(dz3=p["dz3"] * sz, dz1=p["dz1"] * sz / 4, u=p["u"] * su, rstd3=p["rstd3"], sz=sz)
    return out


def _scale_case(case):
    rows = 3 * _sms() * T_M + 37
    cfg = types.SimpleNamespace(**BASE)
    kw = SCALE_CASES[case]
    buf, state, idx, rows_idx, total = _setup(cfg, SCALE_DIMS, rows, seed=5, net_edit=kw.get("net_edit"))
    if kw.get("buf_edit"):
        kw["buf_edit"](buf, rows_idx)
    r64 = ref.update(cfg, buf, state, rows_idx, SCALE_DIMS, vn_beta=cfg.vn_beta)
    live = float(buf["active_masks"][rows_idx].sum())
    # both nets run with their active-mask options on (BASE): the row weights divide by sum(active)
    assert cfg.use_policy_active_masks and cfg.use_value_active_masks
    peaks, by_rows = _scaled_peaks(r64, state, live), _scaled_peaks(r64, state, rows)
    for net in ("pol", "cri"):
        p, q = peaks[net], by_rows[net]
        print(f"\n  scale-{case} {net}: scaled peaks dZ3 {p['dz3']:.3e}  dZ1 {p['dz1']:.3e}  U {p['u']:.3e}  (limit {ref.FP16_MAX:.0f}; "
              f"scaled by the row count instead: dZ3 {q['dz3']:.3e}  U {q['u']:.3e}); max rstd3 {p['rstd3']:.2e}, "
              f"{live:.0f} of {rows} rows active")
    k = _launch(cfg, SCALE_DIMS, buf, state, rows, idx, 0, total, h.gae_stats(buf),
                h.mb_stats(rows_idx.contiguous(), buf["returns"], buf["active_masks"]))
    return cfg, buf, state, rows_idx, r64, k, peaks, by_rows


@pytest.mark.parametrize("case", list(SCALE_CASES))
def test_operand_scale_edges(no_tf32, case):
    """Backward operands pushed up against the split-fp16 range: few active rows (row weights active / sum(active)),
    large advantages with use_adv_normalize off (the advantages are still normalised over the active rows, as in
    ppo.py, so they end up at unit spread), a narrow LayerNorm-3 input (large rstd3), and all three at once.  Prints, per
    net, the float64 peaks of the scaled dZ3, dZ1 and U at the kernel's scales against 65504: none may reach it.  The
    combined case would exceed it if the scales followed the row count rather than sum(active)."""
    cfg, buf, state, rows_idx, r64, k, peaks, by_rows = _scale_case(case)
    for net in ("pol", "cri"):
        assert max(peaks[net]["dz3"], peaks[net]["dz1"], peaks[net]["u"]) < ref.FP16_MAX, (net, peaks[net])
    if case == "combined":
        assert max(by_rows["pol"]["dz3"], by_rows["pol"]["u"]) > ref.FP16_MAX, by_rows["pol"]
    r32 = ffma_ref64.update(cfg, buf, state, rows_idx, SCALE_DIMS, "categorical", torch.float32, vn_beta=cfg.vn_beta)
    compare(f"scale-{case}-{rows_idx.numel()}rows", SCALE_DIMS, k, r64, r32, state, cfg)


def test_saturated_dz3_mutant_is_detected(no_tf32):
    """dZ3-saturated: the combined operand-scale case with the policy's dZ3 clamped at 65504 at the scale the row count
    would give.  The kernel passes against the correct reference and the mutant violates TAU x S in fc3.0.weight."""
    cfg, buf, state, rows_idx, r64, k, peaks, by_rows = _scale_case("combined")
    what, block = ref.TC_MUTANTS["dZ3-saturated"]
    lim = ref.FP16_MAX / by_rows["pol"]["sz"]
    bad = ref.mutant_grad_pol("dZ3-saturated", cfg, buf, state, rows_idx, SCALE_DIMS, r64, vn_beta=cfg.vn_beta,
                              clamp_dz3={"pol": lim})
    name = block.split(".", 1)[1]
    s = ref.blocks(SCALE_DIMS, "pol")[name]
    S = float(r64["terms_pol"][name][1].norm())
    got = k["grad_pol"][s].double()
    e_good, e_bad = float((got - r64["grad_pol"][s]).norm()) / S, float((got - bad[s]).norm()) / S
    print(f"\n  dZ3-saturated ({what}): {block} err/S against the reference {e_good:.2e}, against the mutant {e_bad:.2e} "
          f"= {e_bad / TAU:.1f} TAU")
    assert e_good <= TAU and e_bad > TAU, (e_good, e_bad)
