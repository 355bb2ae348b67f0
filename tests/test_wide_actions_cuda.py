"""Discrete action spaces of 9..64 actions on the feed-forward policy: the wide Categorical head of the host act
(rollout_kernel<*, ORL_ENV_NONE, 64>), of orl_policy_eval (policy_eval_wide_kernel) and of the FFMA PPO update
(ppo_fwdbwd_kernel<64, ...>).

Bars: the reference's traces on the masked env widened to 9 and 64 actions (tests/golden/trace_wide_actions_*.npz)
through PPOAgent over HostVecEnv in parity mode, at the bars of tests/test_host_action_masks_cuda.py; the FFMA update at
a C5-sized buffer (1024 envs x 128 steps) against float64 through tests/scale_harness.py at PPO_FLOOR, for head widths on
both sides of every 4-wide block edge, obs widths 9 and 64, one-legal-action and all-legal masks and every loss option at
n = 64; the act and the policy eval against a float64 forward row by row; and the sampler's first-max mode, legality at
1024 envs x 128 steps, the agreement of the two host loops and one fixed-seed chi-square test of its distribution."""
import copy
import os
import types

import numpy as np
import pytest
import torch

import ffma_ref64 as ref
import scale_harness as h
from conftest import GOLDEN
from helpers import KEYS, make_agent
from scale_harness import ATOL, CASES, PPO_FLOOR, Checker, no_tf32  # noqa: F401  (no_tf32: pytest fixture)
from wide_actions_oracle import WIDTHS, wide_target_vec

pytestmark = pytest.mark.gpu

C5_ROWS = 1024 * 128


class _Host:
    """The reference's host vec-env duck type over a MaskedTargetVec; `step_range` steps envs [lo, hi) only."""

    def __init__(self, inner):
        from openrl_b200 import spaces

        self.inner, self.parallel_env_num, self.agent_num = inner, inner.N, 1
        self.observation_space = spaces.Box(0.0, 1.0, (inner.obs_dim,), np.float32)
        self.action_space = spaces.Discrete(inner.n_actions)

    def reset(self, seed=None):
        return self.inner.reset(seed=seed), self.inner.last_infos

    def step(self, actions):
        return self.inner.step(actions)

    def step_range(self, lo, hi, actions):
        sub = copy.copy(self.inner)
        sub.N, sub.envs = hi - lo, self.inner.envs[lo:hi]
        out = sub.step(actions)
        if hi == self.inner.N:
            self.inner.calls += 1
        return out


def _host(n_envs, n_actions):
    from openrl_b200.envs.vec_env import HostVecEnv

    return HostVecEnv(_Host(wide_target_vec(n_actions)(n_envs)))


def _illegal(actions, action_masks):
    a = actions[..., 0].astype(np.int64)
    return int((np.take_along_axis(action_masks[:-1], a[..., None], axis=-1) == 0).sum())


# ---------------------------------------------------------------- the reference's traces ------------------------------

@pytest.mark.parametrize("n", WIDTHS)
def test_wide_actions_reproduce_reference_trace(cuda, n):
    d = np.load(os.path.join(GOLDEN, f"trace_wide_actions_{n}.npz"), allow_pickle=True)
    iters, N = int(d["meta/iters"]), int(d["meta/env_num"])
    flags = str(d["meta/flags"]).split() + ["--parity_mode", "true", "--log_interval", "1"]
    cfg, net, agent = make_agent(_host(N, n), flags, golden=d)
    drv = agent.driver
    b = drv.buffer.data
    assert not b.action_masks_trivial and not drv.trainer.use_tensor_cores and drv.trainer.n == n
    for it in range(iters):
        t = f"it{it}"
        drv.episode = it
        drv.actor_rollout()
        assert np.array_equal(b.actions.cpu().numpy(), d[f"{t}/actions"]), t
        assert np.array_equal(b.policy_obs.cpu().numpy(), d[f"{t}/policy_obs"]), t
        assert np.array_equal(b.masks.cpu().numpy(), d[f"{t}/masks"]), t
        assert np.array_equal(b.action_masks.cpu().numpy(), d[f"{t}/action_masks"]), t
        np.testing.assert_allclose(b.action_log_probs.cpu().numpy(), d[f"{t}/action_log_probs"], rtol=0, atol=2e-5)
        drv.compute_returns()
        np.testing.assert_allclose(b.value_preds.cpu().numpy()[:-1], d[f"{t}/value_preds"][:-1], rtol=0, atol=2e-5)
        info = drv.trainer.train(b)
        want = d[f"{t}/updates"].mean(axis=0)
        for col, name in enumerate(KEYS):
            np.testing.assert_allclose(info[name], want[col], rtol=2e-4, atol=1e-5, err_msg=f"{t} {name}")
        for mk in ("policy", "critic"):
            for k, v in net.module.models[mk].state_dict().items():
                gk = f"{t}/params/{mk}.{k}"
                if gk in d and "value_normalizer" not in k:
                    np.testing.assert_allclose(v.cpu().numpy(), d[gk], rtol=2e-3, atol=2e-5, err_msg=gk)
        b.after_update()


# ---------------------------------------------------------------- the update against float64 -------------------------

def _grid():
    return max(1, torch.cuda.get_device_properties(0).multi_processor_count // 2)


def _remask(cfg, dims, buf, state, rows_idx, masks, seed):
    """Replaces the synthetic buffer's action masks (`masks`: "one-legal" keeps only each row's action, "all-legal" all
    ones) and redraws the minibatch's old log-probs, value predictions and returns off every kink of the loss against
    the new masks, as ppo_synthetic draws them."""
    from oracle import nets

    d, n, dc = dims
    am = buf["action_masks"]
    if masks == "one-legal":
        am.zero_()
        am[torch.arange(am.shape[0], device="cuda"), buf["actions"][:, 0].long()] = 1.0
    else:
        am.fill_(1.0)
    g = torch.Generator(device="cuda").manual_seed(seed + 99)
    ncfg = types.SimpleNamespace(layer_N=1, activation_id=cfg.activation_id, use_recurrent_policy=False, use_policy_active_masks=True)
    pol = ref.unflatten(state["pol"].double(), d, n, "categorical")
    cri = ref.unflatten(state["cri"].double(), dc, 1, "critic")
    x = lambda k: buf[k].double()[rows_idx]   # noqa: E731
    with torch.no_grad():
        logp, _ = nets.policy_eval(pol, ncfg, x("policy_obs"), x("actions"), x("action_masks"))
        v, _ = nets.critic_forward(cri, ncfg, x("critic_obs"))
    h.draw_kink_free(g, cfg, state["vn"], logp, v, buf["action_log_probs"], rows_idx, buf["value_preds"], buf["returns"],
                     rows_idx, both_clip_sides=masks != "one-legal", huber_branches=True)


def _compare(case, dims, k, r64, r32, state, cfg):
    d, n, dc = dims
    chk = Checker(case, PPO_FLOOR)
    nets = (("pol", d, n, "categorical"), ("cri", dc, 1, "critic"))
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
    if cfg.use_valuenorm:
        chk("vn_state", k["vn"], r64["vn"], r32["vn"])
    assert k["steps"] == [r64["pol_step"], r64["cri_step"]]
    chk.done()


def _run(case, cfg, dims, num_mini_batch, masks=None, seed=0):
    """One FFMA update of a C5-sized synthetic buffer with a Categorical head of n = dims[1] actions: the whole buffer
    (contiguous) or a shuffled 1 / num_mini_batch of it, against the float64 and float32 references."""
    lb, L = h.lib()
    d, n, dc = dims
    G = _grid()
    total = C5_ROWS
    batch_rows = total // num_mini_batch
    idx, rows_idx = h.minibatch(total, batch_rows, None if num_mini_batch > 1 else 0, seed)
    buf, state = h.ppo_synthetic(cfg, dims, "categorical", total, rows_idx, seed)
    if masks:
        _remask(cfg, dims, buf, state, rows_idx, masks, seed)
    stride, gstride = L.orl_ppo_stride(d, dc, n), L.orl_ppo_grads_stride(d, dc, n)
    partials = torch.zeros(2 * G, stride, device="cuda")
    folded = torch.zeros(2, stride, device="cuda")
    grads = torch.zeros(2, gstride, device="cuda")
    dev = {k: state[k].clone() for k in ("pol", "cri", "pol_m", "pol_v", "cri_m", "cri_v", "vn")}
    assert dev["pol"].numel() == L.orl_net_param_count(d, n)
    steps = torch.tensor(state["steps"], dtype=torch.int32, device="cuda")
    lrs = torch.tensor([cfg.lr, cfg.critic_lr], dtype=torch.float32, device="cuda")
    stats = h.gae_stats(buf), h.mb_stats(rows_idx.contiguous(), buf["returns"], buf["active_masks"])
    train_info = torch.zeros(6, device="cuda")
    a = h.ppo_args(cfg, dims, lb.HEAD_CATEGORICAL, h.ppo_flags(cfg), G, buf, batch_rows, total, idx, 0, stats, dev, steps, lrs,
                   train_info, partials, folded, grads)
    s = lb.current_stream()
    lb.check(L.orl_ppo_fwdbwd(a, s), "orl_ppo_fwdbwd")
    lb.check(L.orl_ppo_reduce(a, s), "orl_ppo_reduce")
    lb.check(L.orl_ppo_apply(a, s), "orl_ppo_apply")
    torch.cuda.synchronize()
    k = dict(grad_pol=grads[0, :dev["pol"].numel()], grad_cri=grads[1, :dev["cri"].numel()], losses=h.loss_sums(folded, stride),
             info=train_info, steps=[int(x) for x in steps], **dev)
    r64, r32 = (ref.update(cfg, buf, state, rows_idx, dims, "categorical", dt, vn_beta=cfg.vn_beta)
                for dt in (torch.float64, torch.float32))
    print(f"\n  {case}: {batch_rows} rows, {-(-batch_rows // 128)} tiles, {G} CTAs per net")
    if masks == "one-legal":   # no policy gradient and no entropy: only the critic learns
        assert float(k["grad_pol"].abs().max()) == 0.0 and float(k["losses"][1]) == 0.0
    _compare(case, dims, k, r64, r32, state, cfg)
    torch.cuda.empty_cache()
    return k


WIDE = [(n, d) for n in (9, 12, 17, 33, 64) for d in (9, 64)]


@pytest.mark.parametrize("mb", [1, 4])
@pytest.mark.parametrize("n,d", WIDE, ids=[f"n{n}-d{d}" for n, d in WIDE])
def test_wide_update_matches_float64(no_tf32, n, d, mb):
    """Head widths on both sides of the 4-wide head blocks (JB = 3, 3, 5, 9, 16) at obs widths 9 and 64 (the largest
    shared-memory layout), on the whole C5-sized buffer (contiguous) and on a shuffled quarter of it."""
    cfg = types.SimpleNamespace(**h.BASE)
    _run(f"wide-n{n}-d{d}-mb{mb}", cfg, (d, n, d), mb, seed=n * 7 + d + mb)


@pytest.mark.parametrize("masks", ["one-legal", "all-legal"])
def test_wide_update_mask_edges(no_tf32, masks):
    """n = 64 with one legal action per row (no policy gradient, zero entropy) and with every action legal."""
    cfg = types.SimpleNamespace(**h.BASE)
    _run(f"wide-n64-d27-{masks}", cfg, (27, 64, 27), 4, masks=masks, seed=5)


@pytest.mark.parametrize("flags", CASES, ids=[" ".join(c) or "default" for c in CASES])
def test_wide_update_flag_sweep(no_tf32, flags):
    """Every option of tests/test_ppo_flags_cuda.py at n = 64, d = 27, on a shuffled quarter of the C5-sized buffer."""
    cfg = h.flag_cfg(flags)
    _run("wide-n64-flags-" + ("-".join(flags) or "default"), cfg, (27, 64, 27), 4, seed=77)


# ---------------------------------------------------------------- the act and the policy eval -------------------------

@pytest.fixture(scope="module")
def wide_agent():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    cfg, net, agent = make_agent(_host(16, 64), ["--seed", "9", "--episode_length", "8"])
    # larger head weights than the init's 0.01 gain, so that the softmax is far from uniform
    pol = net.module.models["policy"]
    with torch.no_grad():
        pol.state_dict()["act.action_out.linear.weight"].normal_(0.0, 0.5, generator=torch.Generator(device="cuda").manual_seed(1))
    return cfg, net, agent


def _rows64(rows, seed):
    rng = np.random.default_rng(seed)
    obs = rng.standard_normal((rows, 64)).astype(np.float32)
    m = (rng.random((rows, 64)) < 0.5).astype(np.float32)
    m[np.arange(rows), rng.integers(0, 64, rows)] = 1.0
    m[::7] = 1.0                       # some rows all legal
    m[3::11] = 0.0                     # and some with a single legal action
    m[np.arange(3, rows, 11), rng.integers(0, 64, len(range(3, rows, 11)))] = 1.0
    return obs, m


def _logits64(net, obs, m):
    from oracle import nets

    pol = net.module.models["policy"]
    p = ref.unflatten(pol.flat_params.double(), 64, 64, "categorical")
    ncfg = types.SimpleNamespace(layer_N=1, activation_id=pol.activation_id, use_recurrent_policy=False)
    with torch.no_grad():
        feat, _ = nets.policy_features(p, ncfg, torch.from_numpy(obs).cuda().double())
        return nets.categorical_logits(p, feat, torch.from_numpy(m).cuda().double())


def test_wide_act_and_eval_match_float64(wide_agent):
    """4096 rows at n = 64: the host act's log-probs of the actions it took and orl_policy_eval's log-probs and
    entropy of given actions against a float64 forward, row by row; the act takes legal actions only."""
    cfg, net, agent = wide_agent
    rows = 4096
    obs, m = _rows64(rows, 0)
    logits = _logits64(net, obs, m)
    logp64 = torch.log_softmax(logits, -1)
    acts, lp = net.module.act(obs, action_masks=m)
    a = acts[:, 0].long()
    assert (torch.from_numpy(m).cuda()[torch.arange(rows, device="cuda"), a] == 1).all()
    assert int(a.max()) >= 32
    np.testing.assert_allclose(lp[:, 0].cpu().numpy(), logp64.gather(-1, a[:, None])[:, 0].cpu().numpy(), rtol=0, atol=ATOL)
    given = np.random.default_rng(1).integers(0, 64, rows).astype(np.float32)
    _, elp, ent, _ = net.module.evaluate_actions(obs, obs, None, None, given, None, action_masks=m)
    p64 = logp64.exp()
    want_lp = logp64.gather(-1, torch.from_numpy(given).cuda().long()[:, None])[:, 0]
    legal = torch.from_numpy(m).cuda()[torch.arange(rows, device="cuda"), torch.from_numpy(given).cuda().long()] == 1
    # a masked-out given action sits at -6e4: compare those relative to their size
    np.testing.assert_allclose(elp[legal.cpu().numpy(), 0].cpu().numpy(), want_lp[legal].cpu().numpy(), rtol=0, atol=ATOL)
    np.testing.assert_allclose(elp[~legal.cpu().numpy(), 0].cpu().numpy(), want_lp[~legal].cpu().numpy(), rtol=1e-6, atol=0)
    want_ent = -(p64 * logp64).sum(-1).mean()
    np.testing.assert_allclose(float(ent), float(want_ent), rtol=0, atol=ATOL)


def test_wide_deterministic_act_picks_first_max(wide_agent):
    """Deterministic mode is the first maximum of the masked probabilities: rows with tied top logits (two legal
    actions with equal weights rows) take the lower index."""
    cfg, net, agent = wide_agent
    rows = 1024
    obs, m = _rows64(rows, 2)
    acts, _ = net.module.act(obs, action_masks=m, deterministic=True)
    want = _logits64(net, obs, m).float().argmax(-1)     # torch.argmax returns the first maximal index
    got = acts[:, 0].long()
    agree = (got == want).float().mean()
    assert float(agree) > 0.999, float(agree)
    # exact ties: copy row 40 of the head weights into row 50 and 20; a row whose top action is 40 must then pick 20
    pol = net.module.models["policy"]
    w = pol.state_dict()["act.action_out.linear.weight"]
    bias = pol.state_dict()["act.action_out.linear.bias"]
    saved = w.clone(), bias.clone()
    try:
        with torch.no_grad():
            w[20].copy_(w[40]); w[50].copy_(w[40]); bias[20] = bias[40]; bias[50] = bias[40]
        ones = np.ones_like(m)
        acts, _ = net.module.act(obs, action_masks=ones, deterministic=True)
        got = acts[:, 0].long().cpu().numpy()
        assert not ((got == 40) | (got == 50)).any()
        assert (got == 20).any()
    finally:
        with torch.no_grad():
            w.copy_(saved[0]); bias.copy_(saved[1])


def test_wide_sampling_matches_softmax_chi_square(wide_agent):
    """Philox sampling at n = 64: 200000 draws of one row (masks leave 48 legal actions) against its float64 softmax,
    one fixed-seed chi-square test over the legal actions with expected count >= 5."""
    from scipy import stats

    cfg, net, agent = wide_agent
    rows = 200000
    obs1, m1 = _rows64(8, 3)
    m1 = m1[:1].copy()
    m1[0] = 1.0
    m1[0, :16] = 0.0
    obs = np.repeat(obs1[:1], rows, axis=0)
    m = np.repeat(m1, rows, axis=0)
    acts, _ = net.module.act(obs, action_masks=m, rng_seed=12345, rng_step=0)
    counts = np.bincount(acts[:, 0].long().cpu().numpy(), minlength=64)
    assert counts[:16].sum() == 0
    p = torch.softmax(_logits64(net, obs1[:1], m1), -1)[0].cpu().numpy()
    exp = p * rows
    keep = exp >= 5
    assert keep.sum() > 10
    chi2 = ((counts[keep] - exp[keep]) ** 2 / exp[keep]).sum()
    pval = stats.chi2.sf(chi2, int(keep.sum()) - 1)
    print(f"\n  chi-square {chi2:.1f} over {int(keep.sum())} actions, p = {pval:.3f}")
    assert pval > 1e-3, (chi2, pval)


def test_wide_host_loops_legal_and_agree(cuda):
    """1024 envs, T = 128, n = 64, Philox sampling: no illegal action in either host loop, and the synchronous and the
    two-group loop write the same bits over two iterations with an update between them."""
    N, T = 1024, 128
    flags = ["--seed", "3", "--episode_length", str(T), "--ppo_epoch", "1", "--num_mini_batch", "2", "--log_interval", "1"]
    runs, init = [], None
    for grouped in (False, True):
        env = _host(N, 64)
        assert env.supports_groups
        cfg, net, agent = make_agent(env, flags + ["--host_env_groups", "true" if grouped else "false"], like=init)
        if init is None:
            init = {mk: {k: v.clone() for k, v in net.module.models[mk].state_dict().items()} for mk in ("policy", "critic")}
        drv, b = agent.driver, agent.driver.buffer.data
        env.env.inner.reset(seed=11)
        drv.reset_and_buffer_init()
        bufs = []
        for it in range(2):
            drv.episode = it
            drv.actor_rollout()
            torch.cuda.synchronize()
            bufs.append({k: getattr(b, k).cpu().numpy().copy()
                         for k in ("actions", "action_log_probs", "policy_obs", "masks", "rewards", "action_masks")})
            assert _illegal(bufs[-1]["actions"], bufs[-1]["action_masks"]) == 0
            assert (bufs[-1]["action_masks"] == 0).mean() > 0.2 and bufs[-1]["actions"].max() >= 56
            drv.compute_returns()
            torch.manual_seed(7)
            drv.trainer.train(b)
            b.after_update()
        runs.append(bufs)
    for it in range(2):
        for k in runs[0][it]:
            assert np.array_equal(runs[0][it][k], runs[1][it][k]), (it, k)
