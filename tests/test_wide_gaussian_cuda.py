"""DiagGaussian heads of 9..64 dimensions on the feed-forward policy (cfg.use_wide_gaussian_head,
ORL_HEAD_GAUSSIAN_WIDE): the host act (rollout_gaussian_wide_kernel), orl_policy_eval (policy_eval_gaussian_wide_kernel)
and the FFMA PPO update (ppo_fwdbwd_gaussian_wide_kernel).

Bars: the reference's traces (tests/golden/trace_wide_gaussian_{21,64}.npz) through PPOAgent over make()'s host vec-env
in parity mode, at the bars of the Gaussian traces (actions 1e-5, log-probs and values 2e-5, update scalars 2e-4,
parameters 2e-3); the Philox noise against the host Box-Muller of lanes 2 + 2k / 3 + 2k, dimensions 0..7 bit for bit
against ORL_HEAD_GAUSSIAN; the sampling moments and correlations of dimensions 8..63; the act and the eval against a
float64 forward row by row; the FFMA update at a C5-sized buffer (1024 envs x 128 steps) against float64 through
tests/scale_harness.py at PPO_FLOOR, with ffma_ref64's Gaussian mutants rejected; and the two host loops."""
import copy
import os
import types

import numpy as np
import pytest
import torch

import ffma_ref64 as ref
import scale_harness as h
from conftest import GOLDEN
from helpers import KEYS, make_agent, philox_units
from scale_harness import ATOL, CASES, PPO_FLOOR, Checker, no_tf32  # noqa: F401  (no_tf32: pytest fixture)
from wide_gaussian_oracle import TRACES, spaced_wide_gaussian_env

pytestmark = pytest.mark.gpu

OPT = ["--use_wide_gaussian_head", "true", "--use_wide_observations", "true"]
C5_ROWS = 1024 * 128
SEED, STEP = 0x2468_ACE0_1357, (1 << 32) + 5
LOG_SQRT_2PI = np.float32(0.9189385332046727)
ENTROPY_CONST = np.float32(1.4189385332046727)


def _make(n, d, N, flags):
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.common import make

    cls = spaced_wide_gaussian_env(d, n)
    return make("WideGaussianTarget", env_num=N, make_custom_envs=lambda id, env_num, render_mode=None, **kw: [cls for _ in range(env_num)],
                cfg=create_config_parser().parse_args(flags))


# ---------------------------------------------------------------- the reference's traces ------------------------------

@pytest.mark.parametrize("n", sorted(TRACES))
def test_wide_gaussian_reproduces_reference_trace(cuda, n):
    from openrl_b200 import lib

    d = np.load(os.path.join(GOLDEN, f"trace_wide_gaussian_{n}.npz"), allow_pickle=True)
    iters, N = int(d["meta/iters"]), int(d["meta/env_num"])
    flags = str(d["meta/flags"]).split() + ["--parity_mode", "true", "--log_interval", "1"] + OPT
    env = _make(n, TRACES[n], N, flags)
    cfg, net, agent = make_agent(env, flags, golden=d)
    drv, tr = agent.driver, agent.driver.trainer
    b = drv.buffer.data
    assert not tr.use_tensor_cores and tr.n == n and tr.head_kind == lib.HEAD_GAUSSIAN_WIDE
    for it in range(iters):
        t = f"it{it}"
        drv.episode = it
        drv.actor_rollout()
        np.testing.assert_allclose(b.actions.cpu().numpy(), d[f"{t}/actions"], rtol=1e-5, atol=1e-6, err_msg=t)
        np.testing.assert_allclose(b.rewards.cpu().numpy(), d[f"{t}/rewards"], rtol=1e-5, atol=1e-6, err_msg=t)
        assert np.array_equal(b.policy_obs.cpu().numpy(), d[f"{t}/policy_obs"]), t
        assert np.array_equal(b.masks.cpu().numpy(), d[f"{t}/masks"]), t
        np.testing.assert_allclose(b.action_log_probs.cpu().numpy(), d[f"{t}/action_log_probs"], rtol=0, atol=2e-5, err_msg=t)
        drv.compute_returns()
        np.testing.assert_allclose(b.value_preds.cpu().numpy()[:-1], d[f"{t}/value_preds"][:-1], rtol=0, atol=2e-5, err_msg=t)
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


# ---------------------------------------------------------------- the act and the eval --------------------------------

def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _module(d, n, wide=True, head_scale=5.0, zero_head=False):
    from openrl_b200 import spaces
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.modules.common import PPONet
    from oracle import loop

    class Env:
        agent_num, parallel_env_num = 1, 1
        observation_space, action_space = spaces.Box(-5, 5, (d,), np.float32), spaces.Box(-1, 1, (n,), np.float32)

        def reset(self, seed=None):
            return np.zeros((1, 1, d), np.float32)

    flags = ["--seed", "7"] + (OPT if wide else ["--use_wide_observations", "true"])
    cfg = create_config_parser().parse_args(flags)
    cfg.quiet = True
    module = PPONet(Env(), cfg=cfg, device="cuda:0").module
    sd = module.models["policy"].state_dict()
    if zero_head:   # the means are the bias (0): actions are the noise
        sd["act.action_out.fc_mean.weight"].zero_()
        sd["act.action_out.logstd._bias"].zero_()
    else:
        sd["act.action_out.fc_mean.weight"].mul_(head_scale)
        sd["act.action_out.logstd._bias"].copy_(torch.linspace(-0.5, 0.5, n).view(n, 1))
    return module, loop.cfg_from_flags(" ".join(flags[:2]))


def _params64(model):
    return {k: v.detach().cpu().double() for k, v in model.named_parameters()}


def _logstd(module):
    return module.models["policy"].state_dict()["act.action_out.logstd._bias"].cpu().numpy()[:, 0]


def _obs(rows, d, seed):
    return np.random.default_rng(seed).normal(size=(rows, d)).astype(np.float32)


def _box_muller(rows, n, seed=SEED, step=STEP):
    k = (n + 3) // 4
    u = philox_units(1, rows, seed, step, 0, tuple(range(2, 2 + 2 * k)))[0].astype(np.float64)   # (rows, 8k)
    u1 = np.concatenate([u[:, 8 * i:8 * i + 4] for i in range(k)], 1)
    u2 = np.concatenate([u[:, 8 * i + 4:8 * i + 8] for i in range(k)], 1)
    return (np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2))[:, :n]


ACT_SHAPES = [(d, n) for d in (9, 64, 65, 256) for n in (9, 21, 64)]


@pytest.mark.parametrize("d,n", ACT_SHAPES, ids=[f"d{d}-n{n}" for d, n in ACT_SHAPES])
def test_act_and_eval_match_float64(cuda, d, n):
    """The host act with a normal-noise table and deterministic, and orl_policy_eval, against a float64 forward row by
    row: 128 x SMs + 37 act rows (32 rows per CTA, a partial CTA, more than one wave) and 2 x SMs x 128 + 37 eval rows
    (CTAs walk two tiles, the last partial)."""
    from openrl_b200 import lib
    from oracle import nets

    module, ocfg = _module(d, n)
    pol = module.models["policy"]
    assert pol.head_kind == lib.HEAD_GAUSSIAN_WIDE
    p = _params64(pol)
    rows = 128 * _sm_count() + 37
    obs = _obs(rows, d, rows)
    noise = np.random.default_rng(rows + 1).normal(size=(rows, n)).astype(np.float32)
    act, logp = module.act(obs, exp_noise=noise)
    mean_d, logp_d = module.act(obs, deterministic=True)
    torch.cuda.synchronize()
    with torch.no_grad():
        want_act, want_logp = nets.policy_act_gaussian(p, ocfg, torch.from_numpy(obs).double(), normal_noise=torch.from_numpy(noise).double())
        mean, _ = nets.policy_act_gaussian(p, ocfg, torch.from_numpy(obs).double(), deterministic=True)
    np.testing.assert_allclose(act.cpu().numpy(), want_act.numpy(), rtol=0, atol=1e-5)
    np.testing.assert_allclose(logp.cpu().numpy(), want_logp.numpy(), rtol=0, atol=1e-5)
    np.testing.assert_allclose(mean_d.cpu().numpy(), mean.numpy(), rtol=0, atol=1e-5)
    want = np.broadcast_to(-_logstd(module) - LOG_SQRT_2PI, (rows, n))
    assert np.array_equal(logp_d.cpu().numpy().view(np.int32), want.view(np.int32))

    rows = 2 * _sm_count() * 128 + 37
    obs = _obs(rows, d, 7)
    with torch.no_grad():
        mean, _ = nets.policy_act_gaussian(p, ocfg, torch.from_numpy(obs).double(), deterministic=True)
    actions = (mean.numpy() + np.exp(_logstd(module)) * np.random.default_rng(rows).normal(size=(rows, n))).astype(np.float32)
    o, a = torch.from_numpy(obs).cuda(), torch.from_numpy(actions).cuda()
    lp = torch.empty(rows, n, device="cuda")
    ent = torch.empty(rows, n, device="cuda")
    lib.check(module._lib.orl_policy_eval(lib.ptr(pol.flat_params), d, n, pol.activation_id, lib.HEAD_GAUSSIAN_WIDE, lib.ptr(o),
                                          lib.ptr(a), None, lib.ptr(lp), lib.ptr(ent), rows, lib.current_stream()), "orl_policy_eval")
    torch.cuda.synchronize()
    with torch.no_grad():
        want_lp, _ = nets.policy_eval_gaussian(p, ocfg, torch.from_numpy(obs).double(), torch.from_numpy(actions).double())
    np.testing.assert_allclose(lp.cpu().numpy(), want_lp.numpy(), rtol=0, atol=1e-5)
    want = np.broadcast_to(ENTROPY_CONST + _logstd(module), (rows, n))
    assert np.array_equal(ent.cpu().numpy().view(np.int32), want.view(np.int32))
    # evaluate_actions: the (rows, n) log-probs and the entropy mean
    _, elp, e, _ = module.evaluate_actions(obs, obs, None, None, actions, None)
    np.testing.assert_allclose(elp.cpu().numpy(), want_lp.numpy(), rtol=0, atol=1e-5)
    np.testing.assert_allclose(float(e), float(want.astype(np.float64).mean()), rtol=1e-6)


@pytest.mark.parametrize("n", [9, 17, 64])
def test_philox_noise_is_box_muller_of_lanes_2_to_33(cuda, n):
    """With the means 0 and std 1 an action is its noise: dimensions [4k, 4k + 4) are Box-Muller of u1 from lane 2 + 2k
    and u2 from lane 3 + 2k; dimensions 0..7 are bit for bit those of a Box(8) row on ORL_HEAD_GAUSSIAN."""
    module, _ = _module(27, n, zero_head=True)
    rows = 64 * _sm_count() + 5
    obs = _obs(rows, 27, 5)
    act, _ = module.act(obs, rng_seed=SEED, rng_step=STEP)
    narrow, _ = _module(27, 8, wide=False, zero_head=True)
    act8, _ = narrow.act(obs, rng_seed=SEED, rng_step=STEP)
    torch.cuda.synchronize()
    got = act.cpu().numpy()
    np.testing.assert_allclose(got.astype(np.float64), _box_muller(rows, n), rtol=0, atol=1e-5)
    assert np.array_equal(got[:, :8].view(np.int32), act8.cpu().numpy().view(np.int32))


def test_sampling_statistics_of_dimensions_8_to_63(cuda):
    """Philox sampling of Box(64), 65536 rows x 4 steps: on dimensions 8..63 the first four moments of the noise are
    those of N(0, 1), and the correlations between dimensions and between consecutive steps of a row vanish, at the bars
    of tests/test_sampling_cuda.py's (5 standard errors)."""
    module, _ = _module(27, 64, zero_head=True)
    rows, T = 65536, 4
    obs = _obs(rows, 27, 11)
    x = np.stack([module.act(obs, rng_seed=SEED, rng_step=100 + t)[0].cpu().numpy() for t in range(T)]).astype(np.float64)
    e = x[..., 8:]                                 # (T, rows, 56)
    flat = e.reshape(-1)
    m = flat.size
    for k, want, se in ((1, 0.0, 1 / np.sqrt(m)), (2, 1.0, np.sqrt(2 / m)), (3, 0.0, np.sqrt(15 / m)), (4, 3.0, np.sqrt(96 / m))):
        got = (flat ** k).mean()
        assert abs(got - want) < 5 * se, (k, got)
    per_dim = e.reshape(-1, 56)
    c = np.corrcoef(per_dim, rowvar=False)
    off = c[~np.eye(56, dtype=bool)]
    assert np.abs(off).max() < 5 / np.sqrt(per_dim.shape[0]) * 1.5, np.abs(off).max()
    lag = (e[1:] * e[:-1]).mean(axis=(0, 1))          # consecutive steps of a row, per dimension
    assert np.abs(lag).max() < 5 / np.sqrt((T - 1) * rows), np.abs(lag).max()
    # dimension j against j + 1 within a lane group and across the lane pairs (j = 11 / 12, the edge of lanes 4 / 6)
    assert abs(np.corrcoef(per_dim[:, 3], per_dim[:, 4])[0, 1]) < 5 / np.sqrt(per_dim.shape[0])


# ---------------------------------------------------------------- the update against float64 -------------------------

def _grid():
    return max(1, _sm_count() // 2)


def _compare(case, dims, k, r64, r32, state, cfg):
    d, n, dc = dims
    chk = Checker(case, PPO_FLOOR)
    nets = (("pol", d, n, "gaussian"), ("cri", dc, 1, "critic"))
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
    return chk


def _kernel(cfg, dims, num_mini_batch, seed):
    """One FFMA update of a C5-sized synthetic buffer with a wide DiagGaussian head: the whole buffer (contiguous) or a
    shuffled 1 / num_mini_batch of it.  Returns the kernel's results and what the references need."""
    lb, L = h.lib()
    d, n, dc = dims
    G = _grid()
    total = C5_ROWS
    batch_rows = total // num_mini_batch
    idx, rows_idx = h.minibatch(total, batch_rows, None if num_mini_batch > 1 else 0, seed)
    buf, state = h.ppo_synthetic(cfg, dims, "gaussian", total, rows_idx, seed)
    stride, gstride = L.orl_ppo_stride(d, dc, n), L.orl_ppo_grads_stride(d, dc, n)
    partials = torch.zeros(2 * G, stride, device="cuda")
    folded = torch.zeros(2, stride, device="cuda")
    grads = torch.zeros(2, gstride, device="cuda")
    dev = {k: state[k].clone() for k in ("pol", "cri", "pol_m", "pol_v", "cri_m", "cri_v", "vn")}
    assert dev["pol"].numel() == L.orl_net_param_count(d, n) + n
    steps = torch.tensor(state["steps"], dtype=torch.int32, device="cuda")
    lrs = torch.tensor([cfg.lr, cfg.critic_lr], dtype=torch.float32, device="cuda")
    stats = h.gae_stats(buf), h.mb_stats(rows_idx.contiguous(), buf["returns"], buf["active_masks"])
    train_info = torch.zeros(6, device="cuda")
    a = h.ppo_args(cfg, dims, lb.HEAD_GAUSSIAN_WIDE, h.ppo_flags(cfg), G, buf, batch_rows, total, idx, 0, stats, dev, steps, lrs,
                   train_info, partials, folded, grads)
    s = lb.current_stream()
    lb.check(L.orl_ppo_fwdbwd(a, s), "orl_ppo_fwdbwd")
    lb.check(L.orl_ppo_reduce(a, s), "orl_ppo_reduce")
    lb.check(L.orl_ppo_apply(a, s), "orl_ppo_apply")
    torch.cuda.synchronize()
    k = dict(grad_pol=grads[0, :dev["pol"].numel()], grad_cri=grads[1, :dev["cri"].numel()], losses=h.loss_sums(folded, stride),
             info=train_info, steps=[int(x) for x in steps], **dev)
    return k, buf, state, rows_idx


def _run(case, cfg, dims, num_mini_batch, seed=0):
    k, buf, state, rows_idx = _kernel(cfg, dims, num_mini_batch, seed)
    r64, r32 = (ref.update(cfg, buf, state, rows_idx, dims, "gaussian", dt, vn_beta=cfg.vn_beta) for dt in (torch.float64, torch.float32))
    print(f"\n  {case}: {rows_idx.numel()} rows, {_grid()} CTAs per net")
    # logstd really moves: its gradient and update are not zero
    nb = ref.blocks(dims[0], dims[1], "gaussian")
    ls = [s for name, s in nb.items() if "logstd" in name][0]
    assert float(k["grad_pol"][ls].abs().max()) > 0 and not torch.equal(k["pol"][ls], state["pol"][ls])
    _compare(case, dims, k, r64, r32, state, cfg).done()
    torch.cuda.empty_cache()
    return k


WIDE = [(n, d) for n in (9, 12, 17, 21, 33, 38, 64) for d in (9, 64, 65, 256)]


@pytest.mark.parametrize("n,d", WIDE, ids=[f"n{n}-d{d}" for n, d in WIDE])
def test_wide_gaussian_update_matches_float64(no_tf32, n, d):
    """Every head width on both sides of the 4-wide blocks at obs widths 9, 64, 65 and 256 (the panelled fc1 and the
    shared-memory worst case), on a shuffled quarter of a C5-sized buffer."""
    cfg = types.SimpleNamespace(**h.BASE)
    _run(f"gauss-n{n}-d{d}-mb4", cfg, (d, n, d), 4, seed=n * 7 + d)


@pytest.mark.parametrize("n,d", [(9, 64), (21, 67), (64, 256)], ids=["n9-d64", "n21-d67", "n64-d256"])
def test_wide_gaussian_update_contiguous_and_rerun_bits(no_tf32, n, d):
    """The whole C5-sized buffer (contiguous, every CTA walks 15-16 tiles); a second run writes the same bits."""
    cfg = types.SimpleNamespace(**h.BASE)
    k1 = _run(f"gauss-n{n}-d{d}-contiguous", cfg, (d, n, d), 1, seed=n + d)
    k2, _, _, _ = _kernel(cfg, (d, n, d), 1, seed=n + d)
    for key in ("pol", "cri", "pol_m", "pol_v", "grad_pol", "losses"):
        assert torch.equal(k1[key], k2[key]), key


@pytest.mark.parametrize("masks", [True, False], ids=["policy-active-masks", "no-policy-active-masks"])
@pytest.mark.parametrize("flags", CASES, ids=[" ".join(c) or "default" for c in CASES])
def test_wide_gaussian_update_flag_sweep(no_tf32, flags, masks):
    """Every option of tests/test_ppo_flags_cuda.py at n = 21, d = 67, with and without policy active masks."""
    cfg = h.flag_cfg(flags)
    cfg.use_policy_active_masks = masks
    _run("gauss-n21-flags-" + ("-".join(flags) or "default") + ("" if masks else "-nopam"), cfg, (67, 21, 67), 4, seed=77)


@pytest.mark.parametrize("mutant", ["entropy-weight-1/rows", "one-ratio-per-row", "logstd-grad-without-entropy"])
def test_wide_gaussian_mutants_are_detected(no_tf32, mutant):
    """The kernel against a float64 reference with one deliberate mistake of ffma_ref64: the block the mistake lands in
    must violate its bar, and pass it against the correct reference."""
    _, what, opts, _ = ref.MUTANTS[mutant]
    cfg = types.SimpleNamespace(**{**h.BASE, **opts})
    dims = (67, 21, 67)
    k, buf, state, rows_idx = _kernel(cfg, dims, 4, seed=31)
    r64, r32 = (ref.update(cfg, buf, state, rows_idx, dims, "gaussian", dt, vn_beta=cfg.vn_beta) for dt in (torch.float64, torch.float32))
    bad = ref.update(cfg, buf, state, rows_idx, dims, "gaussian", torch.float64, vn_beta=cfg.vn_beta, mutant=mutant)
    net, name = what.split(" ")[1].split(".", 1)
    s = ref.blocks(67, 21 if net == "pol" else 1, "gaussian" if net == "pol" else "critic")[name]
    got, want, wrong, r32s = k["grad_" + net][s], r64["grad_" + net][s], bad["grad_" + net][s], r32["grad_" + net][s]
    good = Checker(f"gauss-{mutant}", PPO_FLOOR)
    good(what, got, want, r32s)
    good.done()
    e_bad, bar = h.rel(got, wrong), good.bar(h.rel(r32s, want))
    print(f"  gauss-{mutant}: kernel against the mutant {e_bad:.2e}, bar {bar:.2e}")
    assert e_bad > bar, f"{mutant}: the mistake ({ref.MUTANTS[mutant][0]}) passed the bar of {what}"


# ---------------------------------------------------------------- the host loops --------------------------------------

class _Host:
    """The reference's host vec-env duck type over a wide_gaussian_vec; `step_range` steps envs [lo, hi) only."""

    def __init__(self, inner):
        from openrl_b200 import spaces

        self.inner, self.parallel_env_num, self.agent_num = inner, inner.N, 1
        self.observation_space = spaces.Box(0.0, 1.0, (inner.obs_dim,), np.float32)
        self.action_space = spaces.Box(-1.0, 1.0, (inner.act_dim,), np.float32)

    def reset(self, seed=None):
        return self.inner.reset(seed=seed)

    def step(self, actions):
        return self.inner.step(actions)

    def step_range(self, lo, hi, actions):
        sub = copy.copy(self.inner)
        sub.N, sub.envs = hi - lo, self.inner.envs[lo:hi]
        return sub.step(actions)


def test_host_loops_agree(cuda):
    """1024 envs, T = 128, Box(21) at d = 67, Philox sampling: the synchronous and the two-group loop write the same bits
    over two iterations with an update between them."""
    from openrl_b200.envs.vec_env import HostVecEnv
    from wide_gaussian_oracle import wide_gaussian_vec

    N, T = 1024, 128
    flags = ["--seed", "3", "--episode_length", str(T), "--ppo_epoch", "1", "--num_mini_batch", "2", "--log_interval", "1"] + OPT
    runs, init = [], None
    for grouped in (False, True):
        env = HostVecEnv(_Host(wide_gaussian_vec(67, 21)(N)))
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
            bufs.append({k: getattr(b, k).cpu().numpy().copy() for k in ("actions", "action_log_probs", "policy_obs", "masks", "rewards")})
            assert bufs[-1]["actions"].shape[-1] == 21
            drv.compute_returns()
            torch.manual_seed(7)
            drv.trainer.train(b)
            b.after_update()
        runs.append(bufs)
    for it in range(2):
        for k in runs[0][it]:
            assert np.array_equal(runs[0][it][k], runs[1][it][k]), (it, k)


def test_three_agent_env_trains_and_evaluates(cuda):
    """A 3-agent host env with Box(12) actions (dm_control quadruped's width) runs through PPOAgent.train and
    evaluate_policy; without the option the same env is refused as before."""
    from openrl_b200 import spaces
    from openrl_b200.envs.vec_env import HostVecEnv
    from openrl_b200.utils.evaluation import evaluate_policy
    from openrl_b200.utils.logger import Logger

    class ThreeAgent:
        def __init__(self, N):
            self.parallel_env_num, self.agent_num = N, 3
            self.observation_space = spaces.Box(-np.inf, np.inf, (30,), np.float32)
            self.action_space = spaces.Box(-1.0, 1.0, (12,), np.float32)
            self.rng = np.random.default_rng(0)
            self.t = 0

        def reset(self, seed=None):
            self.t = 0
            return self.rng.random((self.parallel_env_num, 3, 30)).astype(np.float32)

        def step(self, actions):
            self.t += 1
            a = np.asarray(actions).reshape(self.parallel_env_num, 3, 12)
            r = -np.abs(a).mean(-1, keepdims=True)
            done = np.full((self.parallel_env_num, 3), self.t % 8 == 0)
            return (self.rng.random((self.parallel_env_num, 3, 30)).astype(np.float32), r, done,
                    [{} for _ in range(self.parallel_env_num)])

    flags = ["--seed", "1", "--episode_length", "16", "--ppo_epoch", "2", "--num_mini_batch", "2", "--log_interval", "1"]
    with pytest.raises(NotImplementedError, match="width up to 8"):
        make_agent(HostVecEnv(ThreeAgent(8)), flags, start=False)
    cfg, net, agent = make_agent(HostVecEnv(ThreeAgent(8)), flags + OPT, start=False)
    logger = Logger(quiet=True)
    agent.train(total_time_steps=16 * 8 * 3, logger=logger)
    got = [h_[1] for h_ in logger.history if "policy_loss" in h_[1]]
    assert got and all(np.isfinite(v) for row in got for v in row.values())
    out = evaluate_policy(agent, HostVecEnv(ThreeAgent(4)), n_eval_episodes=2)
    assert np.isfinite(np.asarray(out[0] if isinstance(out, tuple) else out, dtype=np.float64)).all()
