"""Observations of 65..256 features on the feed-forward policy and critic (cfg.use_wide_observations): fc1 as a loop over
64-wide panels of the observation (orl_mlp.cuh, fc1_panels) in the host act (rollout_kernel<*, ORL_ENV_NONE, *, true>),
orl_critic_values (critic_values_kernel<true>), orl_policy_eval (policy_eval_kernel<true>, policy_eval_wide_kernel<true>)
and the FFMA PPO update (the panelled ppo_fwdbwd_kernel<NB, PANELS_POLICY, PANELS_CRITIC> instances), and the insert of a critic
section wider than 64 (orl_host_insert_wide_obs).

Bars: the reference's traces on the envs of tests/wide_obs_oracle.py through PPOAgent in parity mode; the FFMA update on a shuffled minibatch of a C5-sized buffer (1024 envs x 128 steps) with a partial last tile,
against float64 through tests/scale_harness.py at PPO_FLOOR, at widths on both sides of every panel edge, with either
net wide, with the wide head, at the shared-memory worst case (d = dc = 256, n = 64), with a Gaussian head and under
every loss option; the act, the values and the policy eval against a float64 forward row by row, at the larger of
ATOL and RATIO x the float32 forward's error (the host act at each of its row tiles); the insert bit for bit against its rule; a SMAC-8m-shaped env through
PPOAgent.train in both host loops; and bit-identical parameters from two identical updates."""
import types

import numpy as np
import pytest
import torch

import ffma_ref64 as ref
import scale_harness as h
from helpers import make_agent
from scale_harness import ATOL, CASES, PPO_FLOOR, RATIO, Checker, no_tf32  # noqa: F401  (no_tf32: pytest fixture)

pytestmark = pytest.mark.gpu

C5_ROWS = 1024 * 128
MB_ROWS = C5_ROWS // 4 - 91   # a shuffled quarter of the buffer less 91 rows: 255 full tiles and one of 37 rows
WIDE_FLAGS = ["--use_wide_observations", "true"]


class _DictHost:
    """A agents per env, Dict {"policy": Box(d), "critic": Box(dc)} observations ~ N(0, 1), Discrete(n) with per-agent
    (A, n) masks, an env finishing with probability 0.15 per step.  Every draw is keyed by (env, the env's step count),
    so a sub-range step (`step_range`) returns what the whole-range step would."""

    def __init__(self, n, A=8, d=80, dc=168, n_act=14):
        from openrl_b200 import spaces

        box = lambda w: spaces.Box(-np.inf, np.inf, (w,), np.float32)  # noqa: E731
        self.parallel_env_num, self.agent_num, self.d, self.dc, self.n_act = n, A, d, dc, n_act
        self.observation_space = spaces.Dict({"policy": box(d), "critic": box(dc)})
        self.action_space = spaces.Discrete(n_act)
        self.t, self.masks = np.zeros(n, np.int64), {}

    def _draw(self, e):
        g = np.random.default_rng((11, e, int(self.t[e])))
        A = self.agent_num
        pol = g.standard_normal((A, self.d)).astype(np.float32)
        cri = g.standard_normal((A, self.dc)).astype(np.float32)
        m = (g.random((A, self.n_act)) < 0.6).astype(np.int8)
        m[np.arange(A), g.integers(0, self.n_act, A)] = 1
        self.masks[e] = m
        return pol, cri, m, g.random() < 0.15, g.standard_normal((A, 1))

    def _out(self, lo, hi):
        draws = [self._draw(e) for e in range(lo, hi)]
        obs = {"policy": np.stack([x[0] for x in draws]), "critic": np.stack([x[1] for x in draws])}
        dones = np.repeat(np.array([x[3] for x in draws])[:, None], self.agent_num, axis=1)
        return obs, np.stack([x[4] for x in draws]), dones, [{"action_masks": x[2]} for x in draws]

    def reset(self, seed=None):
        self.t[:] = 0
        obs, _, _, infos = self._out(0, self.parallel_env_num)
        return obs, infos

    def step(self, actions):
        return self.step_range(0, self.parallel_env_num, actions)

    def step_range(self, lo, hi, actions):
        acts = np.asarray(actions).reshape(hi - lo, self.agent_num)
        for i, e in enumerate(range(lo, hi)):   # the env checks its actions against the masks it reported
            assert (self.masks[e][np.arange(self.agent_num), acts[i]] == 1).all(), "illegal action"
        self.t[lo:hi] += 1
        return self._out(lo, hi)


class _BoxHost:
    """One agent per env, flat Box(d) observations ~ N(0, 1), Box(4) actions (a DiagGaussian head)."""

    def __init__(self, n, d):
        from openrl_b200 import spaces

        self.parallel_env_num, self.agent_num, self.d = n, 1, d
        self.observation_space = spaces.Box(-np.inf, np.inf, (d,), np.float32)
        self.action_space = spaces.Box(-1, 1, (4,), np.float32)
        self.rng = np.random.default_rng(0)

    def reset(self, seed=None):
        return self.rng.standard_normal((self.parallel_env_num, 1, self.d)).astype(np.float32)

    def step(self, actions):
        n = self.parallel_env_num
        return (self.rng.standard_normal((n, 1, self.d)).astype(np.float32), self.rng.standard_normal((n, 1, 1)),
                self.rng.random((n, 1)) < 0.05, [{} for _ in range(n)])


# ---------------------------------------------------------------- the reference's traces ------------------------------

@pytest.mark.parametrize("tag", ["wide_obs_dict", "wide_obs_box_256"])
def test_wide_obs_reproduce_reference_trace(cuda, tag):
    """PPOAgent over make()'s host vec-env in parity mode against the reference's runs on the envs of
    tests/wide_obs_oracle.py: SMAC 8m's shapes (Dict 80 / 168, Discrete(14)) and Box(256) observations with a Box(4)
    DiagGaussian head.  Categorical actions bit for bit; Gaussian actions (mean + std * noise, the mean a 256-term
    float32 sum in another order than torch's) and the rewards computed from them at the bars of
    tests/test_gaussian_cuda.py; log-probs and values 2e-5, the update scalars 2e-4, parameters 2e-3."""
    import os

    from conftest import GOLDEN
    from helpers import KEYS
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.common import make
    from wide_obs_oracle import SpacedWideBoxTargetEnv, SpacedWideDictTargetEnv

    d = np.load(os.path.join(GOLDEN, f"trace_{tag}.npz"), allow_pickle=True)
    iters, N = int(d["meta/iters"]), int(d["meta/env_num"])
    flags = str(d["meta/flags"]).split() + ["--parity_mode", "true", "--log_interval", "1"] + WIDE_FLAGS
    dict_obs = tag == "wide_obs_dict"
    cls = SpacedWideDictTargetEnv if dict_obs else SpacedWideBoxTargetEnv
    env = make("WideTarget", env_num=N, make_custom_envs=lambda id, env_num, render_mode=None, **kw: [cls for _ in range(env_num)],
               cfg=create_config_parser().parse_args(flags))
    assert (env.obs_dim, env.critic_obs_dim) == ((80, 168) if dict_obs else (256, 256))
    cfg, net, agent = make_agent(env, flags, golden=d)
    drv, tr = agent.driver, agent.driver.trainer
    b = drv.buffer.data
    assert not tr.use_tensor_cores and tr.n == (14 if dict_obs else 4)
    for it in range(iters):
        t = f"it{it}"
        drv.episode = it
        drv.actor_rollout()
        if dict_obs:
            assert np.array_equal(b.actions.cpu().numpy(), d[f"{t}/actions"]), t
            assert np.array_equal(b.critic_obs.cpu().numpy(), d[f"{t}/critic_obs"]), t
            assert np.array_equal(b.rewards.cpu().numpy(), d[f"{t}/rewards"]), t
        else:
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


# ---------------------------------------------------------------- the update against float64 -------------------------

def _grid():
    return max(1, torch.cuda.get_device_properties(0).multi_processor_count // 2)


def _remask(cfg, dims, buf, state, rows_idx, masks, seed):
    """Replaces the synthetic buffer's action masks ("one-legal": only each row's action, "all-legal": all ones) and
    redraws the minibatch's old log-probs, value predictions and returns off every kink of the loss against them."""
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


def _compare(case, dims, head, k, r64, r32, state, cfg):
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
    if cfg.use_valuenorm:
        chk("vn_state", k["vn"], r64["vn"], r32["vn"])
    assert k["steps"] == [r64["pol_step"], r64["cri_step"]]
    chk.done()


def _kernel(cfg, dims, head, buf, state, idx, rows_idx, batch_rows):
    """One FFMA update (fwdbwd + reduce + apply) from `state` on the synthetic buffer; the kernel's outputs."""
    lb, L = h.lib()
    d, n, dc = dims
    G = _grid()
    gauss = head == "gaussian"
    stride, gstride = L.orl_ppo_stride(d, dc, n), L.orl_ppo_grads_stride(d, dc, n)
    partials = torch.full((2 * G, stride), float("nan"), device="cuda")   # every element the kernel reads it writes first
    folded = torch.zeros(2, stride, device="cuda")
    grads = torch.zeros(2, gstride, device="cuda")
    dev = {k: state[k].clone() for k in ("pol", "cri", "pol_m", "pol_v", "cri_m", "cri_v", "vn")}
    assert dev["pol"].numel() == L.orl_net_param_count(d, n) + (n if gauss else 0)
    steps = torch.tensor(state["steps"], dtype=torch.int32, device="cuda")
    lrs = torch.tensor([cfg.lr, cfg.critic_lr], dtype=torch.float32, device="cuda")
    stats = h.gae_stats(buf), h.mb_stats(rows_idx.contiguous(), buf["returns"], buf["active_masks"])
    train_info = torch.zeros(6, device="cuda")
    a = h.ppo_args(cfg, dims, lb.HEAD_GAUSSIAN if gauss else lb.HEAD_CATEGORICAL, h.ppo_flags(cfg), G, buf, batch_rows,
                   C5_ROWS, idx, 0, stats, dev, steps, lrs, train_info, partials, folded, grads)
    s = lb.current_stream()
    lb.check(L.orl_ppo_fwdbwd(a, s), "orl_ppo_fwdbwd")
    lb.check(L.orl_ppo_reduce(a, s), "orl_ppo_reduce")
    lb.check(L.orl_ppo_apply(a, s), "orl_ppo_apply")
    torch.cuda.synchronize()
    return dict(grad_pol=grads[0, :dev["pol"].numel()], grad_cri=grads[1, :dev["cri"].numel()], losses=h.loss_sums(folded, stride),
                info=train_info, steps=[int(x) for x in steps], **dev)


def _run(case, cfg, dims, head="categorical", masks=None, seed=0):
    """One FFMA update of a shuffled MB_ROWS-row minibatch of a C5-sized synthetic buffer against the float64 and
    float32 references."""
    idx, rows_idx = h.minibatch(C5_ROWS, MB_ROWS, None, seed)
    buf, state = h.ppo_synthetic(cfg, dims, head, C5_ROWS, rows_idx, seed)
    if masks:
        _remask(cfg, dims, buf, state, rows_idx, masks, seed)
    k = _kernel(cfg, dims, head, buf, state, idx, rows_idx, MB_ROWS)
    r64, r32 = (ref.update(cfg, buf, state, rows_idx, dims, head, dt, vn_beta=cfg.vn_beta) for dt in (torch.float64, torch.float32))
    print(f"\n  {case}: {MB_ROWS} rows, {-(-MB_ROWS // 128)} tiles, {_grid()} CTAs per net")
    if masks == "one-legal":   # no policy gradient and no entropy: only the critic learns
        assert float(k["grad_pol"].abs().max()) == 0.0 and float(k["losses"][1]) == 0.0
    _compare(case, dims, head, k, r64, r32, state, cfg)
    torch.cuda.empty_cache()


PANEL_EDGES = (65, 68, 127, 128, 129, 192, 255, 256)


@pytest.mark.parametrize("d", PANEL_EDGES)
def test_update_at_panel_edges(no_tf32, d):
    """d = dc on both sides of each 64-column panel edge (one to four panels, partial last panels of 1, 4, 63 and 64
    columns), a Categorical head of 5 actions."""
    cfg = types.SimpleNamespace(**h.BASE)
    _run(f"panels-d{d}-dc{d}-n5", cfg, (d, 5, d), seed=d)


@pytest.mark.parametrize("dims", [(200, 5, 40), (18, 5, 216)], ids=["policy-wide", "critic-wide"])
def test_update_one_net_wide(no_tf32, dims):
    """One net panelled and the other one narrow in the same launch: a 200-wide policy with a 40-wide critic, and the
    simple_spread-with-6-agents shape (policy 18, critic 216)."""
    cfg = types.SimpleNamespace(**h.BASE)
    _run(f"mixed-d{dims[0]}-dc{dims[2]}", cfg, dims, seed=dims[0])


@pytest.mark.parametrize("masks", [None, "one-legal", "all-legal"])
def test_update_smac_8m_shape(no_tf32, masks):
    """SMAC 8m's shapes (observation 80, state 168, 14 actions): both nets panelled and the wide head, with random,
    one-legal and all-legal masks."""
    cfg = types.SimpleNamespace(**h.BASE)
    _run(f"8m-d80-dc168-n14-{masks or 'random'}", cfg, (80, 14, 168), masks=masks, seed=8)


def test_update_shared_memory_worst_case(no_tf32):
    """d = dc = 256 with a 64-action head: the largest shared-memory layout of the update."""
    cfg = types.SimpleNamespace(**h.BASE)
    _run("worst-d256-dc256-n64", cfg, (256, 64, 256), seed=64)


def test_update_gaussian_head(no_tf32):
    """A DiagGaussian head of 8 outputs at d = dc = 256."""
    cfg = types.SimpleNamespace(**h.BASE)
    _run("gauss-d256-dc256-n8", cfg, (256, 8, 256), head="gaussian", seed=3)


@pytest.mark.parametrize("flags", CASES, ids=[" ".join(c) or "default" for c in CASES])
def test_update_flag_sweep(no_tf32, flags):
    """Every option of tests/test_ppo_flags_cuda.py at SMAC 8m's shapes."""
    cfg = h.flag_cfg(flags)
    _run("8m-flags-" + ("-".join(flags) or "default"), cfg, (80, 14, 168), seed=77)


def test_update_is_deterministic(no_tf32):
    """Two identical updates at d = dc = 256 give bit-identical parameters, Adam moments and loss sums."""
    cfg = types.SimpleNamespace(**h.BASE)
    dims = (256, 14, 256)
    idx, rows_idx = h.minibatch(C5_ROWS, MB_ROWS, None, 5)
    buf, state = h.ppo_synthetic(cfg, dims, "categorical", C5_ROWS, rows_idx, 5)
    k1 = _kernel(cfg, dims, "categorical", buf, state, idx, rows_idx, MB_ROWS)
    k2 = _kernel(cfg, dims, "categorical", buf, state, idx, rows_idx, MB_ROWS)
    for key in ("pol", "cri", "pol_m", "pol_v", "cri_m", "cri_v", "grad_pol", "grad_cri", "losses", "info"):
        assert torch.equal(k1[key], k2[key]), key
    assert bool(torch.isfinite(k1["pol"]).all()) and bool(torch.isfinite(k1["cri"]).all())


# ---------------------------------------------------------------- the act, the values and the policy eval -------------

def _forward_bar(what, got, r64, r32):
    """Element-wise: the kernel's largest error against float64 at most the larger of ATOL and RATIO x float32's."""
    ek = float((got.double() - r64).abs().max())
    e32 = float((r32.double() - r64).abs().max())
    bar = max(ATOL, RATIO * e32)
    print(f"  {what:40s} kernel {ek:9.2e}  fp32 {e32:9.2e}  bar {bar:9.2e}")
    assert ek <= bar, f"{what}: kernel {ek:.3e} > bar {bar:.3e}"


FORWARD = [(65, 65), (128, 80), (129, 168), (256, 256), (18, 216)]


@pytest.mark.parametrize("d,dc", FORWARD, ids=[f"d{d}-dc{dc}" for d, dc in FORWARD])
@pytest.mark.parametrize("n", [5, 14])
def test_categorical_forwards_match_float64(cuda, d, dc, n):
    """4133 rows (a partial last tile) of a Dict env: orl_critic_values, the host act (deterministic: the first
    maximum, and its log-prob) and orl_policy_eval (log-probs and entropy of given actions) against a float64 forward
    of the oracle nets, for the narrow (5) and the wide (14) Categorical head."""
    from oracle import nets

    rows = 4133
    cfg, net, agent = make_agent(_DictHost(4, A=1, d=d, dc=dc, n_act=n), WIDE_FLAGS + ["--seed", str(d)], start=False)
    pol, cri = net.module.models["policy"], net.module.models["critic"]
    with torch.no_grad():   # head weights far from the init's 0.01 gain, so that the softmax is far from uniform
        pol.state_dict()["act.action_out.linear.weight"].normal_(0.0, 0.5, generator=torch.Generator(device="cuda").manual_seed(1))
    rng = np.random.default_rng(d + dc)
    obs = rng.standard_normal((rows, d)).astype(np.float32)
    cobs = rng.standard_normal((rows, dc)).astype(np.float32)
    m = (rng.random((rows, n)) < 0.6).astype(np.float32)
    m[np.arange(rows), rng.integers(0, n, rows)] = 1.0
    ncfg = types.SimpleNamespace(layer_N=1, activation_id=pol.activation_id, use_recurrent_policy=False)

    def fwd(dt):
        p = ref.unflatten(pol.flat_params.to(dt), d, n, "categorical")
        c = ref.unflatten(cri.flat_params.to(dt), dc, 1, "critic")
        with torch.no_grad():
            feat, _ = nets.policy_features(p, ncfg, torch.from_numpy(obs).cuda().to(dt))
            logits = nets.categorical_logits(p, feat, torch.from_numpy(m).cuda().to(dt))
            v, _ = nets.critic_forward(c, ncfg, torch.from_numpy(cobs).cuda().to(dt))
        return torch.log_softmax(logits, -1), v

    lp64, v64 = fwd(torch.float64)
    lp32, v32 = fwd(torch.float32)
    _forward_bar(f"values d{d} dc{dc}", net.module.get_values(cobs)[:, 0], v64[:, 0], v32[:, 0])

    acts, lp = net.module.act(obs, action_masks=m, deterministic=True)
    a = acts[:, 0].long()
    assert (torch.from_numpy(m).cuda()[torch.arange(rows, device="cuda"), a] == 1).all()
    # the first maximum up to rounding: the float64 log-prob of the chosen action is the row's largest
    assert float((lp64.max(-1).values - lp64.gather(-1, a[:, None])[:, 0]).max()) < 1e-4
    _forward_bar(f"act log-probs d{d} n{n}", lp[:, 0], lp64.gather(-1, a[:, None])[:, 0], lp32.gather(-1, a[:, None])[:, 0].double())

    given = torch.from_numpy(rng.integers(0, n, rows).astype(np.float32)).cuda()
    legal = torch.from_numpy(m).cuda()[torch.arange(rows, device="cuda"), given.long()] == 1
    _, elp, ent, _ = net.module.evaluate_actions(cobs, obs, None, None, given.cpu().numpy()[:, None], None, action_masks=m)
    g = given.long()[:, None]
    _forward_bar(f"eval log-probs d{d} n{n}", elp[legal, 0], lp64.gather(-1, g)[legal, 0], lp32.gather(-1, g)[legal, 0])
    ent64 = -(lp64.exp() * lp64).sum(-1).mean()
    ent32 = -(lp32.exp() * lp32).sum(-1).mean()
    _forward_bar(f"eval entropy d{d} n{n}", ent.reshape(1), ent64.reshape(1), ent32.reshape(1))


@pytest.mark.parametrize("rows_per_cta", [16, 32])
@pytest.mark.parametrize("n", [5, 14])
def test_host_act_row_tiles(cuda, rows_per_cta, n):
    """The host act's instances of 16 and 32 rows per CTA (orl_rollout picks them when the batch has at least 16 resp.
    32 rows for each of 4 CTAs per SM) at d = 200: deterministic actions are the float64 first maximum up to rounding,
    legal, and their log-probs match float64."""
    from oracle import nets

    want = 4 * torch.cuda.get_device_properties(0).multi_processor_count
    rows = rows_per_cta * want + 37          # enough rows for this tile size, too few for the next one
    d = 200
    cfg, net, agent = make_agent(_DictHost(4, A=1, d=d, dc=40, n_act=n), WIDE_FLAGS + ["--seed", "4"], start=False)
    pol = net.module.models["policy"]
    with torch.no_grad():
        pol.state_dict()["act.action_out.linear.weight"].normal_(0.0, 0.5, generator=torch.Generator(device="cuda").manual_seed(2))
    rng = np.random.default_rng(rows)
    obs = rng.standard_normal((rows, d)).astype(np.float32)
    m = (rng.random((rows, n)) < 0.6).astype(np.float32)
    m[np.arange(rows), rng.integers(0, n, rows)] = 1.0
    ncfg = types.SimpleNamespace(layer_N=1, activation_id=pol.activation_id, use_recurrent_policy=False)

    def logp(dt):
        p = ref.unflatten(pol.flat_params.to(dt), d, n, "categorical")
        with torch.no_grad():
            feat, _ = nets.policy_features(p, ncfg, torch.from_numpy(obs).cuda().to(dt))
            return torch.log_softmax(nets.categorical_logits(p, feat, torch.from_numpy(m).cuda().to(dt)), -1)

    lp64, lp32 = logp(torch.float64), logp(torch.float32)
    acts, lp = net.module.act(obs, action_masks=m, deterministic=True)
    a = acts[:, 0].long()
    assert (torch.from_numpy(m).cuda()[torch.arange(rows, device="cuda"), a] == 1).all()
    assert float((lp64.max(-1).values - lp64.gather(-1, a[:, None])[:, 0]).max()) < 1e-4
    _forward_bar(f"act log-probs {rows} rows n{n}", lp[:, 0], lp64.gather(-1, a[:, None])[:, 0],
                 lp32.gather(-1, a[:, None])[:, 0].double())


@pytest.mark.parametrize("d", [65, 129, 256])
def test_gaussian_forwards_match_float64(cuda, d):
    """4133 rows of a Box(d) env with Box(4) actions: the deterministic host act (the mean) and its log-probs, and
    orl_policy_eval's per-dimension log-probs of given actions against a float64 forward."""
    from oracle import nets

    rows = 4133
    cfg, net, agent = make_agent(_BoxHost(4, d), WIDE_FLAGS + ["--seed", str(d)], start=False)
    pol = net.module.models["policy"]
    rng = np.random.default_rng(d)
    obs = rng.standard_normal((rows, d)).astype(np.float32)
    given = rng.standard_normal((rows, 4)).astype(np.float32)
    ncfg = types.SimpleNamespace(layer_N=1, activation_id=pol.activation_id, use_recurrent_policy=False)

    def fwd(dt):
        p = ref.unflatten(pol.flat_params.to(dt), d, 4, "gaussian")
        with torch.no_grad():
            feat, _ = nets.policy_features(p, ncfg, torch.from_numpy(obs).cuda().to(dt))
            mean, std = nets.gaussian_params(p, feat)
            lp_given = torch.distributions.Normal(mean, std).log_prob(torch.from_numpy(given).cuda().to(dt))
        return mean, std, lp_given

    m64, s64, g64 = fwd(torch.float64)
    m32, s32, g32 = fwd(torch.float32)
    acts, lp = net.module.act(obs, deterministic=True)
    _forward_bar(f"act mean d{d}", acts, m64, m32)
    want = torch.distributions.Normal(m64, s64).log_prob(acts.double())
    assert float((lp.double() - want).abs().max()) <= ATOL
    _, elp, ent, _ = net.module.evaluate_actions(obs, obs, None, None, given, None)
    _forward_bar(f"eval log-probs d{d}", elp, g64, g32)


# ---------------------------------------------------------------- the insert ------------------------------------------

def test_insert_wide_critic_section(cuda):
    """orl_host_insert_wide_obs on staged blocks with critic sections of 65 and 256 features (8 agents, masks of 14
    actions): every output is what the insert rule gives, bit for bit; orl_host_insert refuses those sections and
    orl_host_insert_wide_obs refuses 257."""
    from openrl_b200 import lib

    L = lib.load()
    rng = np.random.default_rng(3)
    n_envs, A, d, n = 37, 8, 80, 14
    B = n_envs * A
    for dc in (65, 256):
        obs, cri, rew = (rng.standard_normal(B * w).astype(np.float32) for w in (d, dc, 1))
        dones = (rng.random((n_envs, A)) < 0.4).astype(np.float32)
        dones[rng.random(n_envs) < 0.3] = 1.0      # some envs with every agent done
        am = (rng.random(B * n) < 0.5).astype(np.float32)
        blk = torch.from_numpy(np.concatenate([obs, cri, rew, dones.reshape(-1), am])).cuda()
        o = dict(obs=torch.full((B, d), -9.0, device="cuda"), rew=torch.full((B,), -9.0, device="cuda"),
                 masks=torch.full((B,), -9.0, device="cuda"), active=torch.full((B,), -9.0, device="cuda"),
                 am=torch.full((B, n), -9.0, device="cuda"), cri=torch.full((B, dc), -9.0, device="cuda"))
        args = (lib.ptr(blk), n_envs, A, d, lib.ptr(o["obs"]), lib.ptr(o["rew"]), lib.ptr(o["masks"]), lib.ptr(o["active"]),
                lib.ptr(o["am"]), n, lib.ptr(o["cri"]), dc, lib.current_stream())
        assert L.orl_host_insert(*args) == 10001
        assert L.orl_host_insert_wide_obs(*args) == 0
        torch.cuda.synchronize()
        env_done = np.repeat(dones.all(1, keepdims=True), A, axis=1).reshape(-1)
        dn = dones.reshape(-1) != 0
        assert np.array_equal(o["obs"].cpu().numpy(), obs.reshape(B, d))
        assert np.array_equal(o["cri"].cpu().numpy(), cri.reshape(B, dc))
        assert np.array_equal(o["rew"].cpu().numpy(), rew)
        assert np.array_equal(o["am"].cpu().numpy(), am.reshape(B, n))
        assert np.array_equal(o["masks"].cpu().numpy(), np.where(env_done, 0.0, 1.0).astype(np.float32))
        assert np.array_equal(o["active"].cpu().numpy(), np.where(dn & ~env_done, 0.0, 1.0).astype(np.float32))
        assert env_done.any() and (~env_done).any()
    p = lib.ptr(blk)
    assert L.orl_host_insert_wide_obs(p, 2, 1, 4, p, p, p, p, None, 0, p, 257, lib.current_stream()) == 10001
    assert b"1..256" in L.orl_last_error()


# ---------------------------------------------------------------- end to end ------------------------------------------

def test_smac_8m_shaped_env_trains_in_both_host_loops(cuda, tmp_path):
    """A SMAC-8m-shaped env (8 agents, Dict {"policy": 80, "critic": 168}, Discrete(14), masks): PPOAgent.train for
    two iterations in the synchronous and in the two-group host loop from the same weights.  The two loops' buffers
    agree bit for bit, every logged scalar is finite, and the pickled-module checkpoint round-trips."""
    from openrl_b200.envs.vec_env import HostVecEnv
    from openrl_b200.utils.logger import Logger

    N, T = 64, 32
    flags = WIDE_FLAGS + ["--seed", "2", "--episode_length", str(T), "--ppo_epoch", "2", "--num_mini_batch", "2",
                          "--log_interval", "1"]
    runs, init = [], None
    for grouped in (False, True):
        env = HostVecEnv(_DictHost(N), wide_observations=True)
        assert (env.obs_dim, env.critic_obs_dim) == (80, 168) and env.supports_groups
        cfg, net, agent = make_agent(env, flags + ["--host_env_groups", "true" if grouped else "false"], like=init)
        if init is None:
            init = {mk: {k: v.clone() for k, v in net.module.models[mk].state_dict().items()} for mk in ("policy", "critic")}
        drv, b = agent.driver, agent.driver.buffer.data
        assert not drv.trainer.use_tensor_cores and (drv.trainer.d, drv.trainer.dc, drv.trainer.n) == (80, 168, 14)
        env.env.reset()
        drv.reset_and_buffer_init()
        bufs = []
        for it in range(2):
            drv.episode = it
            drv.actor_rollout()
            drv.compute_returns()
            torch.cuda.synchronize()
            bufs.append({k: getattr(b, k).cpu().numpy().copy()
                         for k in ("actions", "action_log_probs", "policy_obs", "critic_obs", "masks", "active_masks",
                                   "rewards", "action_masks", "value_preds", "returns")})
            for k, v in bufs[-1].items():
                assert np.isfinite(v).all(), k
            torch.manual_seed(7)
            info = drv.trainer.train(b)
            assert all(np.isfinite(float(v)) for v in info.values()), info
            b.after_update()
        runs.append(bufs)
    for it in range(2):
        for k in runs[0][it]:
            assert np.array_equal(runs[0][it][k], runs[1][it][k]), (it, k)

    logger = Logger(quiet=True)
    agent.train(total_time_steps=T * N * 2, logger=logger)
    logs = [x[1] for x in logger.history if "value_loss" in x[1]]
    assert logs and all(np.isfinite(list(v.values())).all() for v in logs), logs
    obs = np.random.default_rng(0).standard_normal((16, 80)).astype(np.float32)
    before = net.module.act(obs, deterministic=True)
    saved = {mk: {k: v.clone() for k, v in net.module.models[mk].state_dict().items()} for mk in ("policy", "critic")}
    agent.save(tmp_path / "wide")
    with torch.no_grad():
        for mk in ("policy", "critic"):
            for v in net.module.models[mk].state_dict().values():
                v.zero_()
    agent.load(tmp_path / "wide")
    for mk in ("policy", "critic"):
        for k, v in net.module.models[mk].state_dict().items():
            assert torch.equal(v, saved[mk][k]), (mk, k)
    after = net.module.act(obs, deterministic=True)
    assert torch.equal(before[0], after[0]) and torch.equal(before[1], after[1])
