"""GRU policies with DiagGaussian heads of 9..64 dimensions on host-stepped Box-action envs
(cfg.use_wide_recurrent_gaussian_head): the host act (rnn_act_rows_warp_kernel<R, 64, DX, ORL_HEAD_GAUSSIAN_WIDE>), the
chunked update (rnn_chunk_warp_kernel<true, false, R, 64, DX, ORL_HEAD_GAUSSIAN_WIDE>, its TAPE_GAUSS_WIDE rows and the
logstd column sum over TW_DLSW) and the optimiser (rnn_apply_kernel<ORL_HEAD_GAUSSIAN>, which the wide kind runs as).

Bars: the act row by row against a float64 forward (means, log-probs, the noise table, the mean when deterministic) at
one and two rows per warp and at d = 241 (one row per warp by shared memory), and its Philox noise against Box-Muller of
lanes 2..33, bit for bit against the feed-forward wide act of the same key and, on dimensions 0..7, against the 8-wide
GRU act; one update over every chunk of a host rollout against the float64 oracle (tests/gru_gaussian_oracle.py) per
gradient block, logstd its own block, at 4x the float32 oracle's error with a 2e-6 floor and a 1e-3 ceiling, over head
widths 9, 21 and 64, observation widths 9, 64, 65, 241 and 256, chunk lengths 1, 3 and 32, row counts beside the tape's
1024-row blocks and every loss option; reruns bit for bit; three mistakes of the Gaussian loss that the bars reject; both
host loops writing the same bits; the reference's two traces in parity mode; and a 3-agent Box(21) env end to end
through PPOAgent.train, a checkpoint, PPOAgent.act and evaluate_policy."""
import types

import numpy as np
import pytest
import torch

import gru_gaussian_oracle as ggo
from helpers import KEYS, make_agent, philox_units

pytestmark = pytest.mark.gpu

OPT = ["--use_recurrent_gaussian_head", "true", "--use_wide_recurrent_gaussian_head", "true",
       "--use_wide_recurrent_observations", "true"]
LOG_SQRT_2PI = np.float32(0.9189385332046727)
SEED, STEP = 0x1234_5678_9ABC, 11


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


class _Host:
    """N envs x A agents, observations (A, d) ~ N(0, 1), Box(n) actions, rewards ~ N(0, 1); an env finishes with
    probability 0.15 per step, and agents 1.. are done on their own with probability 0.2.  Every draw is keyed by (env, the env's step count), so `step_range` returns what the
    whole-range step would."""

    def __init__(self, N, n, d, A=1, seed=0):
        from openrl_b200 import spaces

        self.parallel_env_num, self.agent_num, self.n, self.d, self.seed = N, A, n, d, seed
        self.observation_space = spaces.Box(-np.inf, np.inf, (d,), np.float32)
        self.action_space = spaces.Box(-1.0, 1.0, (n,), np.float32)
        self.t = np.zeros(N, np.int64)

    def _draw(self, e):
        # with several agents, agent a > 0 is also done on its own with probability 0.2, so active masks have zeros
        g = np.random.default_rng((self.seed, e, int(self.t[e])))
        obs = g.standard_normal((self.agent_num, self.d)).astype(np.float32)
        env_done = g.random() < 0.15
        own = g.random(self.agent_num) < 0.2 if self.agent_num > 1 else np.zeros(1, bool)
        own[0] = False
        return obs, env_done | own, g.standard_normal((self.agent_num, 1))

    def _out(self, lo, hi):
        draws = [self._draw(e) for e in range(lo, hi)]
        dones = np.stack([x[1] for x in draws])
        return np.stack([x[0] for x in draws]), np.stack([x[2] for x in draws]), dones, [{} for _ in draws]

    def reset(self, seed=None):
        self.t[:] = 0
        return self._out(0, self.parallel_env_num)[0]

    def step(self, actions):
        return self.step_range(0, self.parallel_env_num, actions)

    def step_range(self, lo, hi, actions):
        a = np.asarray(actions).reshape(hi - lo, self.agent_num, self.n)
        assert np.isfinite(a).all()
        self.t[lo:hi] += 1
        return self._out(lo, hi)


def _venv(host):
    from openrl_b200.envs.vec_env import HostVecEnv

    return HostVecEnv(host, wide_observations=True)


def _ocfg(flags):
    from oracle import loop

    cfg = loop.cfg_from_flags(" ".join(flags))
    cfg.use_naive_recurrent_policy = "--use_naive_recurrent_policy" in flags
    return cfg


# ---------------------------------------------------------------- the act ---------------------------------------------

def _module(d, n, zero_head=False, recurrent=True):
    from openrl_b200 import spaces
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.modules.common import PPONet

    class Env:
        agent_num, parallel_env_num = 1, 1
        observation_space, action_space = spaces.Box(-5, 5, (d,), np.float32), spaces.Box(-1, 1, (n,), np.float32)

        def reset(self, seed=None):
            return np.zeros((1, 1, d), np.float32)

    ff = ["--use_wide_observations", "true", "--use_wide_gaussian_head", "true"]
    flags = ["--seed", "7"] + (["--use_recurrent_policy", "true"] + OPT if recurrent else ff)
    cfg = create_config_parser().parse_args(flags)
    cfg.quiet = True
    module = PPONet(Env(), cfg=cfg, device="cuda:0").module
    sd = module.models["policy"].state_dict()
    if zero_head:   # the means are the bias (0) and std 1: an action is its noise
        sd["act.action_out.fc_mean.weight"].zero_()
        sd["act.action_out.logstd._bias"].zero_()
    else:
        sd["act.action_out.fc_mean.weight"].mul_(5.0)
        sd["act.action_out.logstd._bias"].copy_(torch.linspace(-0.5, 0.5, n).view(n, 1))
    return module, _ocfg(flags[:2] + (["--use_recurrent_policy", "true"] if recurrent else []))


def _params64(model):
    return {k: v.detach().cpu().double() for k, v in model.named_parameters()}


def _box_muller(rows, n, seed=SEED, step=STEP):
    """Dimensions [4k, 4k + 4): Box-Muller of Philox lanes 2 + 2k (u1) and 3 + 2k (u2), k = 0..15, in float64."""
    u = philox_units(1, rows, seed, step, 0, tuple(range(2, 34)))[0].astype(np.float64)   # (rows, 128)
    u1 = np.concatenate([u[:, 8 * k:8 * k + 4] for k in range(16)], 1)
    u2 = np.concatenate([u[:, 8 * k + 4:8 * k + 8] for k in range(16)], 1)
    return (np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2))[:, :n]


ACT_SHAPES = [(d, n) for d in (9, 64, 65, 241, 256) for n in (9, 21, 64)]


@pytest.mark.parametrize("d,n", ACT_SHAPES, ids=[f"d{d}-n{n}" for d, n in ACT_SHAPES])
def test_act_matches_float64(cuda, d, n):
    """PPOModule.act of a GRU policy with a noise table and deterministic against a float64 forward row by row, at one
    row per warp (16 x SMs rows) and two (64 x SMs + 37 rows; one at d = 241), from nonzero states and with masks that
    zero some."""
    from openrl_b200 import lib

    module, ocfg = _module(d, n)
    pol = module.models["policy"]
    assert pol.head_kind == lib.HEAD_GAUSSIAN_WIDE and pol.recurrent
    p = _params64(pol)
    for rows in (16 * _sm_count(), 64 * _sm_count() + 37):
        g = np.random.default_rng(rows + d + n)
        obs = g.normal(size=(rows, d)).astype(np.float32)
        h = g.normal(size=(rows, 1, 64)).astype(np.float32)
        masks = (g.random((rows, 1)) < 0.8).astype(np.float32)
        noise = g.normal(size=(rows, n)).astype(np.float32)
        act, logp, h2 = module.act(obs, h, masks, exp_noise=noise)
        mean_d, logp_d, h2_d = module.act(obs, h, masks, deterministic=True)
        torch.cuda.synchronize()
        assert act.shape == (rows, n) and logp.shape == (rows, n)
        t = lambda x: torch.from_numpy(x).double()  # noqa: E731
        with torch.no_grad():
            want_act, want_logp, want_h = ggo.policy_act_gaussian(p, ocfg, t(obs), t(h), t(masks), normal_noise=t(noise))
            mean, _, _ = ggo.policy_act_gaussian(p, ocfg, t(obs), t(h), t(masks), deterministic=True)
        np.testing.assert_allclose(act.cpu().numpy(), want_act.numpy(), rtol=0, atol=1e-5)
        np.testing.assert_allclose(logp.cpu().numpy(), want_logp.numpy(), rtol=0, atol=2e-5)
        np.testing.assert_allclose(h2.cpu().numpy(), want_h.numpy(), rtol=0, atol=2e-5)
        np.testing.assert_allclose(mean_d.cpu().numpy(), mean.numpy(), rtol=0, atol=1e-5)
        assert np.array_equal(h2_d.cpu().numpy(), h2.cpu().numpy())
        ls = pol.state_dict()["act.action_out.logstd._bias"].cpu().numpy()[:, 0]
        want = np.broadcast_to(-ls - LOG_SQRT_2PI, (rows, n))
        assert np.array_equal(logp_d.cpu().numpy().view(np.int32), want.view(np.int32))


@pytest.mark.parametrize("n", [9, 21, 64])
def test_philox_noise_is_the_feed_forward_acts(cuda, n):
    """With the means 0 and std 1 an action is its noise: Box-Muller of Philox lanes 2..33 of (seed, step, row), bit for
    bit what the feed-forward wide act draws for the same key, and on dimensions 0..7 what the 8-wide GRU act draws, at
    one and at two rows per warp."""
    module, _ = _module(27, n, zero_head=True)
    ff, _ = _module(27, n, zero_head=True, recurrent=False)
    narrow, _ = _module(27, 8, zero_head=True)
    for rows in (16 * _sm_count(), 64 * _sm_count() + 5):
        obs = np.random.default_rng(rows).normal(size=(rows, 27)).astype(np.float32)
        act, _, _ = module.act(obs, rng_seed=SEED, rng_step=STEP)
        act_ff, _ = ff.act(obs, rng_seed=SEED, rng_step=STEP)
        act_8, _, _ = narrow.act(obs, rng_seed=SEED, rng_step=STEP)
        torch.cuda.synchronize()
        got = act.cpu().numpy()
        np.testing.assert_allclose(got.astype(np.float64), _box_muller(rows, n), rtol=0, atol=1e-5)
        assert np.array_equal(got.view(np.int32), act_ff.cpu().numpy().view(np.int32))
        assert np.array_equal(got[:, :8].view(np.int32), act_8.cpu().numpy().view(np.int32))


# ---------------------------------------------------------------- the update ------------------------------------------

def _rollout(n, d, N, T, L, A=1, extra=(), seed=0, naive=False):
    """A host rollout of N envs x A agents x T steps with Philox sampling, then the policy's weights moved slightly off the
    ones that acted (ratios leave 1 but stay far from the clip's kinks, where float32 and float64 may pick different
    branches).  Returns (flags, net, agent)."""
    rec = ["--use_naive_recurrent_policy", "true"] if naive else ["--use_recurrent_policy", "true"]
    flags = ["--seed", str(5 + seed), *rec, *OPT, "--episode_length", str(T), "--data_chunk_length", str(L),
             "--ppo_epoch", "1", "--num_mini_batch", "1", "--use_valuenorm", "false", "--host_env_groups", "false", *extra]
    cfg, net, agent = make_agent(_venv(_Host(N, n, d, A=A, seed=seed)), flags)
    pol = net.module.models["policy"]
    with torch.no_grad():
        sd = pol.state_dict()
        sd["act.action_out.logstd._bias"].copy_(torch.linspace(-0.4, 0.3, n).view(n, 1))
    drv = agent.driver
    drv.actor_rollout()
    drv.compute_returns()
    with torch.no_grad():
        g = torch.Generator(device="cuda").manual_seed(seed)
        pol.flat_params.add_(torch.randn(pol.flat_params.shape, device="cuda", generator=g), alpha=1e-3)
    return flags, net, agent


def _host_buf(b):
    """The device buffer as the oracle's recurrent generators read it ((T+1, N, A, ...) numpy, states with recurrent_N)."""
    c = lambda x: x.cpu().numpy().copy()  # noqa: E731
    names = ("policy_obs", "critic_obs", "actions", "action_log_probs", "value_preds", "returns", "masks", "active_masks")
    ns = types.SimpleNamespace(**{k: c(getattr(b, k)) for k in names})
    ns.rewards = np.zeros(ns.actions.shape[:3] + (1,), np.float32)
    ns.action_masks = np.ones(ns.masks.shape, np.float32)
    ns.rnn_states, ns.rnn_states_critic = c(b.rnn_states), c(b.rnn_states_critic)
    return ns


def _oracle_update(ocfg, state, hb, dtype, mutant=None, clip_keys=None):
    """One update of the oracle over every chunk of hb from `state` ({net: {name: tensor}}): (grads before the clip,
    params after, record).  mutant: 'no_entropy_dls' (the entropy term left out of dL/dlogstd) or 'rows_weight' (the
    entropy weighted 1 / rows instead of 1 / (rows n))."""
    from oracle import gae as ogae
    from oracle import loop_ma, ppo

    _, adv = ogae.advantages(hb.returns, hb.value_preds, hb.active_masks, None, ocfg.use_adv_normalize)
    owner = types.SimpleNamespace(cfg=ocfg, buf=hb)
    gen = loop_ma.MATrainer._naive_batches if ocfg.use_naive_recurrent_policy else loop_ma.MATrainer._recurrent_batches
    (_, bt), = list(gen(owner, adv))
    batch = {k: v.to(dtype) for k, v in bt.items()}
    batch["old_logp"] = batch.pop("action_log_probs")
    pol = {k: v.detach().clone().to(dtype) for k, v in state["policy"].items()}
    cri = {k: v.detach().clone().to(dtype) for k, v in state["critic"].items()}
    opt_p, opt_c = ppo.make_optimizers(ocfg, pol, cri)
    rec = {}
    evaluate = ggo.policy_eval_gaussian
    if mutant is not None:
        def ev(p, cfg, obs, actions, active, rnn_states, masks):
            from oracle import nets

            feat, _ = nets.policy_features(p, cfg, obs, rnn_states, masks)
            mean, std = nets.gaussian_params(p, feat)
            ent_std = std.detach() if mutant == "no_entropy_dls" else std
            ent = torch.distributions.Normal(mean, ent_std).entropy()
            if mutant == "rows_weight":
                ent = ent.sum(-1).mean()
            elif active is not None and cfg.use_policy_active_masks:
                ent = (ent * active).sum() / active.sum()
            else:
                ent = ent.mean()
            return torch.distributions.Normal(mean, std).log_prob(actions), ent
        evaluate = ev
    out = ggo.ppo_update(ocfg, pol, cri, opt_p, opt_c, None, batch, rec, evaluate=evaluate, clip_keys=clip_keys)
    return rec, {"policy": pol, "critic": cri}, out


def _blocks(flat, model):
    out, off = {}, 0
    for k, v in model.named_parameters():
        out[k] = flat[off:off + v.numel()].view(v.shape).detach().cpu().double()
        off += v.numel()
    return out


def _err(x, ref):
    scale = float(ref.abs().max())
    return float((x - ref).abs().max()) / max(scale, 1e-30), scale


def _check(got, r64, r32, what, errs=None):
    """Per block: the kernel's error (relative to the block's max |.|) at most 4x the float32 oracle's, floor 2e-6,
    ceiling 1e-3."""
    for k in r64:
        e_k, _ = _err(got[k], r64[k])
        e_32, _ = _err(r32[k].double(), r64[k])
        bar = min(max(4.0 * e_32, 2e-6), 1e-3)
        if errs is not None:
            errs[k] = (e_k, bar)
        assert e_k <= bar, f"{what} {k}: {e_k:.3g} > {bar:.3g}"


def _run(n, d, N, T, L, A=1, extra=(), seed=0, naive=False, twice=False):
    flags, net, agent = _rollout(n, d, N, T, L, A=A, extra=extra, seed=seed, naive=naive)
    drv, tr, b = agent.driver, agent.driver.trainer, agent.driver.buffer.data
    models = net.module.models
    assert tr.head_kind == 2 and tr.n == n and tr.d == d
    state = {mk: {k: v.detach().clone() for k, v in models[mk].named_parameters()} for mk in ("policy", "critic")}
    flat0 = {mk: models[mk].flat_params.clone() for mk in ("policy", "critic")}
    opt0 = {mk: (net.module.optimizers[mk].exp_avg.clone(), net.module.optimizers[mk].exp_avg_sq.clone()) for mk in ("policy", "critic")}
    steps0 = net.module.adam_steps.clone()
    hb = _host_buf(b)
    torch.manual_seed(1)
    info = tr.train(b)
    torch.cuda.synchronize()
    ocfg = _ocfg(flags)
    torch.manual_seed(1)
    r64, p64, out64 = _oracle_update(ocfg, {mk: {k: v.cpu() for k, v in s.items()} for mk, s in state.items()}, hb, torch.float64)
    torch.manual_seed(1)
    r32, _, _ = _oracle_update(ocfg, {mk: {k: v.cpu() for k, v in s.items()} for mk, s in state.items()}, hb, torch.float32)
    P = models["policy"].flat_params.numel()
    got_g = _blocks(tr.rnn_grads[0][:P], models["policy"])
    assert "act.action_out.logstd._bias" in got_g
    _check(got_g, r64["grads_policy"], r32["grads_policy"], "policy grad")
    _check(_blocks(tr.rnn_grads[1], models["critic"]), r64["grads_critic"], r32["grads_critic"], "critic grad")
    for mk in ("policy", "critic"):
        # Adam's first step is lr g / (|g| + eps) after the clip: an element whose gradient is near 0 moves its step by
        # lr / eps times the gradient's rounding, so the steps are held at 1e-2 of the largest one (logstd's included)
        for k, v in models[mk].named_parameters():
            d_got = v.detach().cpu().double() - state[mk][k].cpu().double()
            d64 = p64[mk][k].detach() - state[mk][k].cpu().double()
            assert float((d_got - d64).abs().max()) <= 1e-2 * float(d64.abs().max()) + 1e-9, f"{mk} step {k}"
    # the policy loss is a float32 running sum of n surrogates per row that nearly cancel: its rounding grows with n while
    # its value can be near 0, so the absolute bar is the 8-wide head's 1e-6 per 8 dimensions
    want = dict(zip(KEYS, out64))
    for name in KEYS:
        np.testing.assert_allclose(info[name], want[name], rtol=2e-4, atol=1e-6 * n / 8, err_msg=name)
    if twice:   # the same update from the same state: the same bits
        first = {mk: models[mk].flat_params.clone() for mk in ("policy", "critic")}
        for mk in ("policy", "critic"):
            models[mk].flat_params.copy_(flat0[mk])
            net.module.optimizers[mk].exp_avg.copy_(opt0[mk][0])
            net.module.optimizers[mk].exp_avg_sq.copy_(opt0[mk][1])
        net.module.adam_steps.copy_(steps0)
        torch.manual_seed(1)
        tr.train(b)
        torch.cuda.synchronize()
        for mk in ("policy", "critic"):
            assert torch.equal(models[mk].flat_params, first[mk]), mk
    return dict(flags=flags, state=state, hb=hb, ocfg=ocfg, models=models, tr=tr, info=info, r64=r64, r32=r32, P=P, out64=out64)


GRID = [(n, d) for n in (9, 21, 64) for d in (9, 64, 65, 241, 256)]


@pytest.mark.parametrize("n,d", GRID, ids=[f"n{n}-d{d}" for n, d in GRID])
def test_update_matches_float64(cuda, n, d):
    """32 envs x 2 agents x T = 48 at L = 3 (1024 chunks: 3072 tape rows): every gradient block against the float64
    oracle, the Adam steps and the reported scalars.  d = 241 and 256 run one chunk per warp."""
    _run(n, d, N=32, T=48, L=3, A=2, seed=n + d)


CHUNKS = [(1, 1023, 1, 1), (1, 1024, 1, 1), (1, 1025, 1, 1), (3, 32, 96, 3), (32, 8, 64, 32), (32, 5, 64, 32)]


@pytest.mark.parametrize("L,N,T,A", CHUNKS, ids=[f"L{c[0]}-N{c[1]}-T{c[2]}-A{c[3]}" for c in CHUNKS])
def test_update_chunk_lengths_and_row_blocks(cuda, L, N, T, A):
    """Chunk lengths 1, 3 and 32; 1023, 1024 and 1025 tape rows (the reduction's 1024-row blocks); states zeroed by
    episode ends mid-chunk (an env ends with probability 0.15 per step); reruns bit for bit."""
    _run(21, 18, N=N, T=T, L=L, A=A, seed=L + N, twice=True)


def test_update_naive_recurrent_generator(cuda):
    """use_naive_recurrent_policy: every buffer row's whole trajectory is one chunk (Box(256) observations, Box(64))."""
    _run(64, 256, N=16, T=24, L=24, naive=True, seed=3, twice=True)


LOSS_OPTIONS = [[], ["--use_policy_active_masks", "false"], ["--use_huber_loss", "false", "--use_clipped_value_loss", "false"],
                ["--use_adv_normalize", "false"], ["--dual_clip_ppo", "true"], ["--use_max_grad_norm", "false"],
                ["--max_grad_norm", "0.05"], ["--entropy_coef", "0.2"], ["--use_value_active_masks", "false"]]


@pytest.mark.parametrize("extra", LOSS_OPTIONS, ids=["default"] + [" ".join(x) for x in LOSS_OPTIONS[1:]])
def test_update_loss_options(cuda, extra):
    """Every loss option at Box(21) on 18 features, with and without the policy's active masks."""
    _run(21, 18, N=32, T=32, L=4, A=3, extra=extra, seed=11)


def test_mutants_are_rejected(cuda):
    """The bars reject three mistakes of the Gaussian loss: no entropy term in dL/dlogstd, an entropy weight of 1 / rows
    (not 1 / (rows n)), and logstd left out of the clip norm (the reported actor_grad_norm)."""
    r = _run(21, 18, N=32, T=32, L=4, A=2, extra=["--entropy_coef", "0.05", "--max_grad_norm", "0.05",
                                                  "--use_policy_active_masks", "false"], seed=13)
    models, tr = r["models"], r["tr"]
    got = _blocks(tr.rnn_grads[0][:r["P"]], models["policy"])
    key = "act.action_out.logstd._bias"
    errs = {}
    _check({key: got[key]}, {key: r["r64"]["grads_policy"][key]}, {key: r["r32"]["grads_policy"][key]}, "logstd", errs)
    bar = errs[key][1]
    state = {mk: {k: v.cpu() for k, v in s.items()} for mk, s in r["state"].items()}
    for mutant in ("no_entropy_dls", "rows_weight"):
        torch.manual_seed(1)
        rec, _, _ = _oracle_update(r["ocfg"], state, r["hb"], torch.float64, mutant=mutant)
        e_bad, _ = _err(rec["grads_policy"][key], r["r64"]["grads_policy"][key])
        assert e_bad > bar, mutant
        e_k, _ = _err(got[key], rec["grads_policy"][key])
        assert e_k > bar, mutant   # the kernel is not the mutant
    # logstd in the clip norm: the oracle run with the norm over every policy parameter but logstd (clip_keys) reports
    # another actor_grad_norm; the kernel's is the full norm's
    keys = [k for k in state["policy"] if k != key]
    torch.manual_seed(1)
    _, _, out_bad = _oracle_update(r["ocfg"], state, r["hb"], torch.float64, clip_keys=keys)
    full, got_norm = dict(zip(KEYS, r["out64"]))["actor_grad_norm"], r["info"]["actor_grad_norm"]
    bad = dict(zip(KEYS, out_bad))["actor_grad_norm"]
    assert abs(got_norm - full) <= 1e-4 * full
    assert abs(got_norm - bad) > 1e-3 * full


# ---------------------------------------------------------------- the host loops and end to end -----------------------

def test_host_loops_agree(cuda):
    """1024 envs x T = 128 at Box(21) on 17 features: the synchronous and the two-group loop write the same bits over two
    iterations with an update between them."""
    N, T = 1024, 128
    flags = ["--seed", "3", "--use_recurrent_policy", "true", *OPT, "--episode_length", str(T), "--data_chunk_length", "8",
             "--ppo_epoch", "1", "--num_mini_batch", "2", "--log_interval", "1"]
    runs, init = [], None
    for grouped in (False, True):
        env = _venv(_Host(N, 21, 17, seed=4))
        assert env.supports_groups
        cfg, net, agent = make_agent(env, flags + ["--host_env_groups", "true" if grouped else "false"], like=init)
        if init is None:
            init = {mk: {k: v.clone() for k, v in net.module.models[mk].state_dict().items()} for mk in ("policy", "critic")}
        drv, b = agent.driver, agent.driver.buffer.data
        bufs = []
        for it in range(2):
            drv.episode = it
            drv.actor_rollout()
            torch.cuda.synchronize()
            bufs.append({k: getattr(b, k).cpu().numpy().copy()
                         for k in ("actions", "action_log_probs", "policy_obs", "masks", "rewards", "rnn_states")})
            assert bufs[-1]["actions"].shape[-1] == 21
            drv.compute_returns()
            torch.manual_seed(7)
            drv.trainer.train(b)
            b.after_update()
        runs.append(bufs)
    for it in range(2):
        for k in runs[0][it]:
            assert np.array_equal(runs[0][it][k], runs[1][it][k]), (it, k)


def test_three_agent_env_trains_checkpoints_and_evaluates(cuda, tmp_path):
    """A 3-agent env (17 features, Box(21)) with a GRU policy trains through PPOAgent in both host loops; logstd takes its
    Adam steps; the checkpoint keeps the reference's key names and round-trips; PPOAgent.act gives (N, 3, 21) float
    actions; evaluate_policy runs; without the option the same env is refused with the limit of 8."""
    from openrl_b200.utils.evaluation import evaluate_policy
    from openrl_b200.utils.logger import Logger

    base = ["--seed", "2", "--use_recurrent_policy", "true", "--use_recurrent_gaussian_head", "true",
            "--episode_length", "32", "--data_chunk_length", "8", "--ppo_epoch", "2", "--num_mini_batch", "2",
            "--log_interval", "1"]
    with pytest.raises(NotImplementedError, match="up to 8"):
        make_agent(_venv(_Host(8, 21, 17, A=3)), base, start=False)
    for grouped in ("false", "true"):
        flags = base + ["--use_wide_recurrent_gaussian_head", "true", "--host_env_groups", grouped]
        cfg, net, agent = make_agent(_venv(_Host(16, 21, 17, A=3, seed=2)), flags, start=False)
        assert net.module.models["policy"].head_kind == 2
        logger = Logger(quiet=True)
        before = net.module.models["policy"].state_dict()["act.action_out.logstd._bias"].clone()
        agent.train(total_time_steps=32 * 16 * 2, logger=logger)
        got = [h_[1] for h_ in logger.history if "policy_loss" in h_[1]]
        assert got and all(np.isfinite(v) for row in got for v in row.values())
        sd = net.module.models["policy"].state_dict()
        assert not torch.equal(sd["act.action_out.logstd._bias"], before)   # logstd takes its Adam steps
    agent.save(tmp_path / "ck")
    _, net2, agent2 = make_agent(_venv(_Host(16, 21, 17, A=3, seed=5)), flags, start=False)
    agent2.load(tmp_path / "ck")
    for k, v in net.module.models["policy"].state_dict().items():
        assert torch.equal(net2.module.models["policy"].state_dict()[k], v), k
    assert "rnn.rnn.weight_ih_l0" in sd and sd["act.action_out.fc_mean.weight"].shape == (21, 64)
    obs = np.random.default_rng(0).standard_normal((16, 3, 17)).astype(np.float32)
    a1, _ = agent.act(obs, deterministic=True)
    a2, _ = agent2.act(obs, deterministic=True)
    assert a1.shape == (16, 3, 21) and a1.dtype == np.float32 and np.array_equal(a1, a2)
    out = evaluate_policy(agent2, _venv(_Host(4, 21, 17, A=3, seed=6)), n_eval_episodes=2)
    assert np.isfinite(np.asarray(out[0] if isinstance(out, tuple) else out, dtype=np.float64)).all()


def test_module_refusals(cuda):
    """JRPO with a Box space, use_share_model with a GRU, and Box(65) keep their refusals with the option."""
    from openrl_b200.envs.vec_env import HostVecEnv

    base = ["--seed", "1", "--use_recurrent_policy", "true", "--use_recurrent_gaussian_head", "true",
            "--use_wide_recurrent_gaussian_head", "true", "--episode_length", "8"]
    with pytest.raises(NotImplementedError, match="JRPO"):
        make_agent(HostVecEnv(_Host(4, 21, 18, A=3)), base + ["--use_joint_action_loss", "true"])
    with pytest.raises(NotImplementedError, match="share|recurrent"):
        make_agent(HostVecEnv(_Host(4, 21, 18)), base + ["--use_share_model", "true"])
    with pytest.raises(NotImplementedError, match="64"):
        make_agent(HostVecEnv(_Host(4, 65, 18)), base, start=False)


# ---------------------------------------------------------------- the reference's traces ------------------------------

@pytest.mark.parametrize("tag", ["gru_gaussian_wide_21", "gru_gaussian_wide_spread_64"])
def test_reproduces_reference_trace(cuda, tag):
    """PPOAgent over make()'s host vec-env in parity mode against the reference's runs on the envs of
    tests/gru_gaussian_wide_oracle.py: Box(67) observations with Box(21) (use_recurrent_policy), and 3 agents, Dict
    18 / 54, Box(64), agents finishing apart (use_naive_recurrent_policy).  Actions 1e-5, log-probs, hidden states and
    values 2e-5, the update scalars 2e-4, the parameters after the last iteration 2e-3."""
    import os

    from conftest import GOLDEN
    from gru_gaussian_wide_oracle import SPACED
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.common import make

    d = np.load(os.path.join(GOLDEN, f"trace_{tag}.npz"), allow_pickle=True)
    iters, N = int(d["meta/iters"]), int(d["meta/env_num"])
    flags = str(d["meta/flags"]).split() + ["--parity_mode", "true", "--log_interval", "1", *OPT]
    spread = tag == "gru_gaussian_wide_spread_64"
    cls = SPACED[tag]
    env = make("GRUGaussianWide", env_num=N, make_custom_envs=lambda id, env_num, render_mode=None, **kw: [cls for _ in range(env_num)],
               cfg=create_config_parser().parse_args(flags))
    cfg, net, agent = make_agent(env, flags, golden=d)
    drv, tr = agent.driver, agent.driver.trainer
    b = drv.buffer.data
    assert drv.recurrent and tr.n == (64 if spread else 21) and tr.head_kind == 2
    for it in range(iters):
        t = f"it{it}"
        drv.episode = it
        drv.actor_rollout()
        np.testing.assert_allclose(b.actions.cpu().numpy(), d[f"{t}/actions"], rtol=0, atol=1e-5, err_msg=t)
        assert np.array_equal(b.policy_obs.cpu().numpy(), d[f"{t}/policy_obs"]), t
        assert np.array_equal(b.masks.cpu().numpy(), d[f"{t}/masks"]), t
        assert np.array_equal(b.active_masks.cpu().numpy(), d[f"{t}/active_masks"]), t
        if spread:
            assert np.array_equal(b.critic_obs.cpu().numpy(), d[f"{t}/critic_obs"]), t
        np.testing.assert_allclose(b.action_log_probs.cpu().numpy(), d[f"{t}/action_log_probs"], rtol=0, atol=2e-5, err_msg=t)
        np.testing.assert_allclose(b.rnn_states.cpu().numpy(), d[f"{t}/rnn_states"], rtol=0, atol=2e-5, err_msg=t)
        drv.compute_returns()
        np.testing.assert_allclose(b.value_preds.cpu().numpy()[:-1], d[f"{t}/value_preds"][:-1], rtol=0, atol=2e-5, err_msg=t)
        info = tr.train(b)
        want = d[f"{t}/updates"].mean(axis=0)
        for col, name in enumerate(KEYS):
            np.testing.assert_allclose(info[name], want[col], rtol=2e-4, atol=1e-5, err_msg=f"{t} {name}")
        checked = 0
        for mk in ("policy", "critic"):
            for k, v in net.module.models[mk].state_dict().items():
                gk = f"{t}/params/{mk}.{k}"
                if gk in d and "value_normalizer" not in k:
                    np.testing.assert_allclose(v.cpu().numpy().reshape(d[gk].shape), d[gk], rtol=2e-3, atol=2e-5, err_msg=gk)
                    checked += 1
        assert checked > 0 or it < iters - 1, t
        b.after_update()
