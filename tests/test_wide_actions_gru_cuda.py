"""Discrete action spaces of 9..64 actions on the GRU policy: the wide head of the host act (rnn_act_rows_warp_kernel<R, 64, DX>)
and of the chunked recurrent update (the policy instance rnn_chunk_warp_kernel<true, false, R, 64, DX>, its tape rows of
TAPE_WIDE floats and their reduction).

Bars: the reference's traces on the masked env widened to 9 and 64 actions with a GRU policy
(tests/golden/trace_wide_actions_gru_*.npz) through PPOAgent over HostVecEnv in parity mode, at the bars of
tests/test_host_action_masks_cuda.py; one update over the whole buffer of a host rollout against rnn_ref64 driven with the
masks (tests/rnn_ref64_masked.py) through tests/scale_harness.py at RNN_FLOOR, for head widths on both sides of the 4- and
16-wide edges, obs widths 9 and 64, chunk lengths 1, 3 and 32, row counts at and beside the tape's 1024-row blocks,
one-legal and all-legal masks, every loss option at n = 64 and a SMAC-3m-shaped multi-agent case; the same rollout's act
teacher-forced against float64 row by row (log-probs and next hidden states at the bars of tests/test_rnn_scale_cuda.py);
each Philox-sampled action against argmax(p / q) with q from the host Philox; the first-max mode; legality at 1024 envs x
128 steps and the agreement of the two host loops; one fixed-seed chi-square test of the sampler; and the refusals."""
import copy
import os
import types

import numpy as np
import pytest
import torch

import rnn_ref64
import rnn_ref64_masked
from conftest import GOLDEN
from helpers import KEYS, make_agent, philox_units
from scale_harness import ATOL, CASES, RNN_FLOOR, Checker, c3_buf, drive, moment_scale, no_tf32  # noqa: F401  (no_tf32: fixture)
from wide_actions_oracle import WIDTHS, wide_target_vec

pytestmark = pytest.mark.gpu

# a GRU policy with the wide head (9..64 actions)
WIDE_GRU = ["--use_recurrent_policy", "true", "--use_wide_recurrent_head", "true"]
# Philox lanes of a wide head's actions: 0, 1 for actions 0..7, 8..21 for actions 8..63 (orl_envstep.cuh)
WIDE_LANES = [0, 1] + list(range(8, 22))


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


def _illegal(actions, action_masks):
    a = actions[..., 0].astype(np.int64)
    return int((np.take_along_axis(action_masks[:-1], a[..., None], axis=-1) == 0).sum())


class _WideHost:
    """N envs x A agents, observations (A, d) ~ N(0, 1) (or a Dict {"policy": (A, d), "critic": (A, dc)}), Discrete(n) with
    per-agent (A, n) masks in `info["action_masks"]`: "random" (each action legal with probability 0.5, the agent's
    first row of every eight with a single legal action, another with all legal), "one" (a single legal action) or "all".
    An env finishes with probability 0.15 per step, so hidden states are zeroed mid-chunk.  Every draw is keyed by (env,
    the env's step count): a sub-range step (`step_range`) returns what the whole-range step would."""

    def __init__(self, N, n, d, A=1, dc=None, legal="random", seed=0):
        from openrl_b200 import spaces

        box = lambda w: spaces.Box(-np.inf, np.inf, (w,), np.float32)  # noqa: E731
        self.parallel_env_num, self.agent_num, self.n, self.d, self.dc, self.legal, self.seed = N, A, n, d, dc, legal, seed
        self.observation_space = spaces.Dict({"policy": box(d), "critic": box(dc)}) if dc else box(d)
        self.action_space = spaces.Discrete(n)
        self.t, self.log = np.zeros(N, np.int64), {}

    def _draw(self, e):
        g = np.random.default_rng((self.seed, e, int(self.t[e])))
        A, n = self.agent_num, self.n
        pol = g.standard_normal((A, self.d)).astype(np.float32)
        cri = g.standard_normal((A, self.dc)).astype(np.float32) if self.dc else None
        keep = g.integers(0, n, A)
        if self.legal == "all":
            m = np.ones((A, n), np.int8)
        else:
            m = (g.random((A, n)) < 0.5).astype(np.int8) if self.legal == "random" else np.zeros((A, n), np.int8)
            if self.legal == "random":
                kind = (e * A + np.arange(A) + int(self.t[e])) % 8
                m[kind == 0] = 0
                m[kind == 1] = 1
            m[np.arange(A), keep] = 1
        self.log[e, int(self.t[e])] = m
        return pol, cri, m, g.random() < 0.15, g.standard_normal((A, 1))

    def _out(self, lo, hi):
        draws = [self._draw(e) for e in range(lo, hi)]
        pol = np.stack([x[0] for x in draws])
        obs = {"policy": pol, "critic": np.stack([x[1] for x in draws])} if self.dc else pol
        dones = np.repeat(np.array([x[3] for x in draws])[:, None], self.agent_num, axis=1)
        return obs, np.stack([x[4] for x in draws]), dones, [{"action_masks": x[2]} for x in draws]

    def reset(self, seed=None):
        self.t[:] = 0
        obs, _, _, infos = self._out(0, self.parallel_env_num)
        return obs, infos

    def step(self, actions):
        return self.step_range(0, self.parallel_env_num, actions)

    def step_range(self, lo, hi, actions):
        acts = np.asarray(actions).reshape(hi - lo, self.agent_num).astype(np.int64)
        for i, e in enumerate(range(lo, hi)):   # the env checks its actions against the masks it reported
            assert (self.log[e, int(self.t[e])][np.arange(self.agent_num), acts[i]] == 1).all(), "illegal action"
        self.t[lo:hi] += 1
        return self._out(lo, hi)


def _venv(host):
    from openrl_b200.envs.vec_env import HostVecEnv

    return HostVecEnv(host)


# ---------------------------------------------------------------- the reference's traces ------------------------------

@pytest.mark.parametrize("n", WIDTHS)
def test_wide_gru_reproduces_reference_trace(cuda, n):
    d = np.load(os.path.join(GOLDEN, f"trace_wide_actions_gru_{n}.npz"), allow_pickle=True)
    iters, N = int(d["meta/iters"]), int(d["meta/env_num"])
    flags = str(d["meta/flags"]).split() + ["--parity_mode", "true", "--log_interval", "1",
                                                   "--use_wide_recurrent_head", "true"]
    cfg, net, agent = make_agent(_venv(_Host(wide_target_vec(n)(N))), flags, golden=d)
    drv = agent.driver
    b = drv.buffer.data
    assert drv.recurrent and not b.action_masks_trivial and drv.trainer.n == n
    for it in range(iters):
        t = f"it{it}"
        drv.episode = it
        drv.actor_rollout()
        assert np.array_equal(b.actions.cpu().numpy(), d[f"{t}/actions"]), t
        assert np.array_equal(b.policy_obs.cpu().numpy(), d[f"{t}/policy_obs"]), t
        assert np.array_equal(b.masks.cpu().numpy(), d[f"{t}/masks"]), t
        assert np.array_equal(b.action_masks.cpu().numpy(), d[f"{t}/action_masks"]), t
        np.testing.assert_allclose(b.action_log_probs.cpu().numpy(), d[f"{t}/action_log_probs"], rtol=0, atol=2e-5)
        np.testing.assert_allclose(b.rnn_states.cpu().numpy(), d[f"{t}/rnn_states"], rtol=0, atol=2e-5)
        drv.compute_returns()
        np.testing.assert_allclose(b.rnn_states_critic.cpu().numpy(), d[f"{t}/rnn_states_critic"], rtol=0, atol=2e-5)
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


# ---------------------------------------------------------------- the act and the update against float64 -------------

def _sharpen(net, seed):
    """Head weights well above the init's 0.01 gain, so that the softmax is far from uniform."""
    pol = net.module.models["policy"]
    with torch.no_grad():
        pol.state_dict()["act.action_out.linear.weight"].normal_(0.0, 0.5, generator=torch.Generator(device="cuda").manual_seed(seed))


def _run(case, n, d, N, T, L, A=1, dc=None, legal="random", extra=(), seed=0):
    """A host rollout of N envs x A agents x T steps with a wide GRU policy (Philox sampling), its act checked
    teacher-forced against float64, then one update over every chunk of the buffer against rnn_ref64 with the masks."""
    flags = ["--seed", str(6 + seed), *WIDE_GRU, "--episode_length", str(T), "--data_chunk_length", str(L),
             "--ppo_epoch", "1", "--num_mini_batch", "1", "--use_valuenorm", "true", "--host_env_groups", "false", *extra]
    host = _WideHost(N, n, d, A=A, dc=dc, legal=legal, seed=seed)
    cfg, net, agent = make_agent(_venv(host), flags)
    _sharpen(net, seed)
    drv, tr, b = agent.driver, agent.driver.trainer, agent.driver.buffer.data
    assert tr.n == n and drv.recurrent
    # one warm-up iteration: the compared update is then a second Adam step with nonzero moments, not the first one, which
    # maps every gradient element to about +-lr and so amplifies the rounding of the elements near zero without bound
    drv.actor_rollout()
    drv.compute_returns()
    tr.train(b)
    b.after_update()
    drv.episode = 1
    drv.actor_rollout()
    drv.compute_returns()
    torch.cuda.synchronize()
    B = N * A
    am = b.action_masks.cpu().numpy()
    assert am.shape[-1] == n and _illegal(b.actions.cpu().numpy(), am) == 0
    masks_np = b.masks.cpu().numpy()
    assert (masks_np[1:] == 0).any()   # envs finished inside the rollout: hidden states zeroed mid-chunk

    # the act: log-probs of the recorded actions and rnn_states[t+1], teacher-forced from the device's own rnn_states[t]
    pol, cri = net.module.models["policy"], net.module.models["critic"]
    p = {k: v.detach().double() for k, v in rnn_ref64.unflatten(pol.flat_params.double(), tr.d, tr.n, False).items()}
    ncfg = rnn_ref64.net_cfg(cfg.activation_id, True)
    hid, mk = rnn_ref64.rows(b.rnn_states).double(), rnn_ref64.rows(b.masks).double()
    with torch.no_grad():
        feat, hn = nets_policy_features(p, ncfg, rnn_ref64.rows(b.policy_obs).double()[:T * B], hid[:T * B].unsqueeze(1), mk[:T * B])
        logits = nets_logits(p, feat, rnn_ref64.rows(b.action_masks).double()[:T * B])
        lp = logits.gather(-1, rnn_ref64.rows(b.actions).long())
    np.testing.assert_allclose(rnn_ref64.rows(b.action_log_probs).cpu().numpy(), lp.cpu().numpy(), rtol=0, atol=ATOL)
    np.testing.assert_allclose(hid[B:].cpu().numpy(), (hn[:, 0] * (mk[B:] != 0)).cpu().numpy(), rtol=0, atol=ATOL)

    # the update: one minibatch of every chunk
    m = tr.algo_module
    op, oc = m.optimizers["policy"], m.optimizers["critic"]
    vn = cri.value_normalizer
    live = dict(pol=pol.flat_params, cri=cri.flat_params, pol_m=op.exp_avg, pol_v=op.exp_avg_sq, cri_m=oc.exp_avg,
                cri_v=oc.exp_avg_sq, **({"vn": vn.state} if vn is not None else {}))
    state = dict({k: v.clone() for k, v in live.items()}, steps=[int(x) for x in m.adam_steps])
    assert state["steps"][0] > 0
    total = T * B // L
    ids = torch.randperm(total, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3 + seed)).contiguous()
    need = int(tr._lib.orl_rnn_workspace_floats_for(total * L, tr.rnn_stride, n))
    assert need == total * L * (tr._lib.orl_rnn_tape_width() + 64) + -(-total * L // 1024) * tr.rnn_stride
    tr.tape = torch.empty(need, dtype=torch.float32, device="cuda")
    tr.sync_lrs()
    a = tr._rnn_args(b, ids, b.gae_stats[5:8])
    grads, la, after = drive(a, tr.rnn_grads, tr.loss_acc, live)
    tr.tape = None
    np_, nc = int(pol.flat_params.numel()), int(cri.flat_params.numel())
    k = dict(grad_pol=grads[0, :np_], grad_cri=grads[1, :nc], losses=la, steps=[int(x) for x in m.adam_steps], **after)
    rcfg = types.SimpleNamespace(**vars(cfg), vn_beta=vn.beta if vn is not None else 0.99999)
    dims = (tr.d, tr.n, tr.dc)
    r64, r32 = (rnn_ref64_masked.update(rcfg, c3_buf(b), state, ids, L, dims, b.action_masks, dtype=dt)
                for dt in (torch.float64, torch.float32))
    print(f"\n  {case}: {total} chunks, {total * L} row-steps")
    if legal == "one":   # no policy gradient and no entropy: only the critic learns
        assert float(k["grad_pol"].abs().max()) == 0.0 and float(k["losses"][1]) == 0.0
    _compare(case, dims, k, r64, r32, state, cfg)
    torch.cuda.empty_cache()


def _compare(case, dims, k, r64, r32, state, cfg):
    """scale_harness.rnn_compare with exp_avg measured against the magnitude of the terms the Adam step combines into it
    (moment_scale), as the feed-forward scale tests measure it: after the warm-up step exp_avg = 0.9 m + 0.1 g mixes terms
    of both signs, and a one-element block such as the critic's output bias can cancel to far below its terms."""
    d, n, dc = dims
    chk = Checker(case, RNN_FLOOR)
    nets = (("pol", d, n, False), ("cri", dc, 1, True))
    for net, dd, nn, critic in nets:
        for name, s in rnn_ref64.blocks(dd, nn, critic).items():
            chk(f"grad {net}.{name}", k["grad_" + net][s], r64["grad_" + net][s], r32["grad_" + net][s])
    for i, name in enumerate(("policy loss", "entropy", "ratio sum", "value loss")):
        chk(f"loss_acc[{i}] {name}", k["losses"][i:i + 1], r64["losses"][i:i + 1], r32["losses"][i:i + 1],
            scale=r64["loss_scales"][i])
    mscale = {net: moment_scale(cfg, r64["grad_" + net], r64["norms"][j], state[net], state[net + "_m"])
              for j, net in enumerate(("pol", "cri"))}
    for net, dd, nn, critic in nets:
        for key in ("", "_m", "_v"):
            for name, s in rnn_ref64.blocks(dd, nn, critic).items():
                chk(f"{net}{key or '_param'} {name}", k[net + key][s], r64[net + key][s], r32[net + key][s],
                    scale=mscale[net][s].norm() if key == "_m" else None)
    if cfg.use_valuenorm:
        chk("vn_state", k["vn"], r64["vn"], r32["vn"])
    assert k["steps"] == [r64["pol_step"], r64["cri_step"]]
    chk.done()


def nets_policy_features(*a):
    from oracle import nets

    return nets.policy_features(*a)


def nets_logits(*a):
    from oracle import nets

    return nets.categorical_logits(*a)


WIDE = [(n, d) for n in (9, 12, 17, 33, 64) for d in (9, 64)]


@pytest.mark.parametrize("n,d", WIDE, ids=[f"n{n}-d{d}" for n, d in WIDE])
def test_wide_gru_update_matches_float64(cuda, no_tf32, n, d):
    """Head widths on both sides of the 4-wide (pad4) and 16-wide (tape GEMM M tile) edges at obs widths 9 and 64:
    64 envs x 48 steps, chunks of 3 (3072 row-steps, three tape row blocks)."""
    _run(f"wide-gru-n{n}-d{d}", n, d, 64, 48, 3, seed=n + d)


ROWS = [(1, 89, 23), (3, 341, 3), (3, 683, 3), (32, 64, 32)]


@pytest.mark.parametrize("L,N,T", ROWS, ids=[f"L{L}-rows{N * T}" for L, N, T in ROWS])
def test_wide_gru_update_chunks_and_row_blocks(cuda, no_tf32, L, N, T):
    """Chunk lengths 1, 3 and 32 at 2047, 1023, 2049 and 2048 row-steps (tape row blocks of 1024 rows), n = 33."""
    _run(f"wide-gru-L{L}-rows{N * T}", 33, 17, N, T, L, seed=L)


@pytest.mark.parametrize("legal", ["one", "all"])
def test_wide_gru_update_mask_edges(cuda, no_tf32, legal):
    """n = 64 with one legal action per row (no policy gradient, zero entropy) and with every action legal."""
    _run(f"wide-gru-n64-{legal}-legal", 64, 27, 64, 32, 4, legal=legal, seed=5)


# the options of tests/test_ppo_flags_cuda.py but A2C, whose loss rnn_ref64 does not build (the recurrent update takes it only
# through A2CAlgorithm, which the chunk kernel serves with the same pg_term branch as the feed-forward one)
PPO_CASES = [c for c in CASES if c != ["A2C"]]


@pytest.mark.parametrize("flags", PPO_CASES, ids=[" ".join(c) or "default" for c in PPO_CASES])
def test_wide_gru_update_flag_sweep(cuda, no_tf32, flags):
    """Every PPO option of tests/test_ppo_flags_cuda.py at n = 64, d = 27."""
    _run("wide-gru-n64-flags-" + ("-".join(flags) or "default"), 64, 27, 64, 32, 4, extra=flags, seed=77)


def test_wide_gru_smac_3m_shaped(cuda, no_tf32):
    """SMAC 3m's shapes: 3 agents, policy obs 30, a Dict critic obs of 48, 9 actions with (A, n) masks, chunks of 8."""
    _run("wide-gru-smac-3m", 9, 30, 128, 16, 8, A=3, dc=48, seed=3)


# ---------------------------------------------------------------- the sampler ---------------------------------------

@pytest.fixture(scope="module")
def wide_gru_agent():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    cfg, net, agent = make_agent(_venv(_WideHost(16, 64, 64)), ["--seed", "9", "--episode_length", "8",
                                                                   *WIDE_GRU])
    _sharpen(net, 1)
    return cfg, net, agent


def _rows64(rows, seed):
    rng = np.random.default_rng(seed)
    obs = rng.standard_normal((rows, 64)).astype(np.float32)
    h = (0.5 * rng.standard_normal((rows, 1, 64))).astype(np.float32)
    mk = (rng.random((rows, 1)) < 0.8).astype(np.float32)
    m = (rng.random((rows, 64)) < 0.5).astype(np.float32)
    m[np.arange(rows), rng.integers(0, 64, rows)] = 1.0
    m[::7] = 1.0                       # some rows all legal
    m[3::11] = 0.0                     # and some with a single legal action
    m[np.arange(3, rows, 11), rng.integers(0, 64, len(range(3, rows, 11)))] = 1.0
    return obs, h, mk, m


def _forward64(net, obs, h, mk, m):
    """float64 log-softmax of the masked logits and next hidden states of rows (obs, h, mk)."""
    pol = net.module.models["policy"]
    p = {k: v.detach().double() for k, v in rnn_ref64.unflatten(pol.flat_params.double(), 64, 64, False).items()}
    ncfg = rnn_ref64.net_cfg(pol.activation_id, True)
    c = lambda x: torch.from_numpy(x).cuda().double()  # noqa: E731
    with torch.no_grad():
        feat, hn = nets_policy_features(p, ncfg, c(obs), c(h), c(mk))
        return nets_logits(p, feat, c(m)), hn


@pytest.mark.parametrize("rows", [300, 4096])
def test_wide_gru_act_matches_float64_and_host_philox(wide_gru_agent, rows):
    """n = 64 on one warp per row (300 rows) and on two (4096 rows): log-probs and next hidden states against float64,
    legal actions only, and every action the argmax of p / q with q = -log U from the host Philox of (seed, step, row)
    on lanes 0, 1 (actions 0..7) and 8..21 (actions 8..63), wherever the top two ratios are apart by more than 1e-4."""
    cfg, net, agent = wide_gru_agent
    obs, h, mk, m = _rows64(rows, rows)
    logp64, hn64 = _forward64(net, obs, h, mk, m)
    seed, step = 4242, 17
    acts, lp, hn = net.module.act(obs, rnn_states_actor=torch.from_numpy(h), masks=torch.from_numpy(mk), action_masks=m,
                                  rng_seed=seed, rng_step=step)
    a = acts[:, 0].long()
    assert (torch.from_numpy(m).cuda()[torch.arange(rows, device="cuda"), a] == 1).all()
    assert int(a.max()) >= 32
    np.testing.assert_allclose(lp[:, 0].cpu().numpy(), logp64.gather(-1, a[:, None])[:, 0].cpu().numpy(), rtol=0, atol=ATOL)
    np.testing.assert_allclose(torch.as_tensor(hn).reshape(rows, 64).cpu().numpy(), hn64.reshape(rows, 64).cpu().numpy(),
                               rtol=0, atol=ATOL)
    u = philox_units(1, rows, seed, step, 0, WIDE_LANES)[0]
    q = -np.log(u.astype(np.float64))
    ratio = np.exp(logp64.cpu().numpy()) / q
    srt = np.sort(ratio, axis=-1)
    clear = (srt[:, -1] - srt[:, -2]) > 1e-4 * srt[:, -1]
    assert clear.mean() > 0.99
    got = a.cpu().numpy()
    assert np.array_equal(got[clear], ratio.argmax(-1)[clear])


def test_wide_gru_deterministic_act_picks_first_max(wide_gru_agent):
    """Deterministic mode is the first maximum of the masked probabilities; with head rows 20 and 50 copies of row 40, a
    row whose top action is one of them takes 20."""
    cfg, net, agent = wide_gru_agent
    rows = 1024
    obs, h, mk, m = _rows64(rows, 2)
    th, tmk = torch.from_numpy(h), torch.from_numpy(mk)
    acts, _, _ = net.module.act(obs, rnn_states_actor=th, masks=tmk, action_masks=m, deterministic=True)
    want = _forward64(net, obs, h, mk, m)[0].float().argmax(-1)
    assert float((acts[:, 0].long() == want).float().mean()) > 0.999
    pol = net.module.models["policy"]
    w, bias = pol.state_dict()["act.action_out.linear.weight"], pol.state_dict()["act.action_out.linear.bias"]
    saved = w.clone(), bias.clone()
    try:
        with torch.no_grad():
            w[20].copy_(w[40]); w[50].copy_(w[40]); bias[20] = bias[40]; bias[50] = bias[40]
        acts, _, _ = net.module.act(obs, rnn_states_actor=th, masks=tmk, action_masks=np.ones_like(m), deterministic=True)
        got = acts[:, 0].long().cpu().numpy()
        assert not ((got == 40) | (got == 50)).any()
        assert (got == 20).any()
    finally:
        with torch.no_grad():
            w.copy_(saved[0]); bias.copy_(saved[1])


def test_wide_gru_sampling_matches_softmax_chi_square(wide_gru_agent):
    """Philox sampling at n = 64: 200000 draws of one row (masks leave 48 legal actions) against its float64 softmax,
    one fixed-seed chi-square test over the legal actions with expected count >= 5."""
    from scipy import stats

    cfg, net, agent = wide_gru_agent
    rows = 200000
    obs1, h1, mk1, m1 = _rows64(8, 3)
    m1 = m1[:1].copy()
    m1[0] = 1.0
    m1[0, :16] = 0.0
    rep = lambda x: np.repeat(x[:1], rows, axis=0)  # noqa: E731
    acts, _, _ = net.module.act(rep(obs1), rnn_states_actor=torch.from_numpy(rep(h1)), masks=torch.from_numpy(rep(mk1)),
                                action_masks=rep(m1), rng_seed=12345, rng_step=0)
    counts = np.bincount(acts[:, 0].long().cpu().numpy(), minlength=64)
    assert counts[:16].sum() == 0
    p = _forward64(net, obs1[:1], h1[:1], mk1[:1], m1)[0].exp()[0].cpu().numpy()
    exp = p * rows
    keep = exp >= 5
    assert keep.sum() > 10
    chi2 = ((counts[keep] - exp[keep]) ** 2 / exp[keep]).sum()
    pval = stats.chi2.sf(chi2, int(keep.sum()) - 1)
    print(f"\n  chi-square {chi2:.1f} over {int(keep.sum())} actions, p = {pval:.3f}")
    assert pval > 1e-3, (chi2, pval)


def test_wide_gru_host_loops_legal_and_agree(cuda):
    """1024 envs, T = 128, n = 64, Philox sampling: no illegal action in either host loop, and the synchronous and the
    two-group loop write the same bits over two iterations with an update between them."""
    N, T = 1024, 128
    flags = ["--seed", "3", "--episode_length", str(T), "--ppo_epoch", "1", "--num_mini_batch", "2", "--log_interval", "1",
             *WIDE_GRU, "--data_chunk_length", "8"]
    runs, init = [], None
    for grouped in (False, True):
        env = _venv(_WideHost(N, 64, 27, seed=11))
        assert env.supports_groups
        cfg, net, agent = make_agent(env, flags + ["--host_env_groups", "true" if grouped else "false"], like=init)
        if init is None:
            _sharpen(net, 2)
            init = {mk: {k: v.clone() for k, v in net.module.models[mk].state_dict().items()} for mk in ("policy", "critic")}
        drv, b = agent.driver, agent.driver.buffer.data
        bufs = []
        for it in range(2):
            drv.episode = it
            drv.actor_rollout()
            torch.cuda.synchronize()
            bufs.append({k: getattr(b, k).cpu().numpy().copy()
                         for k in ("actions", "action_log_probs", "policy_obs", "masks", "rewards", "action_masks", "rnn_states")})
            assert _illegal(bufs[-1]["actions"], bufs[-1]["action_masks"]) == 0
            assert bufs[-1]["actions"].max() >= 56
            drv.compute_returns()
            torch.manual_seed(7)
            drv.trainer.train(b)
            b.after_update()
        runs.append(bufs)
    for it in range(2):
        for k in runs[0][it]:
            assert np.array_equal(runs[0][it][k], runs[1][it][k]), (it, k)


def test_wide_gru_agent_act_and_evaluate_policy(cuda):
    """PPOAgent.act and evaluate_policy run a wide GRU policy on host envs: legal actions only, hidden states carried."""
    from openrl_b200.utils.evaluation import evaluate_policy

    env = _venv(_WideHost(8, 40, 12, seed=4))
    cfg, net, agent = make_agent(env, ["--seed", "1", "--episode_length", "8", *WIDE_GRU])
    agent.net.reset()
    obs, infos = env.reset(seed=2)
    for _ in range(5):   # the env asserts that every action is legal under the masks it reported
        acts, _ = agent.act(obs, info=infos, deterministic=False)
        assert np.asarray(acts).shape[:2] == (8, 1)
        obs, _, _, infos = env.step(acts)
    # evaluate_policy passes no infos: an env whose every action is legal
    mean, std = evaluate_policy(agent, _venv(_WideHost(8, 40, 12, legal="all", seed=5)), n_eval_episodes=4)
    assert np.isfinite(mean) and np.isfinite(std)


# ---------------------------------------------------------------- refusals -----------------------------------------

def test_wide_gru_refuses_joint_action_loss(cuda):
    """JRPO keeps the 8-action limit: a wide head with use_joint_action_loss raises NotImplementedError."""
    env = _venv(_WideHost(4, 9, 6, A=3))
    with pytest.raises(NotImplementedError, match="JRPO.*up to 8 actions"):
        make_agent(env, ["--seed", "1", "--episode_length", "8", *WIDE_GRU,
                         "--use_joint_action_loss", "true"])
