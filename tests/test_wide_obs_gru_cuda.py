"""Observations of 65..256 features on GRU policies and critics (cfg.use_wide_recurrent_observations): the host act
(rnn_act_rows_warp_kernel<R, NB, 256>), the recurrent critic (rnn_critic_warp_kernel<256>), the chunked update
(rnn_chunk_warp_kernel<POLICY, false, R, NB, 256>, its tape rows with the X field and the 64-column dW1 panels) and the insert of
critic sections wider than 64 (orl_host_insert_rnn_wide_obs).

Bars: one update over the whole buffer of a host rollout against rnn_ref64 driven with the masks (tests/rnn_ref64_masked.py)
through tests/scale_harness.py at RNN_FLOOR, after a warm-up step, for widths on both sides of the 4-, 64- and 128-wide
edges and at the shared-memory edge of the wide head's two rows per warp (d = 240 / 241), chunk lengths 1, 3 and 32,
row counts at and beside the tape's 1024-row blocks, either net wide alone, one-legal and all-legal masks and every loss
option at one wide shape; two runs bit for bit; the same rollout's act and critic teacher-forced against float64 row by
row at ATOL; each Philox-sampled action against argmax(p / q) with q from the host Philox; the first-max mode; the
insert bit for bit; a SMAC-8m-shaped env end to end in both host loops; and the reference's traces
(tests/golden/trace_wide_obs_gru_{dict,box_256}.npz) through PPOAgent in parity mode."""
import types

import numpy as np
import pytest
import torch

import rnn_ref64
import rnn_ref64_masked
from helpers import make_agent, philox_units
from scale_harness import ATOL, CASES, RNN_FLOOR, Checker, c3_buf, drive, moment_scale, no_tf32  # noqa: F401  (no_tf32: fixture)

pytestmark = pytest.mark.gpu

# a GRU policy of 1..64 actions over observations of 1..256 features
WIDE_OBS_GRU = ["--use_recurrent_policy", "true", "--use_wide_recurrent_head", "true", "--use_wide_recurrent_observations", "true"]
# Philox lanes of a head's actions: 0, 1 for actions 0..7, 8..21 for actions 8..63 (orl_envstep.cuh)
LANES = [0, 1] + list(range(8, 22))


class _WideHost:
    """N envs x A agents, observations (A, d) ~ N(0, 1) (or a Dict {"policy": (A, d), "critic": (A, dc)}), Discrete(n) with
    per-agent (A, n) masks in `info["action_masks"]`: "random" (each action legal with probability 0.5, the agent's
    first row of every eight with a single legal action, another with all legal), "one" or "all".  An env finishes
    with probability 0.15 per step.  Every draw is keyed by (env, the env's step count), so a sub-range step
    (`step_range`) returns what the whole-range step would."""

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

    return HostVecEnv(host, wide_observations=True)


def _illegal(actions, action_masks):
    a = actions[..., 0].astype(np.int64)
    return int((np.take_along_axis(action_masks[:-1], a[..., None], axis=-1) == 0).sum())


def _sharpen(net, seed):
    """Head weights well above the init's 0.01 gain, so that the softmax is far from uniform."""
    pol = net.module.models["policy"]
    with torch.no_grad():
        pol.state_dict()["act.action_out.linear.weight"].normal_(0.0, 0.5, generator=torch.Generator(device="cuda").manual_seed(seed))


def _policy_features(*a):
    from oracle import nets

    return nets.policy_features(*a)


def _logits(*a):
    from oracle import nets

    return nets.categorical_logits(*a)


def _critic_forward(*a):
    from oracle import nets

    return nets.critic_forward(*a)


# ---------------------------------------------------------------- the reference's traces ------------------------------

@pytest.mark.parametrize("tag", ["wide_obs_gru_dict", "wide_obs_gru_box_256"])
def test_reproduces_reference_trace(cuda, tag):
    """PPOAgent over make()'s host vec-env in parity mode against the reference's recurrent runs on the envs of
    tests/wide_obs_gru_oracle.py: SMAC 8m's shapes with masks (use_recurrent_policy) and Box(256) observations with
    Discrete(5) (use_naive_recurrent_policy).  Actions bit for bit; log-probs, hidden states and values 2e-5, the update
    scalars 2e-4, the parameters after the last iteration (the traces keep no earlier ones) 2e-3."""
    import os

    from conftest import GOLDEN
    from helpers import KEYS
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.common import make
    from wide_obs_gru_oracle import SpacedMaskedWideDictTargetEnv, SpacedWideBoxDiscreteEnv

    d = np.load(os.path.join(GOLDEN, f"trace_{tag}.npz"), allow_pickle=True)
    iters, N = int(d["meta/iters"]), int(d["meta/env_num"])
    flags = str(d["meta/flags"]).split() + ["--parity_mode", "true", "--log_interval", "1", "--use_wide_recurrent_head", "true",
                                            "--use_wide_recurrent_observations", "true"]
    dict_obs = tag == "wide_obs_gru_dict"
    cls = SpacedMaskedWideDictTargetEnv if dict_obs else SpacedWideBoxDiscreteEnv
    env = make("WideTarget", env_num=N, make_custom_envs=lambda id, env_num, render_mode=None, **kw: [cls for _ in range(env_num)],
               cfg=create_config_parser().parse_args(flags))
    assert (env.obs_dim, env.critic_obs_dim) == ((80, 168) if dict_obs else (256, 256))
    cfg, net, agent = make_agent(env, flags, golden=d)
    drv, tr = agent.driver, agent.driver.trainer
    b = drv.buffer.data
    assert drv.recurrent and tr.n == (14 if dict_obs else 5)
    for it in range(iters):
        t = f"it{it}"
        drv.episode = it
        drv.actor_rollout()
        assert np.array_equal(b.actions.cpu().numpy(), d[f"{t}/actions"]), t
        assert np.array_equal(b.policy_obs.cpu().numpy(), d[f"{t}/policy_obs"]), t
        assert np.array_equal(b.masks.cpu().numpy(), d[f"{t}/masks"]), t
        if dict_obs:
            assert not b.action_masks_trivial
            assert np.array_equal(b.critic_obs.cpu().numpy(), d[f"{t}/critic_obs"]), t
            assert np.array_equal(b.action_masks.cpu().numpy(), d[f"{t}/action_masks"]), t
        np.testing.assert_allclose(b.action_log_probs.cpu().numpy(), d[f"{t}/action_log_probs"], rtol=0, atol=2e-5, err_msg=t)
        np.testing.assert_allclose(b.rnn_states.cpu().numpy(), d[f"{t}/rnn_states"], rtol=0, atol=2e-5, err_msg=t)
        drv.compute_returns()
        np.testing.assert_allclose(b.rnn_states_critic.cpu().numpy(), d[f"{t}/rnn_states_critic"], rtol=0, atol=2e-5, err_msg=t)
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
                    np.testing.assert_allclose(v.cpu().numpy(), d[gk], rtol=2e-3, atol=2e-5, err_msg=gk)
                    checked += 1
        assert checked > 0 or it < iters - 1, t
        b.after_update()


# ---------------------------------------------------------------- the update (and the rollout's act and critic) -------

def _run(case, n, d, N, T, L, A=1, dc=None, legal="random", extra=(), seed=0, twice=False):
    """A host rollout of N envs x A agents x T steps with a wide-observation GRU policy (Philox sampling); its act and critic
    teacher-forced against float64; then one update over every chunk of the buffer against rnn_ref64 with the masks.
    twice: the update runs again from the same state and must give the same bits."""
    flags = ["--seed", str(6 + seed), *WIDE_OBS_GRU, "--episode_length", str(T), "--data_chunk_length", str(L),
             "--ppo_epoch", "1", "--num_mini_batch", "1", "--use_valuenorm", "true", "--host_env_groups", "false", *extra]
    host = _WideHost(N, n, d, A=A, dc=dc, legal=legal, seed=seed)
    cfg, net, agent = make_agent(_venv(host), flags)
    _sharpen(net, seed)
    drv, tr, b = agent.driver, agent.driver.trainer, agent.driver.buffer.data
    assert (tr.d, tr.dc, tr.n) == (d, dc or d, n) and drv.recurrent
    drv.actor_rollout()   # warm-up: the compared update is a second Adam step, with nonzero moments
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
    mk = rnn_ref64.rows(b.masks).double()
    assert (b.masks[1:] == 0).any()   # hidden states zeroed mid-chunk

    # the act: log-probs of the recorded actions and rnn_states[t+1], teacher-forced from the device's own rnn_states[t]
    pol, cri = net.module.models["policy"], net.module.models["critic"]
    p = {k: v.detach().double() for k, v in rnn_ref64.unflatten(pol.flat_params.double(), tr.d, tr.n, False).items()}
    ncfg = rnn_ref64.net_cfg(cfg.activation_id, True)
    hid = rnn_ref64.rows(b.rnn_states).double()
    with torch.no_grad():
        feat, hn = _policy_features(p, ncfg, rnn_ref64.rows(b.policy_obs).double()[:T * B], hid[:T * B].unsqueeze(1), mk[:T * B])
        lp = _logits(p, feat, rnn_ref64.rows(b.action_masks).double()[:T * B]).gather(-1, rnn_ref64.rows(b.actions).long())
    np.testing.assert_allclose(rnn_ref64.rows(b.action_log_probs).cpu().numpy(), lp.cpu().numpy(), rtol=0, atol=ATOL)
    np.testing.assert_allclose(hid[B:].cpu().numpy(), (hn[:, 0] * (mk[B:] != 0)).cpu().numpy(), rtol=0, atol=ATOL)
    # the critic over slots 0..T, teacher-forced: value_preds[t] from rnn_states_critic[t], which is zeroed at dones
    pc = {k: v.detach().double() for k, v in rnn_ref64.unflatten(cri.flat_params.double(), tr.dc, 1, True).items()}
    hc = rnn_ref64.rows(b.rnn_states_critic).double()
    with torch.no_grad():
        v64, hcn = _critic_forward(pc, ncfg, rnn_ref64.rows(b.critic_obs).double(), hc.unsqueeze(1), mk)
    if not cfg.use_valuenorm:   # with ValueNorm, value_preds hold the denormalised values
        np.testing.assert_allclose(rnn_ref64.rows(b.value_preds).double().cpu().numpy(), v64.cpu().numpy(), rtol=0, atol=ATOL)
    np.testing.assert_allclose(hc[B:].cpu().numpy(), (hcn[:T * B, 0] * (mk[B:] != 0)).cpu().numpy(), rtol=0, atol=ATOL)
    zeroed = (mk[B:] == 0)[:, 0]
    assert zeroed.any() and float(hc[B:][zeroed].abs().max()) == 0.0

    # the update: one minibatch of every chunk
    m = tr.algo_module
    op, oc = m.optimizers["policy"], m.optimizers["critic"]
    vn = cri.value_normalizer
    live = dict(pol=pol.flat_params, cri=cri.flat_params, pol_m=op.exp_avg, pol_v=op.exp_avg_sq, cri_m=oc.exp_avg,
                cri_v=oc.exp_avg_sq, **({"vn": vn.state} if vn is not None else {}))
    state = dict({k: v.clone() for k, v in live.items()}, steps=[int(x) for x in m.adam_steps])
    total = T * B // L
    ids = torch.randperm(total, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3 + seed)).contiguous()
    need = int(tr._lib.orl_rnn_workspace_floats_wide_obs(total * L, tr.rnn_stride, n, tr.d, tr.dc))
    tw = max(tr._lib.orl_rnn_tape_width() + (64 if n > 8 else 0) + (256 if tr.d > 64 else 0),
             tr._lib.orl_rnn_tape_width() + (256 if tr.dc > 64 else 0))
    assert need == total * L * tw + -(-total * L // 1024) * tr.rnn_stride + 64 * 256
    tr.tape = torch.empty(need, dtype=torch.float32, device="cuda")
    tr.sync_lrs()
    a = tr._rnn_args(b, ids, b.gae_stats[5:8])
    grads, la, after = drive(a, tr.rnn_grads, tr.loss_acc, live)
    if twice:
        steps = [int(x) for x in m.adam_steps]
        for k, v in live.items():
            v.copy_(state[k])
        for i, s in enumerate(state["steps"]):
            m.adam_steps[i] = s
        tr.tape.fill_(float("nan"))   # nothing of the first run's workspace is read
        g2, la2, after2 = drive(a, tr.rnn_grads, tr.loss_acc, live)
        assert torch.equal(grads, g2)
        np.testing.assert_allclose(la.cpu().numpy(), la2.cpu().numpy(), rtol=1e-6, atol=1e-7)   # float-atomic sums over the CTAs
        assert all(torch.equal(after[k], after2[k]) for k in after)
        assert [int(x) for x in m.adam_steps] == steps
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
    """Every gradient block, loss sum, parameter block and Adam moment at RNN_FLOOR; exp_avg against the magnitude of the
    terms the Adam step combines into it (moment_scale)."""
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


GRID = [(d, n) for d in (65, 68, 127, 128, 129, 240, 241, 255, 256) for n in (5, 64)]


@pytest.mark.parametrize("d,n", GRID, ids=[f"d{d}-n{n}" for d, n in GRID])
def test_update_at_width_edges(cuda, no_tf32, d, n):
    """Both nets d wide (a flat Box), heads of 5 (NB = 8) and 64 (NB = 64) actions: pad4, the 64-column panel edges and,
    for the wide head, the switch from two rows per warp to one between d = 240 and 241.  64 envs x 48 steps, chunks of 3
    (3072 row-steps, three tape row blocks)."""
    _run(f"d{d}-n{n}", n, d, 64, 48, 3, seed=d + n)


ROWS = [(1, 89, 23), (3, 341, 3), (3, 683, 3), (32, 64, 32)]


@pytest.mark.parametrize("L,N,T", ROWS, ids=[f"L{L}-rows{N * T}" for L, N, T in ROWS])
def test_update_chunks_and_row_blocks(cuda, no_tf32, L, N, T):
    """Chunk lengths 1, 3 and 32 at 2047, 1023, 2049 and 2048 row-steps (tape row blocks of 1024 rows), d = 129, n = 14."""
    _run(f"L{L}-rows{N * T}", 14, 129, N, T, L, seed=L)


ONE = [(216, 18), (18, 216), (216, 216)]


@pytest.mark.parametrize("d,dc", ONE, ids=[f"d{d}-dc{dc}" for d, dc in ONE])
def test_update_one_net_wide(cuda, no_tf32, d, dc):
    """A Dict observation with only the policy wide, only the critic wide, and both; 3 agents, 14 actions."""
    _run(f"d{d}-dc{dc}", 14, d, 32, 16, 8, A=3, dc=dc, seed=dc)


def test_update_shared_memory_worst_case(cuda, no_tf32):
    """d = dc = 256 with 64 actions: the wide head at one row per warp, the critic at two."""
    _run("worst-case", 64, 256, 32, 16, 8, A=2, dc=256, seed=11)


@pytest.mark.parametrize("legal", ["one", "all"])
def test_update_mask_edges(cuda, no_tf32, legal):
    """SMAC 8m's shapes with one legal action per row (no policy gradient, zero entropy) and with every action legal."""
    _run(f"8m-{legal}-legal", 14, 80, 16, 16, 8, A=8, dc=168, legal=legal, seed=5)


PPO_CASES = [c for c in CASES if c != ["A2C"]]


@pytest.mark.parametrize("flags", PPO_CASES, ids=[" ".join(c) or "default" for c in PPO_CASES])
def test_update_flag_sweep(cuda, no_tf32, flags):
    """Every PPO option of tests/test_ppo_flags_cuda.py (A2C aside: rnn_ref64 builds no A2C loss) at d = 168, n = 14."""
    _run("flags-" + ("-".join(flags) or "default"), 14, 168, 64, 32, 4, extra=flags, seed=77)


def test_update_is_deterministic(cuda, no_tf32):
    """SMAC 8m's shapes: two updates from the same state give the same bits (the tape reductions sum in a fixed order)."""
    _run("8m-twice", 14, 80, 16, 16, 8, A=8, dc=168, seed=21, twice=True)


# ---------------------------------------------------------------- the act, row by row ---------------------------------

def _rows(rows, d, n, seed):
    rng = np.random.default_rng(seed)
    obs = rng.standard_normal((rows, d)).astype(np.float32)
    h = (0.5 * rng.standard_normal((rows, 1, 64))).astype(np.float32)
    mk = (rng.random((rows, 1)) < 0.8).astype(np.float32)
    m = (rng.random((rows, n)) < 0.5).astype(np.float32)
    m[np.arange(rows), rng.integers(0, n, rows)] = 1.0
    m[::7] = 1.0
    return obs, h, mk, m


ACT = [(d, n, rows) for d in (65, 129, 256) for n in (5, 64) for rows in (300, 4096)]


@pytest.mark.parametrize("d,n,rows", ACT, ids=[f"d{d}-n{n}-rows{r}" for d, n, r in ACT])
def test_act_matches_float64_and_host_philox(cuda, d, n, rows):
    """PPOModule.act at one row per warp (300 rows) and two (4096; one at d = 256 with 64 actions): log-probs and next
    hidden states against float64, legal actions only, and every action the argmax of p / q with q = -log U from the host
    Philox wherever the top two ratios are apart by more than 1e-4; deterministic mode is the first maximum."""
    cfg, net, agent = make_agent(_venv(_WideHost(16, n, d)), ["--seed", "9", "--episode_length", "8", *WIDE_OBS_GRU])
    _sharpen(net, d + n)
    obs, h, mk, m = _rows(rows, d, n, rows + d)
    pol = net.module.models["policy"]
    p = {k: v.detach().double() for k, v in rnn_ref64.unflatten(pol.flat_params.double(), d, n, False).items()}
    c = lambda x: torch.from_numpy(x).cuda().double()  # noqa: E731
    with torch.no_grad():
        feat, hn64 = _policy_features(p, rnn_ref64.net_cfg(pol.activation_id, True), c(obs), c(h), c(mk))
        logp64 = _logits(p, feat, c(m))
    seed, step = 4242, 17
    acts, lp, hn = net.module.act(obs, rnn_states_actor=torch.from_numpy(h), masks=torch.from_numpy(mk), action_masks=m,
                                  rng_seed=seed, rng_step=step)
    a = acts[:, 0].long()
    assert (torch.from_numpy(m).cuda()[torch.arange(rows, device="cuda"), a] == 1).all()
    np.testing.assert_allclose(lp[:, 0].cpu().numpy(), logp64.gather(-1, a[:, None])[:, 0].cpu().numpy(), rtol=0, atol=ATOL)
    np.testing.assert_allclose(torch.as_tensor(hn).reshape(rows, 64).cpu().numpy(), hn64.reshape(rows, 64).cpu().numpy(),
                               rtol=0, atol=ATOL)
    u = philox_units(1, rows, seed, step, 0, LANES)[0][:, :n]
    ratio = np.exp(logp64.cpu().numpy()) / -np.log(u.astype(np.float64))
    srt = np.sort(ratio, axis=-1)
    clear = (srt[:, -1] - srt[:, -2]) > 1e-4 * srt[:, -1]
    assert clear.mean() > 0.99
    assert np.array_equal(a.cpu().numpy()[clear], ratio.argmax(-1)[clear])
    det, _, _ = net.module.act(obs, rnn_states_actor=torch.from_numpy(h), masks=torch.from_numpy(mk), action_masks=m,
                               deterministic=True)
    assert float((det[:, 0].long() == logp64.float().argmax(-1)).float().mean()) > 0.999


# ---------------------------------------------------------------- the insert ------------------------------------------

def test_insert_rnn_wide_obs(cuda):
    """orl_host_insert_rnn_wide_obs on staged blocks with critic sections of 65 and 256 features (8 agents, masks of 14
    actions) writes what orl_host_insert_wide_obs writes, bit for bit, and zeroes the hidden states of the finished envs;
    it refuses critic sections of 0 and 257 features, naming 1..256."""
    from openrl_b200 import lib

    L = lib.load()
    rng = np.random.default_rng(4)
    n_envs, A, d, n = 37, 8, 80, 14
    B = n_envs * A
    for dc in (65, 256):
        obs, cri, rew = (rng.standard_normal(B * w).astype(np.float32) for w in (d, dc, 1))
        dones = (rng.random((n_envs, A)) < 0.4).astype(np.float32)
        dones[rng.random(n_envs) < 0.3] = 1.0
        am = (rng.random(B * n) < 0.5).astype(np.float32)
        blk = torch.from_numpy(np.concatenate([obs, cri, rew, dones.reshape(-1), am])).cuda()
        outs = []
        for rnn in (False, True):
            o = dict(obs=torch.full((B, d), -9.0, device="cuda"), rew=torch.full((B,), -9.0, device="cuda"),
                     masks=torch.full((B,), -9.0, device="cuda"), active=torch.full((B,), -9.0, device="cuda"),
                     am=torch.full((B, n), -9.0, device="cuda"), cri=torch.full((B, dc), -9.0, device="cuda"),
                     h=torch.full((B, 64), 5.0, device="cuda"))
            head = (lib.ptr(blk), n_envs, A, d, lib.ptr(o["obs"]), lib.ptr(o["rew"]), lib.ptr(o["masks"]), lib.ptr(o["active"]))
            tail = (lib.ptr(o["am"]), n, lib.ptr(o["cri"]), dc, lib.current_stream())
            if rnn:
                assert L.orl_host_insert_rnn_wide(*head, lib.ptr(o["h"]), *tail) == 10001
                assert L.orl_host_insert_rnn_wide_obs(*head, lib.ptr(o["h"]), *tail) == 0
            else:
                assert L.orl_host_insert_wide_obs(*head, *tail) == 0
            torch.cuda.synchronize()
            outs.append({k: v.cpu().numpy() for k, v in o.items()})
        for key in ("obs", "rew", "masks", "active", "am", "cri"):
            assert np.array_equal(outs[0][key], outs[1][key]), key
        env_done = np.repeat(dones.all(1, keepdims=True), A, axis=1).reshape(-1)
        assert env_done.any() and (~env_done).any()
        assert (outs[1]["h"][env_done] == 0).all() and (outs[1]["h"][~env_done] == 5.0).all()
    p = lib.ptr(blk)
    for dc in (0, 257):
        assert L.orl_host_insert_rnn_wide_obs(p, 2, 1, 4, p, p, p, p, p, None, 0, p, dc, lib.current_stream()) == 10001
        assert b"1..256" in L.orl_last_error()


# ---------------------------------------------------------------- end to end ------------------------------------------

def test_smac_8m_shaped_env_trains_in_both_host_loops(cuda, tmp_path):
    """A SMAC-8m-shaped env (8 agents, Dict {"policy": 80, "critic": 168}, Discrete(14), masks) with a GRU MAPPO config:
    PPOAgent.train for two iterations in the synchronous and in the two-group host loop from the same weights gives the
    same buffers bit for bit; then a checkpoint round trip, PPOAgent.act and evaluate_policy."""
    from openrl_b200.envs.vec_env import HostVecEnv
    from openrl_b200.utils.evaluation import evaluate_policy
    from openrl_b200.utils.logger import Logger

    N, A, T = 16, 8, 16
    flags = WIDE_OBS_GRU + ["--seed", "2", "--episode_length", str(T), "--ppo_epoch", "2", "--num_mini_batch", "2",
                            "--data_chunk_length", "8", "--log_interval", "1"]
    runs, init = [], None
    for grouped in (False, True):
        env = HostVecEnv(_WideHost(N, 14, 80, A=A, dc=168, seed=3), wide_observations=True)
        assert (env.obs_dim, env.critic_obs_dim) == (80, 168)
        cfg, net, agent = make_agent(env, flags + ["--host_env_groups", "true" if grouped else "false"], like=init)
        if init is None:
            init = {mk: {k: v.clone() for k, v in net.module.models[mk].state_dict().items()} for mk in ("policy", "critic")}
        drv, b = agent.driver, agent.driver.buffer.data
        assert drv.recurrent and (drv.trainer.d, drv.trainer.dc, drv.trainer.n) == (80, 168, 14)
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
                                   "rewards", "action_masks", "value_preds", "returns", "rnn_states", "rnn_states_critic")})
            for k, v in bufs[-1].items():
                assert np.isfinite(v).all(), k
            assert _illegal(bufs[-1]["actions"], bufs[-1]["action_masks"]) == 0
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
    saved = {mk: {k: v.clone() for k, v in net.module.models[mk].state_dict().items()} for mk in ("policy", "critic")}
    agent.save(tmp_path / "wide_gru")
    with torch.no_grad():
        for mk in ("policy", "critic"):
            for v in net.module.models[mk].state_dict().values():
                v.zero_()
    agent.load(tmp_path / "wide_gru")
    for mk in ("policy", "critic"):
        for k, v in net.module.models[mk].state_dict().items():
            assert torch.equal(v, saved[mk][k]), (mk, k)
    obs, _ = env.reset()
    acts, states = agent.act(obs, deterministic=True)
    assert np.asarray(acts).shape[:2] == (N, A)
    mean, std = evaluate_policy(agent, HostVecEnv(_WideHost(4, 14, 80, A=A, dc=168, legal="all", seed=5), wide_observations=True),
                                n_eval_episodes=4)
    assert np.isfinite(mean) and np.isfinite(std)
