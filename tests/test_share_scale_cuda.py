"""The shared policy-value kernels (cfg.use_share_model: `share_rollout_kernel`, `share_values_kernel`,
`share_fwdbwd_kernel`, the tape reduction `orl::reduce_tape` at the shared model's tape widths 1104 and 1112, and
`share_apply_kernel`; orl_share.cu, orl_tape.cu, orl_deep_core.h) at C2 scale against a float64 reference.

Here they run (a) on a real C2 buffer (CartPole-v1, 4096 envs, T = 128, 4 epochs x 1 minibatch, Categorical head): the
rollout and value pass teacher-forced on the kernel's own actions, the four epochs on the contiguous whole-buffer path
(524 288 rows, 512 tape row blocks) and a shuffled index list with a partial last row block; (b) on a real C5-shaped
buffer (obs 17, Box(6), 1024 host-stepped envs, DiagGaussian head, 131 072 rows at the 1112-float tape width); (c) on
a GridWorld rollout at 4096 envs; (d) on synthetic buffers at the edges of the kernels' thread and tape mappings, each
named in its test id: row counts around the 1024-row tape block, observation widths 1 .. 64 (the fc1 gemm job's
N = d, zero-padded x on the tape), head widths 1 .. 8 (the head gemm's M = n, the M = 1 value job, the logstd column
job), a contiguous range that starts at row 1000, masked Categorical heads, active masks with zeros and all four
activations; (e) under every loss option of tests/test_ppo_flags_cuda.py with both heads; (f) against deliberately
wrong references (tests/share_ref64.py MUTANTS), to show that the bars catch a subtle kernel error.

The reference is tests/share_ref64.py over the oracle (oracle/ppo.py `ppo_update` with one parameter dict for both
roles), pinned to the reference's traces by tests/test_share_ref64_cpu.py.  Bars are those of
tests/scale_harness.py: per parameter block, the kernel's relative L2 error against float64 may be at most
4x the float32 reference's error against float64, clamped to [FLOOR, 1e-3]; loss sums are relative to the weighted sum
of their absolute terms and Adam's exp_avg to the terms it combines.  The parameters and Adam moments after the step are
compared with the float64 reference's, and also with the float64 step taken from the kernel's own gradient (the
optimiser kernel's error alone).

On the real buffers the references are teacher-forced on the kernel's ReLU branches where a pre-activation lies within
share_ref64.BRANCH_TIE (1e-5) of the kink, as the rollout checks are teacher-forced on the kernel's actions: a float32
dot product of 64 terms can round such a value to either side.  Measured on C2 (H100 SXM): the tape reduction adds
under 1e-7 per block, 2.5e-7 on the two-element head bias (the kernel's gradient against a float64 sum of its own tape); without the forcing, the whole
gradient error of epochs 1 and 2 came from 1 and 6 of the 33.5 million (row, unit) pairs of the common fc1 activation,
at |z| <= 6.3e-7, where the float32 rounding took the other branch (torch's float32 took it at 1 and 3 pairs).  Each
flip moves the gradient by a whole row's term; Adam's division by sqrt(exp_avg_sq) then put a LayerNorm bias 6x torch's
float32 error off.  Synthetic buffers keep every pre-activation ACT_KINK away from the kink instead.  Rollout
quantities are compared element-wise at the 2e-5 absolute bar of tests/test_gru_cuda.py.  Every case prints its kernel / float32 error ratios
(`pytest -s`).

FLOOR is 3e-6 rather than 2e-6, measured on an H100 SXM (700 W): with the dual clip at 1.05 the Gaussian logstd
gradient, a sum of per-row terms that nearly cancel, is 2.6e-6 off float64 (torch's float32 6.3e-7, bar 2.5e-6), and
its exp_avg_sq 2.4e-6.  No other check of this file needs more than 2e-6.
Every mutant below moves its quantity by far more."""
import types

import numpy as np
import pytest
import torch

import scale_harness as h
import share_ref64 as ref
from scale_harness import ATOL, BASE, CASES, Checker, no_tf32  # noqa: F401  (no_tf32: pytest fixture)

pytestmark = pytest.mark.gpu

FLOOR = 3e-6
BLOCK = ref.TAPE_ROW_BLOCK
SEED = 11
C2_FLAGS = ["--seed", "0", "--episode_length", "128", "--ppo_epoch", "4", "--num_mini_batch", "1", "--log_interval", "1000000",
            "--log_each_episode", "false", "--use_share_model", "true"]
C5_FLAGS = ["--seed", "0", "--episode_length", "128", "--ppo_epoch", "4", "--num_mini_batch", "1", "--log_interval", "1",
            "--host_env_groups", "false", "--use_share_model", "true"]


def _compare(case, dims, head, k, r64, r32, state, cfg, check_vn=True):
    chk = Checker(case, FLOOR)
    bl = ref.blocks(*dims, head)
    for name, s in bl.items():
        chk(f"grad {name}", k["grad"][s], r64["grad"][s], r32["grad"][s])
    for i, name in enumerate(("policy loss", "entropy", "ratio sum", "value loss")):
        chk(f"loss sum {name}", k["losses"][i:i + 1], r64["losses"][i:i + 1], r32["losses"][i:i + 1], scale=r64["loss_scales"][i])
    for j, name in ((0, "actor grad norm"), (1, "critic grad norm")):
        chk(f"train_info {name}", k["norms"][j:j + 1], r64["norms"][j:j + 1], r32["norms"][j:j + 1])
    chk("train_info ratio mean", k["info"][5:6], r64["ratio_mean"].reshape(1), r32["ratio_mean"].reshape(1))
    mscale = h.moment_scale(cfg, r64["grad"], r64["norms"][0], state["p"], state["m"])
    for key, label in (("p", "param"), ("m", "exp_avg"), ("v", "exp_avg_sq")):
        for name, s in bl.items():
            chk(f"{label} {name}", k[key][s], r64[key][s], r32[key][s], scale=mscale[s].norm() if key == "m" else None)
    # and the optimiser step alone, from the kernel's own gradient: share_apply_kernel's error without the gradient's
    step64, step32 = (ref.adam_from(cfg, state, k["grad"], dims, head, dt) for dt in (torch.float64, torch.float32))
    for key, label in (("p", "param"), ("m", "exp_avg"), ("v", "exp_avg_sq")):
        for name, s in bl.items():
            chk(f"step-from-kernel-grad {label} {name}", k[key][s], step64[key][s], step32[key][s],
                scale=mscale[s].norm() if key == "m" else None)
    if check_vn:
        chk("vn_state", k["vn"], r64["vn"], r32["vn"])
    assert k["step"] == r64["step"]
    chk.done()


def _check_mutant(case, mutant, k, r64, r32, bad, dims, head):
    """The kernel output against a reference with one deliberate mistake: the quantity the mistake lands in must
    violate its bar, and pass it against the correct reference."""
    what = ref.MUTANTS[mutant][1]
    got, want, wrong, w32 = (ref.target(x, what, dims, head) for x in (k, r64, bad, r32))
    good = Checker(case, FLOOR)
    good(what, got, want, w32)
    good.done()
    e_bad, bar = h.rel(got, wrong), good.bar(h.rel(w32, want))
    print(f"  {case}: kernel against the mutant {e_bad:.2e}, bar {bar:.2e} ({e_bad / bar:.1f}x the bar)")
    assert e_bad > bar, f"{mutant}: the mistake ({ref.MUTANTS[mutant][0]}) passed the bar of {what}"


def _peak(tag):
    print(f"  {tag}: peak device memory {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


# ---------------------------------------------------------------- real buffers -----------------------------------------

def _device_driver(env_id, n_envs, flags, reset_table=None):
    """PPONet + PPOAlgorithm + buffer + OnPolicyDriver on a device env; CartPole's PCG64 streams seeded as
    CartPoleVec.reset(seed=SEED) seeds them."""
    from openrl_b200.algorithms.ppo import PPOAlgorithm
    from openrl_b200.buffers import NormalReplayBuffer
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.drivers.onpolicy_driver import OnPolicyDriver
    from openrl_b200.envs.common import make
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent

    torch.manual_seed(0)
    cfg = create_config_parser().parse_args(flags)
    cfg.quiet = True
    env = make(env_id, env_num=n_envs) if reset_table is None else make(env_id, env_num=n_envs, reset_table=reset_table)
    net = PPONet(env, cfg=cfg, device="cuda:0")
    agent = PPOAgent(net)
    trainer = PPOAlgorithm(cfg, net.module, agent_num=1, device=net.device)
    buf = NormalReplayBuffer(cfg, 1, env.observation_space, env.action_space, device=net.device)
    drv = OnPolicyDriver({"cfg": cfg, "num_agents": 1, "run_dir": None, "envs": env, "device": net.device}, trainer, buf, agent)
    if env_id == "CartPole-v1":
        env._seed_streams(SEED)
    drv.reset_and_buffer_init()
    return cfg, env, net, drv


def _real(cfg, drv, head):
    """What the update tests read from a driver after a rollout and compute_returns."""
    tr, b = drv.trainer, drv.buffer.data
    m = tr.algo_module
    model, opt = m.models["model"], m.optimizers["model"]
    assert tr.share and m.models["policy"] is model and m.models["critic"] is model
    T, N = b.episode_length, b.n_rollout_threads
    rows = T * N * b.num_agents
    d, w = tr.d, b.actions.shape[-1]
    live = dict(p=model.flat_params, m=opt.exp_avg, v=opt.exp_avg_sq, vn=model.value_normalizer.state)
    buf = dict(obs=b.policy_obs.reshape(-1, d), actions=b.actions.reshape(-1, w), action_log_probs=b.action_log_probs.reshape(-1, w),
               advantages=b.advantages.reshape(-1, 1)[:rows], value_preds=b.value_preds.reshape(-1, 1),
               returns=b.returns.reshape(-1, 1), active_masks=b.active_masks.reshape(-1, 1))
    if not (b.action_masks_trivial or b.continuous):
        buf["action_masks"] = b.action_masks.reshape(-1, tr.n)
    p0 = model.flat_params.clone()
    return types.SimpleNamespace(cfg=cfg, drv=drv, tr=tr, b=b, m=m, rows=rows, dims=(d, tr.n), head=head, live=live, buf=buf,
                                 p0=p0, vn_beta=model.value_normalizer.beta)


@pytest.fixture(scope="module")
def c2():
    """One rollout of C2 with use_share_model (share_rollout_kernel<CARTPOLE>), its value pass and returns."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    cfg, env, net, drv = _device_driver("CartPole-v1", 4096, C2_FLAGS)
    drv.actor_rollout()
    drv.compute_returns()
    torch.cuda.synchronize()
    c = _real(cfg, drv, "categorical")
    assert (c.b.episode_length, c.b.n_rollout_threads, c.rows, c.dims) == (128, 4096, 524288, (4, 2))
    assert c.tr.head_kind == 0 and c.rows // BLOCK == 512
    yield c
    c.tr.share_ws = None
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def c5s():
    """One rollout of the C5-shaped host env (obs 17, Box(6), 1024 envs) with use_share_model, and its returns."""
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
    c = _real(cfg, drv, "gaussian")
    assert c.rows == 131072 and c.dims == (17, 6) and c.tr.head_kind == 1
    yield c
    c.tr.share_ws = None
    torch.cuda.empty_cache()


def _state(c):
    return dict({k: v.clone() for k, v in c.live.items()}, step=int(c.m.adam_steps[0]))


def _kernel_update(c, idx, stats, rows, critic_lr=None):
    """One PPOAlgorithm.ppo_update as train_async issues it (orl_share_fwdbwd + orl_share_apply); what is compared, and
    the kernel's own ReLU branches from its tape (dL/dz of fc1 and common fc1 is zero where the branch is off; a row of
    zero loss weight has no gradient to steer).  critic_lr: the device's second learning rate for this update (a shared
    model's sync_lrs writes lr into both slots; the shared Adam must read the first)."""
    tr = c.tr
    tr.train_info.zero_()
    tr.sync_lrs()
    saved = tr.lrs.clone()
    if critic_lr is not None:
        tr.lrs[1] = critic_lr
    tr.ppo_update(c.b, rows, idx, 0, mb_stats=stats)
    torch.cuda.synchronize()
    tr.lrs.copy_(saved)
    info = tr.train_info.clone()
    width = 1112 if c.head == "gaussian" else 1104
    tape = tr.share_ws[:rows * width].view(rows, width)
    branches = {"obs_prep": tape[:, 0:64] != 0, "common": tape[:, 128:192] != 0}
    return dict(grad=tr.share_grads[:tr.share_total].clone(), losses=tr.share_loss[:4].clone(), info=info, lrs=saved,
                norms=info[[4, 1]], step=int(c.m.adam_steps[0]), branches=branches, **{k: v.clone() for k, v in c.live.items()})


def _refs(c, k, state, rows_idx, opts=None, mutant=None):
    """float64 and float32 references (and a mutant) teacher-forced on the kernel's branches at ReLU ties."""
    rcfg = types.SimpleNamespace(**{**vars(c.cfg), **(opts or {})})
    kw = dict(vn_beta=c.vn_beta, branches=k["branches"])
    out = [ref.update(rcfg, c.buf, state, rows_idx, c.dims, c.head, dt, **kw) for dt in (torch.float64, torch.float32)]
    if mutant is not None:
        out.append(ref.update(rcfg, c.buf, state, rows_idx, c.dims, c.head, torch.float64, mutant=mutant, **kw))
    return out


def _forward64(c, obs, head):
    """float64 values of `obs` and log-probs of the stored actions, from the parameters the rollout ran with."""
    from oracle import nets

    ncfg = types.SimpleNamespace(layer_N=1, activation_id=c.cfg.activation_id, use_recurrent_policy=False, use_policy_active_masks=True)
    p = ref.unflatten(c.p0.double(), *c.dims, head)
    with torch.no_grad():
        v, _ = nets.critic_forward(p, ncfg, obs.double())
        x = c.buf["obs"].double()[:c.rows]
        if head == "gaussian":
            mean, std = nets.gaussian_params(p, nets.policy_features(p, ncfg, x)[0])
            lp = torch.distributions.Normal(mean, std).log_prob(c.buf["actions"].double())
        else:
            am = c.buf.get("action_masks")
            lp, _ = nets.policy_eval(p, ncfg, x, c.buf["actions"].double(), None if am is None else am[:c.rows].double())
    return v, lp


def test_c2_rollout_teacher_forced(c2):
    """share_rollout_kernel<CARTPOLE> at 4096 envs x 128 steps: observations, rewards and masks bit-exact against the
    numpy CartPole stepped with the kernel's own actions; log-probs of the stored actions and all T + 1 slots of
    value_preds (share_values_kernel) within ATOL of a float64 forward."""
    from oracle.envs import CartPoleVec

    b = c2.b
    obs, acts = b.policy_obs.cpu().numpy(), b.actions.cpu().numpy()
    rew, masks = b.rewards.cpu().numpy(), b.masks.cpu().numpy()
    env = CartPoleVec(4096)
    assert np.array_equal(obs[0], env.reset(seed=SEED))
    assert set(np.unique(acts)) <= {0.0, 1.0}
    done = 0
    for t in range(128):
        o, r, d, _ = env.step(acts[t].astype(np.int64))
        assert np.array_equal(obs[t + 1], o), t
        assert np.array_equal(rew[t], r.astype(np.float32)), t
        assert np.array_equal(masks[t + 1][..., 0], (~d).astype(np.float32)), t
        done += int(d.sum())
    assert done > 1000
    v, lp = _forward64(c2, c2.buf["obs"], "categorical")
    np.testing.assert_allclose(c2.buf["action_log_probs"].cpu().numpy(), lp.cpu().numpy(), rtol=0, atol=ATOL)
    np.testing.assert_allclose(c2.buf["value_preds"].cpu().numpy(), v.cpu().numpy(), rtol=0, atol=ATOL)
    assert c2.buf["value_preds"].shape[0] == c2.rows + 4096
    print(f"\n  c2 rollout: log-prob error {float((c2.buf['action_log_probs'].double() - lp).abs().max()):.1e}, "
          f"value error {float((c2.buf['value_preds'].double() - v).abs().max()):.1e}, {done} episode ends")


def test_c2_four_epochs_contiguous(c2, no_tf32):
    """C2's four updates (indices == NULL, 524 288 rows, 512 tape row blocks, the GAE moments as minibatch moments),
    each teacher-forced from the device's own state.  Epoch 1 has every ratio at 1 up to rounding; epochs 2-4 do not."""
    snap = h.snapshot(c2)
    rows = torch.arange(c2.rows, device="cuda")
    try:
        for epoch in range(4):
            state = _state(c2)
            k = _kernel_update(c2, None, c2.b.gae_stats[5:8], c2.rows)
            r64, r32 = _refs(c2, k, state, rows)
            _compare(f"c2-epoch{epoch + 1}-contiguous-524288rows-512blocks", c2.dims, "categorical", k, r64, r32, state, c2.cfg)
            spread = float(r64["ratio_spread"])
            assert (spread > 1e-4) if epoch else (spread < 1e-4), spread
            del r64, r32
    finally:
        h.restore(c2, snap)
    _peak("c2 four epochs")


def test_c2_shuffled_partial_last_block(c2, no_tf32):
    """A shuffled index list of 131 405 rows (128 full tape row blocks and a partial one of 333 rows),
    orl_minibatch_stats."""
    snap = h.snapshot(c2)
    g = torch.Generator(device="cuda").manual_seed(4)
    idx = torch.randperm(c2.rows, device="cuda", generator=g)[:c2.rows // 4 + 333].contiguous()
    assert idx.numel() % BLOCK == 333
    try:
        state = _state(c2)
        k = _kernel_update(c2, idx, h.mb_stats(idx, c2.b.returns, c2.b.active_masks), idx.numel())
        r64, r32 = _refs(c2, k, state, idx)
        _compare("c2-shuffled-131405rows(partial last block)", c2.dims, "categorical", k, r64, r32, state, c2.cfg)
    finally:
        h.restore(c2, snap)


C2_MUTANTS = [m for m, e in ref.MUTANTS.items() if e[3] == "categorical"]


@pytest.mark.parametrize("mutant", C2_MUTANTS)
def test_c2_mutants_are_detected(c2, no_tf32, mutant):
    """The real kernel output of C2's first update against a float64 reference with one deliberate mistake.  For
    adam-with-critic-lr the kernel runs with critic_lr in the device's second learning-rate slot, so a shared Adam that
    read that slot would fail its bar against the correct reference."""
    _, what, opts, _ = ref.MUTANTS[mutant]
    snap = h.snapshot(c2)
    saved = {k: getattr(c2.tr.cfg, k) for k in opts}
    rows = torch.arange(c2.rows, device="cuda")
    try:
        for key, val in opts.items():   # the kernel reads max_grad_norm from the config
            setattr(c2.tr.cfg, key, val)
        state = _state(c2)
        k = _kernel_update(c2, None, c2.b.gae_stats[5:8], c2.rows, critic_lr=opts.get("critic_lr"))
    finally:
        for key, val in saved.items():
            setattr(c2.tr.cfg, key, val)
        h.restore(c2, snap)
    r64, r32, bad = _refs(c2, k, state, rows, opts, mutant)
    if mutant == "critic-norm-unclipped":
        assert float(r64["norms"][0]) > opts["max_grad_norm"]
    _check_mutant(f"c2-{mutant}", mutant, k, r64, r32, bad, c2.dims, "categorical")


def test_c5_share_log_probs_and_values(c5s):
    """The Gaussian act's log-probs (ENV_NONE share_rollout_kernel<GAUSSIAN>) and all T + 1 slots of value_preds."""
    v, lp = _forward64(c5s, c5s.b.critic_obs.reshape(-1, 17), "gaussian")
    np.testing.assert_allclose(c5s.buf["action_log_probs"].cpu().numpy(), lp.cpu().numpy(), rtol=0, atol=ATOL)
    np.testing.assert_allclose(c5s.buf["value_preds"].cpu().numpy(), v.cpu().numpy(), rtol=0, atol=ATOL)
    assert c5s.buf["value_preds"].shape[0] == c5s.rows + 1024 and float(v.abs().max()) > 0


def test_c5_share_two_epochs_and_shuffled_quarter(c5s, no_tf32):
    """Two teacher-forced updates on the contiguous path (131 072 rows, 128 row blocks of the 1112-float Gaussian
    tape), then a shuffled quarter."""
    snap = h.snapshot(c5s)
    rows = torch.arange(c5s.rows, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(5)
    idx = torch.randperm(c5s.rows, device="cuda", generator=g)[:c5s.rows // 4].contiguous()
    try:
        for epoch in range(2):
            state = _state(c5s)
            k = _kernel_update(c5s, None, c5s.b.gae_stats[5:8], c5s.rows)
            r64, r32 = _refs(c5s, k, state, rows)
            _compare(f"c5share-epoch{epoch + 1}-contiguous-131072rows", c5s.dims, "gaussian", k, r64, r32, state, c5s.cfg)
        state = _state(c5s)
        k = _kernel_update(c5s, idx, h.mb_stats(idx, c5s.b.returns, c5s.b.active_masks), idx.numel())
        r64, r32 = _refs(c5s, k, state, idx)
        _compare("c5share-shuffled-32768rows", c5s.dims, "gaussian", k, r64, r32, state, c5s.cfg)
    finally:
        h.restore(c5s, snap)
    _peak("c5 share")


def test_c5_share_entropy_mutant_is_detected(c5s, no_tf32):
    from openrl_b200 import lib

    mutant = "entropy-weight-1/rows"
    _, what, opts, _ = ref.MUTANTS[mutant]
    snap, flags = h.snapshot(c5s), c5s.tr.flags
    rows = torch.arange(c5s.rows, device="cuda")
    try:
        c5s.tr.flags &= ~lib.PPO_POLICY_ACTIVE_MASKS
        state = _state(c5s)
        k = _kernel_update(c5s, None, c5s.b.gae_stats[5:8], c5s.rows)
    finally:
        c5s.tr.flags = flags
        h.restore(c5s, snap)
    r64, r32, bad = _refs(c5s, k, state, rows, opts, mutant)
    _check_mutant(f"c5share-{mutant}", mutant, k, r64, r32, bad, c5s.dims, "gaussian")


def _gridworld_table(n, k=64, seed=1):
    """Start cells near the goal (1, 1), so that random walks finish episodes inside the rollout."""
    rng = np.random.default_rng(seed)
    table = rng.integers(0, 4, size=(n, k, 2))
    goal = (table == 1).all(-1)
    table[goal] = (3, 3)
    return table


def test_gridworld_share_rollout_at_4096_envs():
    """share_rollout_kernel<GRIDWORLD> (n = 5): observations, rewards and masks bit-exact against the oracle env
    stepped with the kernel's own actions (env i's k-th reset at table[i, k]); log-probs within ATOL of float64."""
    from oracle.envs import GridWorldVec

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    N, T = 4096, 128
    table = _gridworld_table(N)
    flags = ["--seed", "2", "--episode_length", str(T), "--log_interval", "1000000", "--use_share_model", "true"]
    cfg, env, net, drv = _device_driver("GridWorldEnv", N, flags, reset_table=table)
    drv.actor_rollout()
    torch.cuda.synchronize()
    b = drv.buffer.data
    obs, acts = b.policy_obs.cpu().numpy(), b.actions.cpu().numpy()
    rew, masks = b.rewards.cpu().numpy(), b.masks.cpu().numpy()
    # the resets the device env has made before the rollout (PPONet's and the buffer's): every env's slot-0 cell
    k0 = [k for k in range(4) if (obs[0][:, 0, :2] == table[:, k]).all()]
    assert len(k0) >= 1
    k0 = k0[0]

    class PerEnvTable(GridWorldVec):
        def __init__(self, n):
            super().__init__(n)
            self.count = np.full(n, k0 + 1)
            self.pos = table[:, k0].copy()

        def _reset_one(self, i):
            self.steps[i] = 0
            self.pos[i] = table[i, self.count[i]]
            self.count[i] += 1

    ref_env = PerEnvTable(N)
    assert np.array_equal(obs[0], ref_env._obs().astype(np.float32))
    done = 0
    for t in range(T):
        o, r, d, _ = ref_env.step(acts[t].astype(np.int64))
        assert np.array_equal(obs[t + 1], o.astype(np.float32)), t
        assert np.array_equal(rew[t].reshape(-1), r.astype(np.float32).reshape(-1)), t
        assert np.array_equal(masks[t + 1].reshape(-1), (~d).astype(np.float32).reshape(-1)), t
        done += int(d.sum())
    assert done > 1000 and set(np.unique(acts)) == {0.0, 1.0, 2.0, 3.0, 4.0}
    c = _real(cfg, drv, "categorical")
    _, lp = _forward64(c, c.buf["obs"][:8], "categorical")
    np.testing.assert_allclose(c.buf["action_log_probs"].cpu().numpy(), lp.cpu().numpy(), rtol=0, atol=ATOL)


# ---------------------------------------------------------------- synthetic buffers -----------------------------------

def _synthetic(cfg, dims, head, total, rows_idx, seed, masked=False, inactive=0.1):
    """A buffer of `total` random rows and a net with random weights, Adam moments mid-run, a fraction `inactive` of
    active masks at zero and, with `masked`, a Categorical action mask with ~30 % of the actions illegal (never the
    taken one).  As in test_ppo_ffma_scale_cuda.py, the minibatch rows' old log-probs, value predictions and returns are
    drawn from the float64 forward so that no row lies within KINK of a branch point of the loss (ratio clip edges and
    dual-clip coefficient, value clip, Huber threshold, tie of the clipped and unclipped value losses), and no fc1
    pre-activation of obs_prep or common lies within ACT_KINK of the ReLU / LeakyReLU kink."""
    from oracle import nets

    d, n = dims
    gauss = head == "gaussian"
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, device="cuda")        # noqa: E731
    u = lambda *s: torch.rand(*s, generator=g, device="cuda")         # noqa: E731
    buf = dict(obs=r(total, d), advantages=r(total, 1), value_preds=r(total, 1), returns=3 * r(total, 1) + 2.0,
               active_masks=(u(total, 1) >= inactive).float(), action_log_probs=torch.zeros(total, n if gauss else 1, device="cuda"))
    if gauss:
        buf["actions"] = r(total, n)
    else:
        act = torch.randint(0, n, (total,), generator=g, device="cuda")
        buf["actions"] = act.float()[:, None]
        if masked:
            am = (u(total, n) >= 0.3).float()
            am[torch.arange(total, device="cuda"), act] = 1.0
            buf["action_masks"] = am
    state = dict(p=h.random_net(g, ref.param_shapes(d, n, head)), vn=torch.tensor([0.3, 0.5, 0.8], device="cuda"), step=3)
    state["m"] = 1e-3 * r(state["p"].numel())
    state["v"] = 1e-6 * u(state["p"].numel()) + 1e-8

    ncfg = types.SimpleNamespace(layer_N=1, activation_id=cfg.activation_id, use_recurrent_policy=False, use_policy_active_masks=True)
    p = ref.unflatten(state["p"].double(), d, n, head)
    h.redraw_off_act_kink(g, buf["obs"], rows_idx, lambda x: [
        x @ p["obs_prep.mlp.fc1.0.weight"].t() + p["obs_prep.mlp.fc1.0.bias"],
        nets.mlp_base(p, "obs_prep", x, 1, cfg.activation_id) @ p["common.fc1.0.weight"].t() + p["common.fc1.0.bias"]])
    x = lambda k: buf[k].double()[rows_idx]   # noqa: E731
    with torch.no_grad():
        if gauss:
            logp, _ = nets.policy_eval_gaussian(p, ncfg, x("obs"), x("actions"))
        else:
            logp, _ = nets.policy_eval(p, ncfg, x("obs"), x("actions"), x("action_masks") if masked else None)
        v, _ = nets.critic_forward(p, ncfg, x("obs"))
    many = rows_idx.numel() >= 1000   # enough rows to see both sides of every branch
    h.draw_kink_free(g, cfg, state["vn"], logp, v, buf["action_log_probs"], rows_idx, buf["value_preds"], buf["returns"],
                     rows_idx, both_clip_sides=many)
    return buf, state


def _run_synthetic(case, cfg, dims, head, batch_rows, contiguous_from=None, total=None, seed=0, masked=False, inactive=0.1,
                   mutant=None):
    """OrlPpoArgs built by hand for a synthetic buffer; orl_share_fwdbwd + orl_share_apply against both reference runs
    (and, with `mutant`, the check that the mistake fails its bar)."""
    lb, L = h.lib()
    d, n = dims
    gauss = head == "gaussian"
    hk = lb.HEAD_GAUSSIAN if gauss else lb.HEAD_CATEGORICAL
    total = total or batch_rows + 301
    idx, rows_idx = h.minibatch(total, batch_rows, contiguous_from, seed)
    buf, state = _synthetic(cfg, dims, head, total, rows_idx, seed, masked, inactive)
    count = int(L.orl_share_param_count_head(d, n, hk))
    assert state["p"].numel() == count
    ws = torch.empty(int(L.orl_share_workspace_floats_head(batch_rows, d, n, hk)), device="cuda")
    folded = torch.zeros(8, device="cuda")
    grads = torch.zeros((count + 3) & ~3, device="cuda")
    dev = {k: state[k].clone() for k in ("p", "m", "v", "vn")}
    steps = torch.tensor([state["step"], 0], dtype=torch.int32, device="cuda")
    lrs = torch.tensor([cfg.lr, cfg.critic_lr], dtype=torch.float32, device="cuda")
    stats = h.gae_stats(buf), h.mb_stats(rows_idx.contiguous(), buf["returns"], buf["active_masks"])
    train_info = torch.zeros(6, device="cuda")
    one_net = dict(pol=dev["p"], cri=dev["p"], pol_m=dev["m"], cri_m=dev["m"], pol_v=dev["v"], cri_v=dev["v"], vn=dev["vn"])
    a = h.ppo_args(cfg, (d, n, d), hk, h.ppo_flags(cfg), 1, dict(buf, policy_obs=buf["obs"], critic_obs=buf["obs"]), batch_rows,
                   total, idx, contiguous_from or 0, stats, one_net, steps, lrs, train_info, ws, folded, grads)
    s = lb.current_stream()
    lb.check(L.orl_share_fwdbwd(a, s), "orl_share_fwdbwd")
    lb.check(L.orl_share_apply(a, s), "orl_share_apply")
    torch.cuda.synchronize()
    del ws
    k = dict(grad=grads[:count], losses=folded[:4], info=train_info, norms=train_info[[4, 1]], step=int(steps[0]), **dev)
    r64, r32 = (ref.update(cfg, buf, state, rows_idx, dims, head, dt, vn_beta=cfg.vn_beta) for dt in (torch.float64, torch.float32))
    if cfg.use_max_grad_norm and cfg.max_grad_norm < 1:   # the clip case: both clips act, the second one measures the clipped norm
        assert float(r64["norms"][0]) > cfg.max_grad_norm and abs(float(r64["norms"][1]) - cfg.max_grad_norm) < 1e-5
    print(f"\n  {case}: {batch_rows} rows, {-(-batch_rows // BLOCK)} tape row blocks")
    _compare(case, dims, head, k, r64, r32, state, cfg, check_vn=cfg.use_valuenorm)
    if mutant is not None:
        bad = ref.update(cfg, buf, state, rows_idx, dims, head, torch.float64, vn_beta=cfg.vn_beta, mutant=mutant)
        _check_mutant(f"{case}-{mutant}", mutant, k, r64, r32, bad, dims, head)
    torch.cuda.empty_cache()


def _edges():
    """(id, dims (d, n), head, rows, options): every edge is in the id."""
    out = []
    for rows, tag in ((1, "1row"), (127, "127rows"), (1023, "1023rows(block-1)"), (1024, "1024rows(1 block)"),
                      (1025, "1025rows(block+1)"), (3 * BLOCK + 1, "3073rows(3blocks+1)"), (64 * BLOCK - 1, "65535rows(64blocks-1)")):
        out.append((f"{tag}-gauss-d17-n6", (17, 6), "gaussian", rows, {}))
        out.append((f"{tag}-cat-d4-n2", (4, 2), "categorical", rows, {}))
    for d in (1, 4, 17, 63, 64):
        out.append((f"d{d}(fc1 gemm N=d)-gauss-n6-2085rows", (d, 6), "gaussian", 2085, {}))
        out.append((f"d{d}(fc1 gemm N=d)-cat-n4-2085rows", (d, 4), "categorical", 2085, {}))
    for n in (1, 2, 5, 8):
        out.append((f"n{n}(head gemm M=n, logstd job)-gauss-d17-2085rows", (17, n), "gaussian", 2085, {}))
        out.append((f"n{n}(head gemm M=n)-cat-d6-2085rows", (6, n), "categorical", 2085, {}))
    out.append(("5rows(1 partial block)-cat-d6-n4", (6, 4), "categorical", 5, {}))
    out.append(("2085rows(2blocks+37)-cat-d6-n4", (6, 4), "categorical", 2 * BLOCK + 37, {}))
    for head, dims in (("gauss", (17, 6)), ("cat", (6, 5))):
        full = "gaussian" if head == "gauss" else "categorical"
        out.append((f"contiguous-from-row1000-{head}-3149rows", dims, full, 3 * BLOCK + 77, dict(contiguous_from=1000, total=6000)))
        out.append((f"active-masks-30%zero-{head}-3073rows", dims, full, 3 * BLOCK + 1, dict(inactive=0.3)))
        out.append((f"active-masks-all-one-{head}-3073rows", dims, full, 3 * BLOCK + 1, dict(inactive=0.0)))
    out.append(("cat-action-masks-30%illegal-d6-n5-3073rows", (6, 5), "categorical", 3 * BLOCK + 1, dict(masked=True)))
    out.append(("cat-action-masks-30%illegal-d17-n8-1025rows", (17, 8), "categorical", BLOCK + 1, dict(masked=True)))
    for act, name in enumerate(("tanh", "relu", "leaky-relu", "elu")):
        out.append((f"act{act}-{name}-gauss-d17-n6-2085rows", (17, 6), "gaussian", 2085, dict(activation_id=act)))
        out.append((f"act{act}-{name}-cat-d6-n5-masked-2085rows", (6, 5), "categorical", 2085, dict(activation_id=act, masked=True)))
    return out


EDGES = _edges()


@pytest.mark.parametrize("case,dims,head,rows,opts", EDGES, ids=[e[0] for e in EDGES])
def test_update_synthetic_edges(no_tf32, case, dims, head, rows, opts):
    opts = dict(opts)
    cfg = types.SimpleNamespace(**{**BASE, "activation_id": opts.pop("activation_id", BASE["activation_id"])})
    _run_synthetic(case, cfg, dims, head, rows, seed=len(case) * 7 + dims[0], **opts)


def test_masked_categorical_mutant_is_detected(no_tf32):
    """action-mask-ignored-in-update against the kernel on a masked Categorical buffer (3 row blocks + 1 row)."""
    cfg = types.SimpleNamespace(**BASE)
    _run_synthetic("masked-cat-d6-n5-3073rows", cfg, (6, 5), "categorical", 3 * BLOCK + 1, seed=21, masked=True,
                   mutant="action-mask-ignored-in-update")


FLAG_CASES = [(flags, head) for flags in CASES for head in ("gaussian", "categorical")]


@pytest.mark.parametrize("flags,head", FLAG_CASES, ids=[f"{' '.join(f) or 'default'}-{h}" for f, h in FLAG_CASES])
def test_update_flag_sweep(no_tf32, flags, head):
    """Every option of tests/test_ppo_flags_cuda.py on the shared model, 3 row blocks + 37 rows: active masks off,
    Huber off, value clip off, ValueNorm off, advantage normalisation, no gradient clip, weight decay with lr != critic_lr
    (the shared Adam steps with lr), the activations, other coefficients, a gradient clip that acts (both logged norms),
    dual clip and A2C; the GAE-only options run the default update."""
    cfg = h.flag_cfg(flags)
    dims = (17, 6) if head == "gaussian" else (6, 5)
    _run_synthetic(f"flags-{'-'.join(flags) or 'default'}-{head}", cfg, dims, head, 3 * BLOCK + 37, seed=77,
                   masked=head == "categorical")
