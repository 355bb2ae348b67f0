"""Legal-move masks reported by host-stepped envs (`info["action_masks"]`): ingest into the device buffer (slot 0 from the
reset infos, slot t+1 by orl_host_insert / orl_host_insert_rnn when every stepped env reported them), applied by the
feed-forward act (orl_rollout), the GRU act (orl_rnn_act_rows) and both updates, and by PPOAgent.act for GRU policies.

Bars: the reference's traces on the masked env (tests/golden/trace_masked_*.npz) through PPOAgent over HostVecEnv in
parity mode — actions, observations, masks and action masks bit-exact, the six logged scalars at rtol 2e-4, parameters
at rtol 2e-3, GRU hidden states at 2e-5; at 1024 envs x 128 steps with Philox sampling no illegal action and
bit-identical buffers from the synchronous and the two-group loop; the edges of the reference's masking."""
import copy
import os

import numpy as np
import pytest

from conftest import GOLDEN
from masked_oracle import MaskedTargetVec
from test_rnn_host_cuda import KEYS, _agent
from test_rnn_scale_cuda import no_tf32  # noqa: F401  (pytest fixture)

pytestmark = pytest.mark.gpu


class _Host:
    """The reference's host vec-env duck type over MaskedTargetVec; `step_range` steps envs [lo, hi) only."""

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
        if hi == self.inner.N:       # one step call of the vec-env per step of all groups (`report` is keyed by it)
            self.inner.calls += 1
        return out


def _host(n, report=None, cls=MaskedTargetVec):
    from openrl_b200.envs.vec_env import HostVecEnv

    return HostVecEnv(_Host(cls(n, report)))


def _illegal(actions, action_masks):
    a = actions[..., 0].astype(np.int64)
    return int((np.take_along_axis(action_masks[:-1], a[..., None], axis=-1) == 0).sum())


@pytest.mark.parametrize("tag", ["masked_ff", "masked_gru"])
def test_host_masks_reproduce_reference_trace(cuda, tag):
    d = np.load(os.path.join(GOLDEN, f"trace_{tag}.npz"), allow_pickle=True)
    iters, N = int(d["meta/iters"]), int(d["meta/env_num"])
    flags = str(d["meta/flags"]).split() + ["--parity_mode", "true", "--log_interval", "1"]
    env = _host(N)
    cfg, net, agent = _agent(env, flags, golden=d)
    drv = agent.driver
    b = drv.buffer.data
    assert not b.action_masks_trivial      # the reset infos carried masks
    for it in range(iters):
        tag_it = f"it{it}"
        drv.episode = it
        drv.actor_rollout()
        assert np.array_equal(b.actions.cpu().numpy(), d[f"{tag_it}/actions"]), tag_it
        assert np.array_equal(b.policy_obs.cpu().numpy(), d[f"{tag_it}/policy_obs"]), tag_it
        assert np.array_equal(b.masks.cpu().numpy(), d[f"{tag_it}/masks"]), tag_it
        assert np.array_equal(b.action_masks.cpu().numpy(), d[f"{tag_it}/action_masks"]), tag_it
        np.testing.assert_allclose(b.action_log_probs.cpu().numpy(), d[f"{tag_it}/action_log_probs"], rtol=0, atol=2e-5)
        if drv.recurrent:
            np.testing.assert_allclose(b.rnn_states.cpu().numpy(), d[f"{tag_it}/rnn_states"], rtol=0, atol=2e-5)
        drv.compute_returns()
        if drv.recurrent:
            np.testing.assert_allclose(b.rnn_states_critic.cpu().numpy(), d[f"{tag_it}/rnn_states_critic"], rtol=0, atol=2e-5)
        np.testing.assert_allclose(b.value_preds.cpu().numpy()[:-1], d[f"{tag_it}/value_preds"][:-1], rtol=0, atol=2e-5)
        np.testing.assert_allclose(b.returns.cpu().numpy()[:-1], d[f"{tag_it}/returns"][:-1], rtol=1e-4, atol=2e-4)
        info = drv.trainer.train(b)
        want = d[f"{tag_it}/updates"].mean(axis=0)
        for col, name in enumerate(KEYS):
            np.testing.assert_allclose(info[name], want[col], rtol=2e-4, atol=1e-5, err_msg=f"{tag_it} {name}")
        for mk in ("policy", "critic"):
            for k, v in net.module.models[mk].state_dict().items():
                gk = f"{tag_it}/params/{mk}.{k}"
                if gk in d and "value_normalizer" not in k:
                    np.testing.assert_allclose(v.cpu().numpy(), d[gk], rtol=2e-3, atol=2e-5, err_msg=gk)
        b.after_update()


@pytest.mark.parametrize("recurrent", [False, True])
def test_host_masks_at_scale_no_illegal_action_and_loops_agree(cuda, recurrent):
    """1024 envs, T = 128, Philox sampling: no illegal action in either host loop, and the synchronous and the two-group
    loop write the same bits (action masks included) over two iterations with an update between them."""
    import torch

    N, T = 1024, 128
    flags = ["--seed", "3", "--episode_length", str(T), "--ppo_epoch", "1", "--num_mini_batch", "2", "--log_interval", "1"]
    if recurrent:
        flags += ["--use_recurrent_policy", "true", "--data_chunk_length", "8"]
    runs, init = [], None
    for grouped in (False, True):
        env = _host(N)
        assert env.supports_groups
        cfg, net, agent = _agent(env, flags + ["--host_env_groups", "true" if grouped else "false"], like=init)
        if init is None:
            init = {mk: {k: v.clone() for k, v in net.module.models[mk].state_dict().items()} for mk in ("policy", "critic")}
        drv, b = agent.driver, agent.driver.buffer.data
        env.env.inner.reset(seed=11)         # the same episodes in both runs
        drv.reset_and_buffer_init()
        bufs = []
        for it in range(2):
            drv.episode = it
            drv.actor_rollout()
            torch.cuda.synchronize()
            bufs.append({k: getattr(b, k).cpu().numpy().copy()
                         for k in ("actions", "action_log_probs", "policy_obs", "masks", "rewards", "action_masks")
                         + (("rnn_states",) if recurrent else ())})
            assert _illegal(bufs[-1]["actions"], bufs[-1]["action_masks"]) == 0
            assert (bufs[-1]["action_masks"] == 0).mean() > 0.2
            drv.compute_returns()
            torch.manual_seed(7)
            drv.trainer.train(b)
            b.after_update()
        runs.append(bufs)
    for it in range(2):
        for k in runs[0][it]:
            assert np.array_equal(runs[0][it][k], runs[1][it][k]), (it, k)


def test_slots_without_masks_keep_their_content(cuda):
    """An env that reports masks on some steps only: unwritten slots keep what they held, as in the reference
    (ones from the allocation, then the previous rollout's value), in both host loops; the update still runs."""
    import torch

    T, N = 8, 6
    report = lambda i, t: t % 3 != 1    # noqa: E731  (every env lacks the key on steps 1, 4, 7, ...)
    flags = ["--seed", "1", "--episode_length", str(T), "--ppo_epoch", "1", "--log_interval", "1"]
    for grouped in ("false", "true"):
        env = _host(N, report)
        cfg, net, agent = _agent(env, flags + ["--host_env_groups", grouped])
        drv, b = agent.driver, agent.driver.buffer.data
        prev = b.action_masks.cpu().numpy().copy()
        for it in range(2):
            drv.episode = it
            drv.actor_rollout()
            torch.cuda.synchronize()
            am = b.action_masks.cpu().numpy()
            calls0 = it * T
            for t in range(T):
                if not report(0, calls0 + t):
                    assert np.array_equal(am[t + 1], prev[t + 1]), (grouped, it, t)
            assert _illegal(b.actions.cpu().numpy(), am) == 0
            prev = am.copy()
            drv.compute_returns()
            drv.trainer.train(b)
            b.after_update()
            assert np.array_equal(b.action_masks[0].cpu().numpy(), am[-1])


class _OneLegal(MaskedTargetVec):
    """Only the target is legal (p_legal = 0), or with `none` every action is masked."""
    none = False

    def __init__(self, n, report=None):
        super().__init__(n, report)
        for e in self.envs:
            e._draw = self._draw_fn(e)

    def _draw_fn(self, e):
        none = self.none

        def draw():
            e.target = int(e.rng.integers(e.n_actions))
            e.mask = np.zeros(e.n_actions, np.int8)
            if not none:
                e.mask[e.target] = 1
        return draw


@pytest.mark.parametrize("recurrent", [False, True])
def test_single_legal_action_and_all_masked_rows(cuda, recurrent):
    """A row with one legal action: that action, log-prob 0, entropy 0, and no policy gradient (the policy parameters do
    not move).  An all-zero row: every logit is -6e4, so the distribution is uniform over all actions, as in the
    reference."""
    import torch

    T, N = 16, 64
    flags = ["--seed", "4", "--episode_length", str(T), "--ppo_epoch", "1", "--log_interval", "1"]
    if recurrent:
        flags += ["--use_recurrent_policy", "true", "--data_chunk_length", "4"]
    env = _host(N, cls=_OneLegal)
    cfg, net, agent = _agent(env, flags)
    drv, b = agent.driver, agent.driver.buffer.data
    drv.actor_rollout()
    acts, obs = b.actions.cpu().numpy()[..., 0], b.policy_obs.cpu().numpy()
    assert np.array_equal(acts, obs[:-1].argmax(-1))
    assert (b.action_log_probs.cpu().numpy() == 0).all()
    before = {k: v.clone() for k, v in net.module.models["policy"].state_dict().items()}
    drv.compute_returns()
    info = drv.trainer.train(b)
    assert info["dist_entropy"] == 0 and info["actor_grad_norm"] == 0, info
    for k, v in net.module.models["policy"].state_dict().items():
        assert torch.equal(v, before[k]), k

    class _NoneLegal(_OneLegal):
        none = True

    env = _host(N, cls=_NoneLegal)
    cfg, net, agent = _agent(env, flags)
    drv, b = agent.driver, agent.driver.buffer.data
    drv.actor_rollout()
    assert not b.action_masks_trivial and (b.action_masks.cpu().numpy() == 0).all()
    # log-softmax at logits of -6e4 (float32 ulp 0.004 there) rounds -ln 5 to -1.609375; the distribution is uniform
    np.testing.assert_allclose(b.action_log_probs.cpu().numpy(), -np.log(5), rtol=0, atol=1e-4)
    counts = np.bincount(b.actions.cpu().numpy().astype(np.int64).ravel(), minlength=5)
    assert (counts > 0.15 * counts.sum()).all(), counts
    drv.compute_returns()
    info = drv.trainer.train(b)
    np.testing.assert_allclose(info["dist_entropy"], np.log(5), rtol=0, atol=1e-4)


def test_recurrent_agent_act_applies_masks(cuda):
    """PPOAgent.act(obs, info) with a GRU policy: the deterministic act picks the best legal action, and the module's
    log-probs of masked rows match the oracle's GRU act (oracle/nets.policy_act) on the same weights."""
    import torch

    from oracle import loop, nets

    N = 32
    flags = ["--seed", "2", "--episode_length", "8", "--use_recurrent_policy", "true", "--data_chunk_length", "4"]
    env = _host(N)
    cfg, net, agent = _agent(env, flags)
    rng = np.random.default_rng(0)
    obs = rng.standard_normal((N, 1, 5)).astype(np.float32)
    m = (rng.random((N, 5)) < 0.5).astype(np.int8)
    m[np.arange(N), rng.integers(0, 5, N)] = 1
    infos = [{"action_masks": m[i]} for i in range(N)]
    agent.net.reset()
    free, _ = agent.act(obs, deterministic=True)
    agent.net.reset()
    masked, _ = agent.act(obs, info=infos, deterministic=True)
    masked = masked[:, 0, 0]
    assert (m[np.arange(N), masked] == 1).all()
    assert (masked[m[np.arange(N), free[:, 0, 0]] == 1] == free[:, 0, 0][m[np.arange(N), free[:, 0, 0]] == 1]).all()
    assert (m[np.arange(N), free[:, 0, 0]] == 0).any()     # some rows had to move to another action
    # log-probs against the oracle's act with the device weights
    ocfg = loop.cfg_from_flags(" ".join(flags))
    pol = {k: v.detach().cpu().clone() for k, v in net.module.models["policy"].state_dict().items()}
    o = torch.from_numpy(obs.reshape(N, 5))
    h0 = torch.zeros(N, 1, 64)
    mk = torch.ones(N, 1)
    want_a, want_lp, _ = nets.policy_act(pol, ocfg, o, torch.from_numpy(m.astype(np.float32)), h0, mk, deterministic=True)
    acts, logp, _ = net.module.act(obs.reshape(N, 5), rnn_states_actor=h0, masks=mk, action_masks=m, deterministic=True)
    assert np.array_equal(acts.cpu().numpy().ravel(), want_a.numpy().ravel())
    np.testing.assert_allclose(logp.cpu().numpy().ravel(), want_lp.numpy().ravel(), rtol=0, atol=2e-5)


class _MaskedMultiAgent:
    """A = 3 agents per env, obs (N, A, 6) ~ N(0, 1), Discrete(5), per-agent masks `info["action_masks"]` of shape
    (A, n): random legal subsets (one in eight rows with a single legal action).  An env finishes with probability 0.15
    per step.  `history` keeps every reported (N, A, n) mask block: reset first, then one per step."""
    OBS, N_ACT, A = 6, 5, 3

    def __init__(self, n, seed=0):
        from openrl_b200 import spaces

        self.parallel_env_num, self.agent_num = n, self.A
        self.observation_space = spaces.Box(-np.inf, np.inf, (self.OBS,), np.float32)
        self.action_space = spaces.Discrete(self.N_ACT)
        self.rng = np.random.default_rng(seed)
        self.history = []

    def _masks(self, n):
        m = (self.rng.random((n, self.A, self.N_ACT)) < 0.6).astype(np.int8)
        keep = self.rng.integers(0, self.N_ACT, (n, self.A))
        single = self.rng.random((n, self.A)) < 0.125
        m[single] = 0
        np.put_along_axis(m, keep[..., None], 1, axis=-1)
        self.history.append(m)
        return [{"action_masks": m[i]} for i in range(n)]

    def _obs(self, n):
        return self.rng.standard_normal((n, self.A, self.OBS)).astype(np.float32)

    def reset(self, seed=None):
        n = self.parallel_env_num
        self.history = []
        return self._obs(n), self._masks(n)

    def step(self, actions):
        n = self.parallel_env_num
        assert actions.shape == (n, self.A, 1)
        m = self.history[-1]
        assert (np.take_along_axis(m, actions.astype(np.int64), axis=-1) == 1).all(), "an illegal action reached the env"
        dones = np.repeat((self.rng.random(n) < 0.15)[:, None], self.A, axis=1)
        return self._obs(n), self.rng.standard_normal((n, self.A, 1)), dones, self._masks(n)


def test_multi_agent_masked_gru_update_matches_float64(cuda, no_tf32):
    """64 envs x 3 agents with per-agent (A, n) masks, T = 16, chunks of 4: the host loop stages the agent rows of every
    env in (env, agent) order, the insert writes them to slot t+1 and the GRU act samples only legal actions with the
    masked log-probs of a float64 teacher-forced forward; then one update over the whole buffer (768 chunks, 3072
    row-steps: three tape row blocks) against rnn_ref64 driven with the masks, at the bars of test_rnn_scale_cuda.py."""
    import types

    import torch

    import rnn_ref64
    import rnn_ref64_masked
    from oracle import nets
    from openrl_b200.envs.vec_env import HostVecEnv
    from test_rnn_scale_cuda import _c3_buf, _compare, _drive

    N, A, T, L = 64, 3, 16, 4
    host = _MaskedMultiAgent(N)
    flags = ["--seed", "6", "--use_recurrent_policy", "true", "--episode_length", str(T), "--data_chunk_length", str(L),
             "--ppo_epoch", "1", "--num_mini_batch", "1", "--use_valuenorm", "true", "--host_env_groups", "false"]
    cfg, net, agent = _agent(HostVecEnv(host), flags)
    drv, tr, b = agent.driver, agent.driver.trainer, agent.driver.buffer.data
    drv.actor_rollout()
    drv.compute_returns()
    torch.cuda.synchronize()
    B = N * A
    am = b.action_masks.cpu().numpy()
    assert np.array_equal(am, np.stack(host.history).reshape(T + 1, N, A, 5).astype(np.float32))
    assert _illegal(b.actions.cpu().numpy(), am) == 0 and (am.sum(-1) == 1).any()

    # the act: masked log-probs of the recorded actions, teacher-forced from the device's own hidden states
    pol, cri = net.module.models["policy"], net.module.models["critic"]
    p = {k: v.detach().double() for k, v in rnn_ref64.unflatten(pol.flat_params.double(), tr.d, tr.n, False).items()}
    ncfg = rnn_ref64.net_cfg(cfg.activation_id, True)
    h, mk = rnn_ref64.rows(b.rnn_states).double(), rnn_ref64.rows(b.masks).double()
    with torch.no_grad():
        feat, _ = nets.policy_features(p, ncfg, rnn_ref64.rows(b.policy_obs).double()[:T * B], h[:T * B].unsqueeze(1), mk[:T * B])
        lp = nets.categorical_logits(p, feat, rnn_ref64.rows(b.action_masks).double()[:T * B]).gather(-1, rnn_ref64.rows(b.actions).long())
    np.testing.assert_allclose(rnn_ref64.rows(b.action_log_probs).cpu().numpy(), lp.cpu().numpy(), rtol=0, atol=2e-5)

    # the update: one minibatch of every chunk, kernel against float64 / float32 references with the masks
    m = tr.algo_module
    op, oc = m.optimizers["policy"], m.optimizers["critic"]
    vn = cri.value_normalizer
    live = dict(pol=pol.flat_params, cri=cri.flat_params, pol_m=op.exp_avg, pol_v=op.exp_avg_sq, cri_m=oc.exp_avg,
                cri_v=oc.exp_avg_sq, vn=vn.state)
    state = dict({k: v.clone() for k, v in live.items()}, steps=[int(x) for x in m.adam_steps])
    total = T * B // L
    ids = torch.randperm(total, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3)).contiguous()
    tr.tape = torch.empty(int(tr._lib.orl_rnn_workspace_floats(total * L, tr.rnn_stride)), dtype=torch.float32, device="cuda")
    tr.sync_lrs()
    a = tr._rnn_args(b, ids, b.gae_stats[5:8])
    assert a.action_masks == b.action_masks.data_ptr()
    grads, la, after = _drive(a, tr.rnn_grads, tr.loss_acc, live)
    tr.tape = None
    np_, nc = int(pol.flat_params.numel()), int(cri.flat_params.numel())
    k = dict(grad_pol=grads[0, :np_], grad_cri=grads[1, :nc], losses=la, steps=[int(x) for x in m.adam_steps], **after)
    rcfg = types.SimpleNamespace(**vars(cfg), vn_beta=vn.beta)
    dims = (tr.d, tr.n, tr.dc)
    buf = _c3_buf(b)
    r64, r32 = (rnn_ref64_masked.update(rcfg, buf, state, ids, L, dims, b.action_masks, dtype=dt)
                for dt in (torch.float64, torch.float32))
    _compare("masked-A3-L4-768chunks-3072rows", dims, k, r64, r32, check_vn=True)
    # the masks matter: without them the float64 policy gradient is another one
    plain = rnn_ref64.update(rcfg, buf, state, ids, L, dims, joint=False, dtype=torch.float64)
    assert float((plain["grad_pol"] - r64["grad_pol"]).norm()) > 1e-3 * float(r64["grad_pol"].norm())
