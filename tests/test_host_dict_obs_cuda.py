"""Host-stepped envs with a Dict {"policy", "critic"} observation space: the critic observation is staged after the policy
observation in the step's one H2D block, written to critic_obs[t+1] by orl_host_insert / orl_host_insert_rnn, and read
by the critic pass and the critic half of the update; the policy keeps reading policy_obs.

Bars: the reference's traces on the Dict toy env (tests/golden/trace_dict_obs_*.npz) through make(...,
make_custom_envs=...) in parity mode — actions and both observations bit-exact, the logged scalars at rtol 1e-4,
parameters at rtol 2e-3; the synchronous and two-group loops bit-identical; critic rows bit-exact against what the host
env returned; a 40-wide critic (FFMA critic and update) against float64 references."""
import types

import numpy as np
import pytest

from helpers import KEYS, make_agent
from scale_harness import no_tf32  # noqa: F401  (pytest fixture)

pytestmark = pytest.mark.gpu


def _make(n):
    from dict_obs_oracle import SpacedDictTargetEnv
    from openrl_b200.envs.common import make

    return make("DictTarget", env_num=n,
                make_custom_envs=lambda id, env_num, render_mode=None, **kw: [SpacedDictTargetEnv for _ in range(env_num)])


class _DictHost:
    """A agents per env, Dict {"policy": Box(d), "critic": Box(dc)} observations ~ N(0, 1), Discrete(n) with per-agent
    (A, n) masks, an env finishing with probability 0.15 per step.  Every draw is keyed by (env, the env's step count),
    so a sub-range step (`step_range`) returns what the whole-range step would; `log[(e, t)]` keeps env e's
    observations and masks after its t-th step (t = 0: reset)."""

    def __init__(self, n, A=3, d=6, dc=40, n_act=5, masks=True):
        from openrl_b200 import spaces

        box = lambda w: spaces.Box(-np.inf, np.inf, (w,), np.float32)  # noqa: E731
        self.parallel_env_num, self.agent_num, self.d, self.dc, self.n_act = n, A, d, dc, n_act
        self.observation_space = spaces.Dict({"policy": box(d), "critic": box(dc)})
        self.action_space = spaces.Discrete(n_act)
        self.masks, self.t, self.log = masks, np.zeros(n, np.int64), {}

    def _draw(self, e):
        g = np.random.default_rng((7, e, int(self.t[e])))
        A = self.agent_num
        pol = g.standard_normal((A, self.d)).astype(np.float32)
        cri = g.standard_normal((A, self.dc)).astype(np.float32)
        m = (g.random((A, self.n_act)) < 0.6).astype(np.int8)
        m[np.arange(A), g.integers(0, self.n_act, A)] = 1
        self.log[e, int(self.t[e])] = (pol, cri, m)
        return pol, cri, m, g.random() < 0.15, g.standard_normal((A, 1))

    def _out(self, lo, hi):
        draws = [self._draw(e) for e in range(lo, hi)]
        obs = {"policy": np.stack([x[0] for x in draws]), "critic": np.stack([x[1] for x in draws])}
        infos = [{"action_masks": x[2]} if self.masks else {} for x in draws]
        dones = np.repeat(np.array([x[3] for x in draws])[:, None], self.agent_num, axis=1)
        return obs, np.stack([x[4] for x in draws]), dones, infos

    def reset(self, seed=None):
        self.t[:] = 0
        obs, _, _, infos = self._out(0, self.parallel_env_num)
        return obs, infos

    def step(self, actions):
        return self.step_range(0, self.parallel_env_num, actions)

    def step_range(self, lo, hi, actions):
        acts = np.asarray(actions).reshape(hi - lo, self.agent_num)
        for i, e in enumerate(range(lo, hi)):
            if self.masks:      # the env checks its actions against the masks it reported
                assert (self.log[e, int(self.t[e])][2][np.arange(self.agent_num), acts[i]] == 1).all(), "illegal action"
        self.t[lo:hi] += 1
        return self._out(lo, hi)

    def slots(self, t0, T):
        """Slots t0 .. t0 + T of the buffer as the env returned them: policy (T+1, N, A, d), critic, masks."""
        N = self.parallel_env_num
        out = [np.stack([np.stack([self.log[e, t][k] for e in range(N)]) for t in range(t0, t0 + T + 1)]) for k in range(3)]
        return out[0], out[1], out[2].astype(np.float32)


@pytest.mark.parametrize("tag", ["dict_obs_ff", "dict_obs_gru"])
def test_dict_obs_host_env_reproduces_reference_trace(cuda, tag):
    import os

    from conftest import GOLDEN

    d = np.load(os.path.join(GOLDEN, f"trace_{tag}.npz"), allow_pickle=True)
    iters, N = int(d["meta/iters"]), int(d["meta/env_num"])
    flags = str(d["meta/flags"]).split() + ["--parity_mode", "true", "--log_interval", "1"]
    env = _make(N)
    assert env.dict_obs and (env.obs_dim, env.critic_obs_dim) == (3, 7)
    cfg, net, agent = make_agent(env, flags, golden=d)
    drv, tr = agent.driver, agent.driver.trainer
    b = drv.buffer.data
    assert b.critic_obs is not b.policy_obs and b.critic_obs.shape[-1] == 7
    assert tr.use_tensor_cores == (not drv.recurrent)      # max(d, dc) = 7 <= 8: the tensor-core update for the MLP
    for it in range(iters):
        tag_it = f"it{it}"
        drv.episode = it
        drv.actor_rollout()
        assert np.array_equal(b.actions.cpu().numpy(), d[f"{tag_it}/actions"]), tag_it
        assert np.array_equal(b.policy_obs.cpu().numpy(), d[f"{tag_it}/policy_obs"]), tag_it
        assert np.array_equal(b.critic_obs.cpu().numpy(), d[f"{tag_it}/critic_obs"]), tag_it
        assert np.array_equal(b.masks.cpu().numpy(), d[f"{tag_it}/masks"]), tag_it
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
            np.testing.assert_allclose(info[name], want[col], rtol=1e-4, atol=1e-5, err_msg=f"{tag_it} {name}")
        for mk in ("policy", "critic"):
            for k, v in net.module.models[mk].state_dict().items():
                gk = f"{tag_it}/params/{mk}.{k}"
                if gk in d and "value_normalizer" not in k:
                    np.testing.assert_allclose(v.cpu().numpy(), d[gk], rtol=2e-3, atol=2e-5, err_msg=gk)
        b.after_update()
        assert np.array_equal(b.critic_obs[0].cpu().numpy(), d[f"{tag_it}/critic_obs"][-1])   # the slot shift


@pytest.mark.parametrize("recurrent", [False, True])
def test_dict_obs_loops_agree_and_critic_rows_are_the_envs(cuda, recurrent):
    """64 envs x 3 agents, (A, 6) policy and (A, 40) critic rows, (A, 5) masks, T = 16, Philox sampling, two iterations
    with an update between them: the synchronous and the two-group loop write the same bits (buffers and parameters),
    and critic_obs slots 0..T — slot 0 after the slot shift, rows of envs that finished included — are what the host env
    returned, bit for bit, as are policy_obs and action_masks."""
    import torch

    from openrl_b200.envs.vec_env import HostVecEnv

    N, A, T = 64, 3, 16
    flags = ["--seed", "3", "--episode_length", str(T), "--ppo_epoch", "1", "--num_mini_batch", "2", "--log_interval", "1"]
    if recurrent:
        flags += ["--use_recurrent_policy", "true", "--data_chunk_length", "4"]
    runs, init = [], None
    for grouped in (False, True):
        host = _DictHost(N, A)
        env = HostVecEnv(host)
        assert env.supports_groups
        cfg, net, agent = make_agent(env, flags + ["--host_env_groups", "true" if grouped else "false"], like=init)
        if init is None:
            init = {mk: {k: v.clone() for k, v in net.module.models[mk].state_dict().items()} for mk in ("policy", "critic")}
        drv, b = agent.driver, agent.driver.buffer.data
        assert not drv.trainer.use_tensor_cores
        keys = ("actions", "action_log_probs", "policy_obs", "critic_obs", "masks", "rewards", "action_masks", "value_preds")
        bufs = []
        for it in range(2):
            drv.episode = it
            drv.actor_rollout()
            drv.compute_returns()
            torch.cuda.synchronize()
            bufs.append({k: getattr(b, k).cpu().numpy().copy() for k in keys + (("rnn_states",) if recurrent else ())})
            pol, cri, am = host.slots(it * T, T)
            assert np.array_equal(bufs[-1]["critic_obs"], cri), it
            assert np.array_equal(bufs[-1]["policy_obs"], pol), it
            assert np.array_equal(bufs[-1]["action_masks"], am), it
            assert (bufs[-1]["masks"][1:] == 0).any()
            torch.manual_seed(7)
            drv.trainer.train(b)
            b.after_update()
        params = {mk: {k: v.cpu().numpy().copy() for k, v in net.module.models[mk].state_dict().items()}
                  for mk in ("policy", "critic")}
        runs.append((bufs, params))
    (b0, p0), (b1, p1) = runs
    for it in range(2):
        for k in b0[it]:
            assert np.array_equal(b0[it][k], b1[it][k]), (it, k)
    for mk in p0:
        for k in p0[mk]:
            assert np.array_equal(p0[mk][k], p1[mk][k]), (mk, k)


def test_wide_critic_feed_forward_update_matches_float64(cuda):
    """d = 6, dc = 40, 3 agents: the FFMA critic pass (orl_critic_values above dc = 8) against a float64 forward of the
    oracle critic, and one FFMA update (max(d, dc) > 8) over the whole buffer against float64 autograd of the oracle
    loss (oracle/ppo.py) on the same rows."""
    import torch

    from oracle import gae as ogae, loop, nets, ppo as oppo
    from openrl_b200.envs.vec_env import HostVecEnv

    N, A, T = 128, 3, 16
    flags = ["--seed", "5", "--episode_length", str(T), "--ppo_epoch", "1", "--num_mini_batch", "1",
             "--use_valuenorm", "false", "--host_env_groups", "false"]
    host = _DictHost(N, A, masks=False)
    cfg, net, agent = make_agent(HostVecEnv(host), flags)
    drv, tr, b = agent.driver, agent.driver.trainer, agent.driver.buffer.data
    assert (tr.d, tr.dc) == (6, 40) and not tr.use_tensor_cores
    drv.actor_rollout()
    drv.compute_returns()
    torch.cuda.synchronize()
    f64 = lambda model: {k: v.detach().cpu().double() for k, v in model.state_dict().items()}  # noqa: E731
    pol, cri = f64(net.module.models["policy"]), f64(net.module.models["critic"])
    ocfg = loop.cfg_from_flags(" ".join(flags))
    rows = lambda x, w: x.detach().cpu().double().reshape(-1, w)  # noqa: E731
    with torch.no_grad():
        v64, _ = nets.critic_forward(cri, ocfg, rows(b.critic_obs, 40), None, None)
    np.testing.assert_allclose(b.value_preds.cpu().numpy().reshape(-1), v64.numpy().reshape(-1), rtol=0, atol=5e-5)

    total = T * N * A
    idx = torch.randperm(total, generator=torch.Generator().manual_seed(2))
    pol = {k: v.clone().requires_grad_(True) for k, v in pol.items() if k in dict(net.module.models["policy"].named_parameters())}
    cri = {k: v.clone().requires_grad_(True) for k, v in cri.items() if k in dict(net.module.models["critic"].named_parameters())}
    opt_p, opt_c = oppo.make_optimizers(ocfg, pol, cri)
    npy = lambda x: x.cpu().numpy().astype(np.float64)  # noqa: E731
    _, adv = ogae.advantages(npy(b.returns), npy(b.value_preds), npy(b.active_masks), None, cfg.use_adv_normalize)
    adv = torch.from_numpy(adv.astype(np.float64)).reshape(-1, 1)
    sl = lambda x, w: rows(x[:T] if x.shape[0] == T + 1 else x, w)[idx]  # noqa: E731
    batch = dict(critic_obs=sl(b.critic_obs, 40), policy_obs=sl(b.policy_obs, 6), actions=sl(b.actions, 1),
                 value_preds=sl(b.value_preds, 1), returns=sl(b.returns, 1), active_masks=sl(b.active_masks, 1),
                 old_logp=sl(b.action_log_probs, 1), adv=adv[idx], action_masks=sl(b.action_masks, 5))
    oppo.ppo_update(ocfg, pol, cri, opt_p, opt_c, None, batch)
    tr.sync_lrs()
    tr.ppo_update(b, total, idx.cuda().contiguous())
    torch.cuda.synchronize()
    grads = tr.grads.cpu().numpy()
    for net_i, params in ((0, pol), (1, cri)):
        want = np.concatenate([p.grad.numpy().reshape(-1) for p in params.values()])
        got = grads[net_i, :want.size]
        scale = np.linalg.norm(got) / max(np.linalg.norm(want), 1e-30)   # clip_grad_norm_ rescaled the oracle's .grad
        np.testing.assert_allclose(got, want * scale, rtol=2e-3, atol=2e-6 * np.abs(got).max())
        assert abs(scale - 1.0) < 1e-3 or np.linalg.norm(got) > cfg.max_grad_norm


def test_wide_critic_gru_update_matches_float64(cuda, no_tf32):
    """d = 6, dc = 40, 64 envs x 3 agents, T = 16, chunks of 4: one recurrent update over the whole buffer (768 chunks,
    3072 row-steps: three tape row blocks) against rnn_ref64 with the critic width dc, at the bars of
    test_rnn_scale_cuda.py; the recurrent critic pass replays critic_obs."""
    import torch

    import rnn_ref64
    from openrl_b200.envs.vec_env import HostVecEnv
    from scale_harness import c3_buf, drive, rnn_compare

    N, A, T, L = 64, 3, 16, 4
    flags = ["--seed", "6", "--use_recurrent_policy", "true", "--episode_length", str(T), "--data_chunk_length", str(L),
             "--ppo_epoch", "1", "--num_mini_batch", "1", "--use_valuenorm", "true", "--host_env_groups", "false"]
    cfg, net, agent = make_agent(HostVecEnv(_DictHost(N, A, masks=False)), flags)
    drv, tr, b = agent.driver, agent.driver.trainer, agent.driver.buffer.data
    assert (tr.d, tr.n, tr.dc) == (6, 5, 40)
    drv.actor_rollout()
    a = drv._rnn_args(0, T, None)
    assert (a.critic_obs, a.critic_obs_dim) == (b.critic_obs.data_ptr(), 40)
    drv.compute_returns()
    torch.cuda.synchronize()
    pol, cri = net.module.models["policy"], net.module.models["critic"]
    m = tr.algo_module
    op, oc = m.optimizers["policy"], m.optimizers["critic"]
    vn = cri.value_normalizer
    live = dict(pol=pol.flat_params, cri=cri.flat_params, pol_m=op.exp_avg, pol_v=op.exp_avg_sq, cri_m=oc.exp_avg,
                cri_v=oc.exp_avg_sq, vn=vn.state)
    state = dict({k: v.clone() for k, v in live.items()}, steps=[int(x) for x in m.adam_steps])
    total = T * N * A // L
    ids = torch.randperm(total, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3)).contiguous()
    tr.tape = torch.empty(int(tr._lib.orl_rnn_workspace_floats(total * L, tr.rnn_stride)), dtype=torch.float32, device="cuda")
    tr.sync_lrs()
    a = tr._rnn_args(b, ids, b.gae_stats[5:8])
    assert (a.critic_obs, a.critic_obs_dim) == (b.critic_obs.data_ptr(), 40)
    grads, la, after = drive(a, tr.rnn_grads, tr.loss_acc, live)
    tr.tape = None
    np_, nc = int(pol.flat_params.numel()), int(cri.flat_params.numel())
    k = dict(grad_pol=grads[0, :np_], grad_cri=grads[1, :nc], losses=la, steps=[int(x) for x in m.adam_steps], **after)
    rcfg = types.SimpleNamespace(**vars(cfg), vn_beta=vn.beta)
    dims = (tr.d, tr.n, tr.dc)
    buf = c3_buf(b)
    r64, r32 = (rnn_ref64.update(rcfg, buf, state, ids, L, dims, joint=False, dtype=dt) for dt in (torch.float64, torch.float32))
    rnn_compare("dict-obs-d6-dc40-A3-L4-768chunks-3072rows", dims, k, r64, r32, check_vn=True)


def _staged_block(rng, B, d, dc, n, with_critic, with_masks, n_agents):
    parts = [rng.standard_normal(B * d)]
    if with_critic:
        parts.append(rng.standard_normal(B * dc))
    parts += [rng.standard_normal(B), (rng.random(B) < 0.4).astype(np.float64)]
    dones = parts[-1].reshape(-1, n_agents)
    dones[rng.random(dones.shape[0]) < 0.3] = 1.0          # some envs with every agent done
    if with_masks:
        parts.append((rng.random(B * n) < 0.5).astype(np.float64))
    return np.concatenate(parts).astype(np.float32)


@pytest.mark.parametrize("rnn", [False, True])
def test_insert_kernels_with_and_without_critic_section(cuda, rnn):
    """orl_host_insert(_rnn) on blocks of the masked host tests' shapes (1 agent x 5 obs x 5 actions, 3 agents x 6 obs x
    5 actions): with critic_obs_next == NULL the block has no critic section and every output is what the insert
    computes from it (the rule of the parent's insert); with a critic section the policy rows, rewards, masks, action
    masks and hidden-state zeroing are the same and critic_obs[t+1] gets the section; critic_obs_dim outside 1..64 is
    rejected."""
    import torch

    from openrl_b200 import lib

    L = lib.load()
    rng = np.random.default_rng(1)
    for n_envs, A, d, n in ((37, 1, 5, 5), (64, 3, 6, 5)):
        B, dc = n_envs * A, 40
        for with_masks in (False, True):
            base = _staged_block(rng, B, d, dc, n, False, with_masks, A)
            crit = rng.standard_normal(B * dc).astype(np.float32)
            blocks = {False: base, True: np.concatenate([base[:B * d], crit, base[B * d:]])}
            outs = {}
            for with_critic, blk in blocks.items():
                dev = torch.from_numpy(blk).cuda()
                o = dict(obs=torch.full((B, d), -9.0, device="cuda"), rew=torch.full((B,), -9.0, device="cuda"),
                         masks=torch.full((B,), -9.0, device="cuda"), active=torch.full((B,), -9.0, device="cuda"),
                         am=torch.full((B, n), -9.0, device="cuda"), cri=torch.full((B, dc), -9.0, device="cuda"),
                         h=torch.full((B, 64), -9.0, device="cuda"))
                args = (lib.ptr(dev), n_envs, A, d, lib.ptr(o["obs"]), lib.ptr(o["rew"]), lib.ptr(o["masks"]),
                        lib.ptr(o["active"]))
                am = lib.ptr(o["am"]) if with_masks else None
                cri = lib.ptr(o["cri"]) if with_critic else None
                s = lib.current_stream()
                if rnn:
                    rc = L.orl_host_insert_rnn(*args, lib.ptr(o["h"]), am, n, cri, dc if with_critic else 0, s)
                else:
                    rc = L.orl_host_insert(*args, am, n, cri, dc if with_critic else 0, s)
                assert rc == 0
                torch.cuda.synchronize()
                outs[with_critic] = {k: v.cpu().numpy() for k, v in o.items()}
            # the insert rule, from the block without a critic section
            obs, rew = base[:B * d].reshape(B, d), base[B * d:B * d + B]
            dn = base[B * d + B:B * (d + 2)].reshape(n_envs, A) != 0
            env_done = np.repeat(dn.all(1, keepdims=True), A, axis=1).reshape(-1)
            want_masks = np.where(env_done, 0.0, 1.0).astype(np.float32)
            want_active = np.where(dn.reshape(-1) & ~env_done, 0.0, 1.0).astype(np.float32)
            for with_critic, o in outs.items():
                assert np.array_equal(o["obs"], obs) and np.array_equal(o["rew"], rew)
                assert np.array_equal(o["masks"], want_masks) and np.array_equal(o["active"], want_active)
                want_am = base[B * (d + 2):].reshape(B, n) if with_masks else np.full((B, n), -9.0, np.float32)
                assert np.array_equal(o["am"], want_am)
                want_cri = crit.reshape(B, dc) if with_critic else np.full((B, dc), -9.0, np.float32)
                assert np.array_equal(o["cri"], want_cri)
                if rnn:
                    assert (o["h"][env_done] == 0).all() and (o["h"][~env_done] == -9.0).all()
                else:
                    assert (o["h"] == -9.0).all()
            assert env_done.any() and (~env_done).any()
    # critic_obs_dim outside 1..64 with a critic pointer
    x = torch.zeros(4096, device="cuda")
    p = lib.ptr(x)
    for dc in (0, 65):
        rc = (L.orl_host_insert_rnn(p, 2, 1, 4, p, p, p, p, p, None, 0, p, dc, lib.current_stream()) if rnn else
              L.orl_host_insert(p, 2, 1, 4, p, p, p, p, None, 0, p, dc, lib.current_stream()))
        assert rc == 10001, (dc, rc)     # ORL_ERR_BAD_ARG


def test_dict_obs_host_refusals(cuda):
    """use_share_model computes the value from policy_obs, so a Dict host env is refused with it; JRPO stays refused on
    host envs, Dict or not."""
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.vec_env import HostVecEnv
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.logger import Logger

    for extra, match in ((["--use_share_model", "true"], "use_share_model"),
                         (["--use_recurrent_policy", "true", "--use_joint_action_loss", "true"], "JRPO")):
        cfg = create_config_parser().parse_args(["--episode_length", "8"] + extra)
        cfg.quiet = True
        agent = PPOAgent(PPONet(HostVecEnv(_DictHost(4, 3, d=6, dc=9)), cfg=cfg, device="cuda:0"))
        with pytest.raises(NotImplementedError, match=match):
            agent.train(total_time_steps=8 * 4, logger=Logger(quiet=True))


@pytest.mark.parametrize("recurrent", [False, True])
def test_dict_obs_host_env_trains_and_evaluates(cuda, recurrent):
    """make(..., make_custom_envs=...) with the Dict toy env: PPOAgent.train in both loops, then evaluate_policy (the
    actor reads obs["policy"]) and EvalCallback during training."""
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.callbacks import EvalCallback
    from openrl_b200.utils.evaluation import evaluate_policy
    from openrl_b200.utils.logger import Logger

    T, N = 16, 6
    flags = ["--episode_length", str(T), "--log_interval", "1"]
    if recurrent:
        flags += ["--use_recurrent_policy", "true", "--data_chunk_length", "4"]
    for grouped in ("false", "true"):
        cfg = create_config_parser().parse_args(flags + ["--host_env_groups", grouped])
        cfg.quiet = True
        agent = PPOAgent(PPONet(_make(N), cfg=cfg, device="cuda:0"))
        logger = Logger(quiet=True)
        cb = EvalCallback(_make(2), n_eval_episodes=2, eval_freq=T)     # after every iteration
        agent.train(total_time_steps=T * N * 2, logger=logger, callback=cb)
        logs = [h[1] for h in logger.history if "value_loss" in h[1]]
        assert len(logs) == 2 and all(np.isfinite(list(v.values())).all() for v in logs), logs
        assert 0.0 <= cb.last_mean_reward <= 5.0 and cb._evals_done == 2
        mean, std = evaluate_policy(agent, _make(3), n_eval_episodes=3)
        assert np.isfinite(mean) and 0.0 <= mean <= 5.0     # five payoffs in [0, 1) per episode
