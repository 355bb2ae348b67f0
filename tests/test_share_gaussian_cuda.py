"""The shared policy-value network (cfg.use_share_model) with a DiagGaussian head on Box action spaces, on host-stepped
envs (BASELINE config 5 class with `use_share_model`).

- Trace parity: PPOAgent.train over the IdentityEnvcontinuous restatement reproduces the reference's trace
  tests/golden/trace_share_gaussian.npz in parity mode; and the synchronous and the two-group host loop write the same
  bits with device Philox noise.
- One update at the config-5 shape (obs 17, Box(6)) over 2 * 1024 + 37 rows (three tape row blocks, the last one
  partial) against torch autograd of the oracle, with and without the active-mask options: the gradient (rtol 2e-3
  after rescaling the oracle's clipped gradient by the norm ratio), both logged grad norms, the logged losses and the
  clip-twice-then-Adam step from the device's own gradient.  tests/test_share_scale_cuda.py holds the same update to
  float64 block by block, without the rescaling.
- The act's noise: eps = (action - mean) / std is the host Box-Muller of Philox lanes 2..5 (as for the FFMA
  rollout_kernel in test_gaussian_head_cuda.py); deterministic acts return the mean bit for bit.
- A config-5-shaped run trains, and Box(9) is refused."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from helpers import KEYS, make_agent, philox_units
from openrl_b200.envs.vec_env import HostVecEnv

pytestmark = pytest.mark.gpu

class _IdentityHost:
    """Host vec-env with the reference's duck type, backed by the oracle's IdentityEnvcontinuous restatement."""

    def __init__(self, n):
        from openrl_b200 import spaces
        from oracle.envs import IdentityContinuousVec

        self.inner = IdentityContinuousVec(n)
        self.parallel_env_num, self.agent_num = n, 1
        self.observation_space = spaces.Box(0, 2, (1,), np.float32)
        self.action_space = spaces.Box(0, 1, (1,), np.float32)

    def reset(self, seed=None):
        return self.inner.reset(seed=seed)

    def step(self, actions):
        o, r, d, _ = self.inner.step(actions)
        return o, r, d, [{} for _ in range(self.parallel_env_num)]


class _BoxHost:
    """Config-5 stand-in that can step a sub-range of its envs: obs ~ N(0, 1) keyed by (env, its step), reward = -|a|^2,
    episodes of 7 steps.  The trajectories depend on the actions only through the rewards."""

    def __init__(self, n, obs_dim=17, act_dim=6):
        from openrl_b200 import spaces

        self.parallel_env_num, self.agent_num, self.obs_dim, self.act_dim = n, 1, obs_dim, act_dim
        self.observation_space = spaces.Box(-np.inf, np.inf, (obs_dim,), np.float32)
        self.action_space = spaces.Box(-1, 1, (act_dim,), np.float32)
        self.t = np.zeros(n, np.int64)

    def _obs(self, lo, hi):
        return np.stack([np.random.default_rng((e, int(self.t[e]))).standard_normal((1, self.obs_dim)) for e in range(lo, hi)]
                        ).astype(np.float32)

    def reset(self, seed=None):
        self.t[:] = 0
        return self._obs(0, self.parallel_env_num)

    def step_range(self, lo, hi, actions):
        assert actions.shape == (hi - lo, 1, self.act_dim) and np.isfinite(actions).all()
        self.t[lo:hi] += 1
        done = self.t[lo:hi] % 7 == 0
        rewards = -(np.asarray(actions, np.float64) ** 2).sum(-1, keepdims=True)
        return self._obs(lo, hi), rewards, done[:, None], [{} for _ in range(hi - lo)]

    def step(self, actions):
        return self.step_range(0, self.parallel_env_num, actions)


@pytest.mark.parametrize("grouped", ["false", "true"])
def test_share_gaussian_host_env_matches_reference_trace(cuda, grouped):
    """Parity mode draws the reference's noise on the host step by step, which keeps the rollout on the synchronous loop
    whatever host_env_groups says; the two-group loop is pinned to it by the next test."""
    from openrl_b200.utils.logger import Logger

    d = np.load(os.path.join(GOLDEN, "trace_share_gaussian.npz"), allow_pickle=True)
    iters, N = int(d["meta/iters"]), int(d["meta/env_num"])
    flags = str(d["meta/flags"]).split() + ["--parity_mode", "true", "--log_interval", "1", "--host_env_groups", grouped]
    env = HostVecEnv(_IdentityHost(N))
    cfg, net, agent = make_agent(env, flags, golden=d, start=False)
    model = net.module.models["model"]
    assert cfg.use_share_model and model.head_kind == 1 and model.n_actions == 1
    keys = [k for k, _ in model.named_parameters()]
    assert keys[-5:] == ["v_out.weight", "v_out.bias", "act.action_out.fc_mean.weight", "act.action_out.fc_mean.bias",
                         "act.action_out.logstd._bias"]
    logger = Logger(quiet=True)
    agent.train(total_time_steps=cfg.episode_length * N * iters, logger=logger)
    logs = [h[1] for h in logger.history if "value_loss" in h[1]]
    assert len(logs) == iters
    for it in range(iters):
        want = d[f"it{it}/updates"].mean(axis=0)
        for col, name in enumerate(KEYS):
            np.testing.assert_allclose(logs[it][name], want[col], rtol=2e-4, atol=5e-6, err_msg=f"it{it} {name}")
    b = agent.driver.buffer.data
    last = iters - 1
    assert b.actions.shape[-1] == 1 and b.action_log_probs.shape[-1] == 1
    np.testing.assert_allclose(b.actions.cpu().numpy(), d[f"it{last}/actions"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(b.action_log_probs.cpu().numpy(), d[f"it{last}/action_log_probs"], rtol=0, atol=2e-5)
    np.testing.assert_array_equal(b.policy_obs.cpu().numpy()[1:], d[f"it{last}/policy_obs"][1:])
    np.testing.assert_allclose(b.rewards.cpu().numpy(), d[f"it{last}/rewards"], rtol=1e-5, atol=1e-6)
    np.testing.assert_array_equal(b.masks.cpu().numpy(), d[f"it{last}/masks"])
    for k, v in model.state_dict().items():
        gk = f"it{last}/params/model.{k}"
        if gk in d and "value_normalizer" not in k:
            np.testing.assert_allclose(v.cpu().numpy(), d[gk], rtol=2e-3, atol=5e-6, err_msg=gk)


def test_share_gaussian_host_loops_agree(cuda):
    """Device Philox noise, 1024 envs: over two `PPOAgent.train` calls the synchronous and the two-group host loop write
    the same actions, log-probs, observations and rewards and train to the same parameters."""
    import torch

    from openrl_b200.utils.logger import Logger

    N, T = 1024, 16
    flags = ["--seed", "3", "--episode_length", str(T), "--ppo_epoch", "1", "--num_mini_batch", "2", "--use_share_model", "true",
             "--log_interval", "1"]
    runs = []
    for grouped in ("false", "true"):
        env = HostVecEnv(_BoxHost(N))
        cfg, net, agent = make_agent(env, flags + ["--host_env_groups", grouped], start=False)   # PPONet re-seeds: same weights
        assert env.supports_groups
        out = []
        for _ in range(2):
            agent.train(total_time_steps=T * N, logger=Logger(quiet=True))
            torch.cuda.synchronize()
            b = agent.driver.buffer.data
            out.append({k: getattr(b, k).cpu().numpy().copy() for k in ("actions", "action_log_probs", "policy_obs", "rewards", "masks")}
                       | {"params": net.module.models["model"].flat_params.cpu().numpy().copy()})
        assert agent.driver.host_act_steps == 2 * T
        runs.append(out)
    assert runs[0][0]["actions"].shape == (T, N, 1, 6)
    for call in range(2):
        for k in runs[0][call]:
            assert np.array_equal(runs[0][call][k], runs[1][call][k]), (call, k)


def _share_module(d, n, flags):
    from openrl_b200 import spaces
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.modules.common import PPONet

    class Env:
        agent_num, parallel_env_num = 1, 1
        observation_space, action_space = spaces.Box(-5, 5, (d,), np.float32), spaces.Box(-1, 1, (n,), np.float32)

        def reset(self, seed=None):
            return np.zeros((1, 1, d), np.float32)

    cfg = create_config_parser().parse_args(flags.split())
    cfg.quiet = True
    return cfg, Env, PPONet(Env(), cfg=cfg, device="cuda:0")


@pytest.mark.parametrize("masks", [True, False])
def test_share_gaussian_update_matches_oracle_autograd(cuda, masks):
    import torch

    from openrl_b200.algorithms.ppo import PPOAlgorithm
    from openrl_b200.buffers.replay_data import ReplayData
    from oracle import loop, nets, ppo as oppo

    d, n, rows = 17, 6, 2 * 1024 + 37
    # max_grad_norm 0.5 (the default 10 is above this minibatch's norm): both clip_grad_norm_ calls act
    flags = "--seed 3 --use_share_model true --max_grad_norm 0.5 --n_rollout_threads 1 --episode_length " + str(rows)
    if not masks:
        flags += " --use_policy_active_masks false --use_value_active_masks false"
    cfg, Env, net = _share_module(d, n, flags)
    model = net.module.models["model"]
    sd = model.state_dict()
    sd["act.action_out.fc_mean.weight"].mul_(5.0)   # means of order 0.5
    sd["act.action_out.logstd._bias"].copy_(torch.linspace(-0.5, 0.5, n).view(n, 1))
    trainer = PPOAlgorithm(cfg, net.module, agent_num=1, device=net.device)
    assert trainer.share and trainer.head_kind == 1
    ocfg = loop.cfg_from_flags(flags)
    assert ocfg.use_policy_active_masks == masks and ocfg.use_value_active_masks == masks
    p = {k: v.detach().cpu().clone() for k, v in model.named_parameters()}
    assert nets.is_shared(p) and sum(v.numel() for v in p.values()) == trainer.share_total
    before = model.flat_params.cpu().numpy().astype(np.float64)

    # away from the loss's branch points: per-dimension ratios within 5% of 1, value predictions within 0.1 of the values,
    # returns ~ N(0, 1), one row in ten inactive
    g = np.random.default_rng(rows + masks)
    f32 = lambda x: torch.from_numpy(np.asarray(x, np.float32))  # noqa: E731
    obs = f32(g.normal(size=(rows, d)))
    with torch.no_grad():
        values = nets.critic_forward(p, ocfg, obs)[0]
        mean, std = nets.gaussian_params(p, nets.policy_features(p, ocfg, obs)[0])
        actions = mean + std * f32(g.normal(size=(rows, n)))
        logp, _ = nets.policy_eval_gaussian(p, ocfg, obs, actions)
    old_logp = logp + f32(g.uniform(-0.05, 0.05, size=(rows, n)))
    value_preds = values + f32(g.uniform(-0.1, 0.1, size=(rows, 1)))
    returns, adv = f32(g.normal(size=(rows, 1))), f32(g.normal(size=(rows, 1)))
    active = f32(g.random((rows, 1)) > 0.1)
    a64, r64, act64 = adv.double().view(-1), returns.double().view(-1), active.double().view(-1)
    gae_stats = torch.stack([a64.sum(), (a64 * a64).sum(), torch.tensor(float(rows), dtype=torch.float64), a64 @ act64,
                             (a64 * a64) @ act64, r64.sum(), r64 @ r64, act64.sum()])
    mean_a = float(gae_stats[3] / gae_stats[7])
    std_a = float(np.float32(np.sqrt(max(float(gae_stats[4] / gae_stats[7]) - mean_a * mean_a, 0.0))))
    adv_n = (adv - float(np.float32(mean_a))) / float(np.float32(std_a + 1e-5))

    buf = ReplayData(cfg, 1, Env.observation_space, Env.action_space, episode_length=rows, device="cuda:0")
    assert buf.actions.shape[-1] == n and buf.action_log_probs.shape[-1] == n
    for name, v in (("policy_obs", obs), ("actions", actions), ("action_log_probs", old_logp), ("value_preds", value_preds),
                    ("returns", returns), ("active_masks", active), ("advantages", adv)):
        getattr(buf, name).view(-1)[:v.numel()].copy_(v.reshape(-1))
    buf.gae_stats.copy_(gae_stats)
    perm = torch.from_numpy(g.permutation(rows)).cuda()
    trainer.lrs.copy_(torch.tensor([cfg.lr, cfg.critic_lr]))
    trainer.ppo_update(buf, rows, perm)
    torch.cuda.synchronize()
    got = trainer.share_grads[:trainer.share_total].cpu().numpy().astype(np.float64)
    info = trainer.train_info.cpu().numpy().astype(np.float64)
    after = model.flat_params.cpu().numpy().astype(np.float64)

    ii = torch.from_numpy(perm.cpu().numpy())
    batch = dict(critic_obs=obs[ii], policy_obs=obs[ii], actions=actions[ii], value_preds=value_preds[ii], returns=returns[ii],
                 active_masks=active[ii], old_logp=old_logp[ii], adv=adv_n[ii], action_masks=None)
    opt, _ = oppo.make_optimizers(ocfg, p, p)
    want_info = oppo.ppo_update(ocfg, p, p, opt, opt, oppo.ValueNormState(), batch)
    want = np.concatenate([v.grad.numpy().reshape(-1) for v in p.values()]).astype(np.float64)
    # gradient: clip_grad_norm_ rescaled the oracle's .grad in place (twice); undo through the norm ratio
    scale = np.linalg.norm(got) / max(np.linalg.norm(want), 1e-30)
    np.testing.assert_allclose(got, want * scale, rtol=2e-3, atol=2e-6 * np.abs(got).max())
    ls = slice(trainer.share_total - n, trainer.share_total)   # the logstd block gets its own look
    np.testing.assert_allclose(got[ls], want[ls] * scale, rtol=2e-3, atol=2e-6 * np.abs(got).max())
    # logged scalars: slots value_loss, critic_grad_norm, policy_loss, dist_entropy, actor_grad_norm, ratio
    norm1 = float(np.linalg.norm(got))
    assert norm1 > cfg.max_grad_norm and abs(info[1] - cfg.max_grad_norm) < 1e-4   # critic_grad_norm: the clipped norm
    for col, name in enumerate(KEYS):
        np.testing.assert_allclose(info[col], want_info[col], rtol=2e-3 if "norm" in name else 2e-4, atol=1e-5, err_msg=name)
    np.testing.assert_allclose(info[4], norm1, rtol=1e-5)
    # clip twice (torch clip_grad_norm_: coef = max_norm / (norm + 1e-6), clamped to 1), then one Adam step (step 1,
    # weight decay 0: the update is lr * g / (|g| + eps)), from the device's own gradient
    c1 = min(1.0, cfg.max_grad_norm / (norm1 + 1e-6))
    g1 = got * c1
    c2 = min(1.0, cfg.max_grad_norm / (np.linalg.norm(g1) + 1e-6))
    g2 = g1 * c2
    step = cfg.lr * g2 / (np.abs(g2) + cfg.opti_eps)
    np.testing.assert_allclose(after[:trainer.share_total], before[:trainer.share_total] - step, rtol=0, atol=2e-7)


@pytest.mark.parametrize("d,n", [(17, 6), (3, 1), (5, 8)])
def test_share_gaussian_act_noise_is_box_muller_of_lanes_2_to_5(cuda, d, n):
    import torch

    from oracle import loop, nets

    seed, step = 0x2468_ACE0_1357, (1 << 32) + 5
    flags = "--seed 7 --use_share_model true"
    cfg, _, net = _share_module(d, n, flags)
    module = net.module
    model = module.models["model"]
    sd = model.state_dict()
    sd["act.action_out.fc_mean.weight"].mul_(5.0)
    sd["act.action_out.logstd._bias"].copy_(torch.linspace(-0.5, 0.5, n).view(n, 1))
    rows = 128 * 3 + 37
    obs = np.random.default_rng(5).normal(size=(rows, d)).astype(np.float32)
    mean, lp_det = module.act(obs, deterministic=True)
    act, _ = module.act(obs, rng_seed=seed, rng_step=step)
    torch.cuda.synchronize()
    assert act.shape == (rows, n)
    logstd = sd["act.action_out.logstd._bias"].cpu().numpy()[:, 0]
    # deterministic: the mean itself (the float64 oracle at the 1e-5 bar) and the log-prob at zero distance, bit for bit
    p64 = {k: v.detach().cpu().double() for k, v in model.named_parameters()}
    with torch.no_grad():
        want_mean, _ = nets.policy_act_gaussian(p64, loop.cfg_from_flags(flags), torch.from_numpy(obs).double(), deterministic=True)
    np.testing.assert_allclose(mean.cpu().numpy(), want_mean.numpy(), rtol=0, atol=1e-5)
    want_lp = np.broadcast_to(-logstd - np.float32(0.9189385332046727), (rows, n))
    assert np.array_equal(lp_det.cpu().numpy().view(np.int32), want_lp.view(np.int32))
    # stochastic: eps = (action - mean) / std is the host Box-Muller of lanes 2..5
    eps = (act.cpu().numpy().astype(np.float64) - mean.cpu().numpy()) / np.exp(logstd.astype(np.float64))
    u = philox_units(1, rows, seed, step, 0, (2, 3, 4, 5))[0].astype(np.float64)
    u1 = np.concatenate([u[:, 0:4], u[:, 8:12]], 1)
    u2 = np.concatenate([u[:, 4:8], u[:, 12:16]], 1)
    want = np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)
    np.testing.assert_allclose(eps, want[:, :n], rtol=0, atol=1e-5)


def test_share_gaussian_config5_shape_trains(cuda):
    """HalfCheetah-shaped workload with use_share_model: obs 17, Box(6), 1024 host envs, two iterations."""
    from openrl_b200.utils.logger import Logger

    flags = ["--seed", "1", "--episode_length", "16", "--ppo_epoch", "2", "--use_share_model", "true", "--log_interval", "1"]
    env = HostVecEnv(_BoxHost(1024))
    cfg, net, agent = make_agent(env, flags, start=False)
    logger = Logger(quiet=True)
    agent.train(total_time_steps=16 * 1024 * 2, logger=logger)
    logs = [h[1] for h in logger.history if "value_loss" in h[1]]
    assert len(logs) == 2 and all(np.isfinite(list(l.values())).all() for l in logs)
    assert abs(logs[0]["dist_entropy"] - 6 * (0.5 + 0.5 * np.log(2 * np.pi))) < 0.05   # 8.51 at logstd = 0
    assert abs(logs[0]["ratio"] - 1.0) < 1e-3
    assert np.isfinite(net.module.models["model"].flat_params.cpu().numpy()).all()


def test_share_gaussian_wider_than_8_is_refused(cuda):
    with pytest.raises(NotImplementedError):
        _share_module(4, 9, "--seed 0 --use_share_model true")
