"""Flag matrix of the PPO update (modelled on the reference's tests/test_buffer/test_generator.py and
test_ppo_algorithm.py flag sweeps): every loss / normalisation / mask / optimiser option of the hot path,
CUDA update vs the torch-CPU oracle on the same synthetic minibatch with NON-trivial active masks."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CASES = [
    [],
    ["--use_huber_loss", "false"],
    ["--use_clipped_value_loss", "false"],
    ["--use_valuenorm", "false"],
    ["--use_value_active_masks", "false", "--use_policy_active_masks", "false"],
    ["--use_adv_normalize", "true"],
    ["--use_max_grad_norm", "false"],
    ["--weight_decay", "0.01", "--lr", "1e-3", "--critic_lr", "2e-3"],
    ["--activation_id", "0"],
    ["--activation_id", "2"],
    ["--activation_id", "3"],
    ["--clip_param", "0.05", "--entropy_coef", "0.05", "--value_loss_coef", "1.0", "--huber_delta", "0.5"],
    ["--max_grad_norm", "0.5"],
    ["--use_proper_time_limits", "true"],
    ["--use_gae", "false"],
    ["--dual_clip_ppo", "true", "--dual_clip_coeff", "1.05"],
    ["A2C"],
]


def _build(flags, env_id="GridWorldEnv", N=24, T=20, seed=3):
    a2c = "A2C" in flags
    flags = [f for f in flags if f != "A2C"]
    import torch

    from openrl_b200.algorithms.ppo import PPOAlgorithm
    from openrl_b200.buffers import NormalReplayBuffer
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.common import make
    from openrl_b200.modules.common import PPONet

    cfg = create_config_parser().parse_args(["--seed", str(seed), "--episode_length", str(T), "--parity_mode", "true"] + flags)
    cfg.quiet = True
    env = make(env_id, env_num=N)
    net = PPONet(env, cfg=cfg, device="cuda:0")
    cfg.n_rollout_threads = N
    from openrl_b200.algorithms import A2CAlgorithm

    trainer = (A2CAlgorithm if a2c else PPOAlgorithm)(cfg, net.module, agent_num=1, device=net.device)
    buf = NormalReplayBuffer(cfg, 1, env.observation_space, env.action_space, device=net.device)
    cfg.a2c = a2c
    return cfg, net, trainer, buf


@pytest.mark.parametrize("flags", CASES, ids=[" ".join(c) or "default" for c in CASES])
def test_update_flag_matrix_vs_oracle(cuda, flags):
    import torch

    from oracle import gae as ogae, loop, ppo as oppo

    cfg, net, trainer, buf = _build(flags)
    b = buf.data
    T, N = cfg.episode_length, cfg.n_rollout_threads
    g = torch.Generator().manual_seed(11)
    b.policy_obs.copy_(torch.randint(0, 10, b.policy_obs.shape, generator=g).float())
    b.actions.copy_(torch.randint(0, 5, b.actions.shape, generator=g).float())
    b.action_log_probs.copy_(-1.6 + 0.15 * torch.randn(b.action_log_probs.shape, generator=g))
    b.rewards.copy_(torch.randn(b.rewards.shape, generator=g))
    b.value_preds.copy_(0.5 * torch.randn(b.value_preds.shape, generator=g))
    b.masks.copy_((torch.rand(b.masks.shape, generator=g) > 0.1).float())
    b.bad_masks.copy_((torch.rand(b.bad_masks.shape, generator=g) > 0.1).float())
    b.active_masks.copy_((torch.rand(b.active_masks.shape, generator=g) > 0.25).float())
    vn = net.module.get_critic_value_normalizer()
    if vn is not None:
        vn.state.copy_(torch.tensor([0.02, 0.3, 0.05]))
    vn_state0 = None if vn is None else vn.state.cpu().numpy().copy()
    b.compute_returns(b.value_preds[-1].clone(), vn)
    torch.cuda.synchronize()

    # ---- oracle on the same data ----
    ocfg = loop.make_cfg(**{k: getattr(cfg, k) for k in loop.DEFAULTS if hasattr(cfg, k)})
    ocfg.a2c = cfg.a2c
    h = lambda x: x.cpu().numpy()
    ret_o, vp_o = ogae.compute_returns(h(b.rewards), h(b.value_preds), h(b.masks), h(b.bad_masks), h(b.value_preds)[-1],
                                       cfg.gamma, cfg.gae_lambda, cfg.use_gae, cfg.use_proper_time_limits,
                                       vn_state0 if (cfg.use_gae or cfg.use_proper_time_limits) else None)
    assert np.array_equal(ret_o[:-1], h(b.returns)[:-1])  # GAE kernel bit-exact in every branch
    _, adv_o = ogae.advantages(ret_o, vp_o, h(b.active_masks), vn_state0, cfg.use_adv_normalize)
    total = T * N
    mb = total // 2
    perm = torch.randperm(total, generator=g)
    idx = perm[:mb]
    pol = {k: v.detach().cpu().clone() for k, v in net.module.models["policy"].named_parameters()}
    cri = {k: v.detach().cpu().clone() for k, v in net.module.models["critic"].named_parameters()}
    opt_p, opt_c = oppo.make_optimizers(ocfg, pol, cri)
    ovn = oppo.ValueNormState(vn_state0) if vn is not None else None
    flat = lambda x: torch.from_numpy(np.ascontiguousarray(x)).reshape(total, -1)
    batch = dict(critic_obs=flat(h(b.policy_obs)[:-1])[idx], policy_obs=flat(h(b.policy_obs)[:-1])[idx],
                 actions=flat(h(b.actions))[idx], value_preds=flat(vp_o[:-1])[idx], returns=flat(ret_o[:-1])[idx],
                 active_masks=flat(h(b.active_masks)[:-1])[idx], old_logp=flat(h(b.action_log_probs))[idx],
                 adv=flat(adv_o)[idx], action_masks=torch.ones(mb, 5))
    want = oppo.ppo_update(ocfg, pol, cri, opt_p, opt_c, ovn, batch)

    # ---- CUDA ----
    trainer.lrs.copy_(torch.tensor([cfg.lr, cfg.critic_lr]))
    trainer.train_info.zero_()
    trainer.ppo_update(b, mb, idx.cuda().contiguous())
    torch.cuda.synchronize()
    got = trainer.train_info.cpu().numpy()
    for col, name in enumerate(["value_loss", "critic_grad_norm", "policy_loss", "dist_entropy", "actor_grad_norm", "ratio"]):
        np.testing.assert_allclose(got[col], want[col], rtol=2e-4, atol=5e-6, err_msg=name)
    for mk, params in (("policy", pol), ("critic", cri)):
        for k, v in net.module.models[mk].named_parameters():
            np.testing.assert_allclose(v.detach().cpu().numpy(), params[k].detach().numpy(), rtol=1e-3, atol=0.1 * max(cfg.lr, cfg.critic_lr),
                                       err_msg=f"{mk}.{k}")
    if vn is not None:
        np.testing.assert_allclose(vn.state.cpu().numpy(), ovn.state(), rtol=1e-5)


def test_fast_mode_multi_minibatch_and_odd_sizes(cuda):
    """Fast mode (wgmma) with num_mini_batch > 1, rows not a multiple of the 128-row tile, device randperm."""
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.common import make
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.logger import Logger

    cfg = create_config_parser().parse_args(["--episode_length", "37", "--ppo_epoch", "3", "--num_mini_batch", "3", "--log_interval", "1"])
    cfg.quiet = True
    env = make("CartPole-v1", env_num=53)
    agent = PPOAgent(PPONet(env, cfg=cfg, device="cuda:0"))
    logger = Logger(quiet=True)
    agent.train(total_time_steps=37 * 53 * 4, logger=logger)
    assert agent.driver.trainer.use_tensor_cores
    logs = [h[1] for h in logger.history if "value_loss" in h[1]]
    assert len(logs) == 4 and all(np.isfinite(list(l.values())).all() for l in logs)
    assert all(abs(l["ratio"] - 1.0) < 0.05 for l in logs)


def test_save_load_roundtrip_and_lr_decay(cuda, tmp_path):
    """agent.save / agent.load (rl_agent.py:187-213) and use_linear_lr_decay (ppo_module.py:91-100)."""
    import torch

    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.common import make
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent

    cfg = create_config_parser().parse_args(["--episode_length", "16", "--ppo_epoch", "2", "--use_linear_lr_decay", "true"])
    cfg.quiet = True
    env = make("CartPole-v1", env_num=8)
    agent = PPOAgent(PPONet(env, cfg=cfg, device="cuda:0"))
    agent.train(total_time_steps=16 * 8 * 4)
    lr_now = agent.net.module.optimizers["policy"].param_groups[0]["lr"]
    assert abs(lr_now - cfg.lr * (1 - 3 / 4)) < 1e-12
    agent.save(tmp_path / "ckpt")
    ref = {k: v.clone() for k, v in agent.net.module.models["policy"].state_dict().items()}
    obs, _ = env.reset(seed=9)
    a1, _ = agent.act(obs, deterministic=True)
    cfg2 = create_config_parser().parse_args(["--episode_length", "16", "--seed", "5"])
    cfg2.quiet = True
    agent2 = PPOAgent(PPONet(make("CartPole-v1", env_num=8), cfg=cfg2, device="cuda:0"))
    agent2.load(tmp_path / "ckpt")
    for k, v in agent2.net.module.models["policy"].state_dict().items():
        assert torch.equal(v, ref[k]), k
    a2, _ = agent2.act(obs, deterministic=True)
    assert np.array_equal(a1, a2)


@pytest.mark.parametrize("n_actions", [2, 3, 5, 8])
def test_tensor_core_kernel_head_width_templates(cuda, n_actions):
    """The wgmma kernel is instantiated for head widths 2, 5 and a generic (runtime n <= 8) variant:
    each must agree with the fp32 kernel on the same synthetic minibatch (incl. a partial last tile)."""
    import torch

    from openrl_b200 import lib, spaces
    from openrl_b200.algorithms.ppo import PPOAlgorithm
    from openrl_b200.buffers import NormalReplayBuffer
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.modules.common import PPONet

    class Env:
        agent_num, parallel_env_num = 1, 37
        observation_space, action_space = spaces.Box(-5, 5, (6,), np.float32), spaces.Discrete(n_actions)

        def reset(self, seed=None):
            return np.zeros((37, 1, 6), np.float32)

    T, N = 23, 37
    res = []
    for tf32 in (False, True):
        cfg = create_config_parser().parse_args(["--seed", "4", "--episode_length", str(T), "--parity_mode", "true"])
        cfg.quiet = True
        net = PPONet(Env(), cfg=cfg, device="cuda:0")
        cfg.n_rollout_threads = N
        trainer = PPOAlgorithm(cfg, net.module, agent_num=1, device=net.device)
        trainer.flags = (trainer.flags | lib.PPO_TENSORCORE) if tf32 else (trainer.flags & ~lib.PPO_TENSORCORE)
        buf = NormalReplayBuffer(cfg, 1, Env.observation_space, Env.action_space, device=net.device)
        b = buf.data
        g = torch.Generator().manual_seed(5)
        b.policy_obs.copy_(torch.randn(b.policy_obs.shape, generator=g))
        b.actions.copy_(torch.randint(0, n_actions, b.actions.shape, generator=g).float())
        b.action_log_probs.copy_(-np.log(n_actions) + 0.1 * torch.randn(b.action_log_probs.shape, generator=g))
        b.rewards.copy_(torch.randn(b.rewards.shape, generator=g))
        b.value_preds.copy_(0.3 * torch.randn(b.value_preds.shape, generator=g))
        b.masks.copy_((torch.rand(b.masks.shape, generator=g) > 0.1).float())
        b.active_masks.copy_((torch.rand(b.active_masks.shape, generator=g) > 0.2).float())
        vn = net.module.get_critic_value_normalizer()
        b.compute_returns(b.value_preds[-1].clone(), vn)
        trainer.lrs.copy_(torch.tensor([cfg.lr, cfg.critic_lr]))
        trainer.train_info.zero_()
        trainer.ppo_update(b, T * N, None, 0, mb_stats=b.gae_stats[5:8])
        torch.cuda.synchronize()
        res.append((trainer.train_info.cpu().numpy().copy(), trainer.grads.cpu().numpy().copy()))
    np.testing.assert_allclose(res[1][0], res[0][0], rtol=1e-4, atol=1e-6)
    for net_i in range(2):
        g32, gtc = res[0][1][net_i], res[1][1][net_i]
        assert np.linalg.norm(gtc - g32) <= 1e-4 * np.linalg.norm(g32), (n_actions, net_i)


def test_checkpoint_is_pickled_module_with_reference_key_names(cuda, tmp_path):
    """module.pt == torch.save(net.module) (rl_agent.py:187-191); the critic's state_dict carries the reference's ValueNorm
    entries (valuenorm.py:27-35) and loads from a dict spelled with them."""
    import torch

    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.common import make
    from openrl_b200.modules.common import PPONet
    from openrl_b200.modules.ppo_module import PPOModule
    from openrl_b200.runners.common import PPOAgent

    cfg = create_config_parser().parse_args(["--episode_length", "16", "--ppo_epoch", "1"])
    cfg.quiet = True
    agent = PPOAgent(PPONet(make("CartPole-v1", env_num=8), cfg=cfg, device="cuda:0"))
    agent.train(total_time_steps=16 * 8 * 2)
    agent.save(tmp_path / "ck")
    obj = torch.load(tmp_path / "ck" / "module.pt", weights_only=False)
    assert isinstance(obj, PPOModule) and set(obj.models) == {"policy", "critic"}
    sd = agent.net.module.models["critic"].state_dict()
    for k in ("value_normalizer.running_mean", "value_normalizer.running_mean_sq", "value_normalizer.debiasing_term"):
        assert k in sd
    assert sd["value_normalizer.running_mean"].shape == (1,) and sd["value_normalizer.debiasing_term"].shape == ()
    assert float(sd["value_normalizer.debiasing_term"]) > 0
    # a reference-spelled critic state_dict loads
    sd2 = {k: v.clone() for k, v in sd.items()}
    sd2["value_normalizer.running_mean"] += 1.0
    agent.net.module.models["critic"].load_state_dict(sd2)
    assert abs(float(agent.net.module.get_critic_value_normalizer().state[0]) - float(sd2["value_normalizer.running_mean"])) < 1e-7
    # the loaded module keeps training (library handle restored, flat parameter views intact)
    agent2 = PPOAgent(PPONet(make("CartPole-v1", env_num=8), cfg=cfg, device="cuda:0"))
    agent2.load(tmp_path / "ck")
    p0 = agent2.net.module.models["policy"].flat_params.clone()
    agent2.train(total_time_steps=16 * 8)
    assert not torch.equal(p0, agent2.net.module.models["policy"].flat_params)
    for k, v in agent2.net.module.models["policy"].state_dict().items():   # named parameters still alias the flat buffer
        assert v.data_ptr() >= agent2.net.module.models["policy"].flat_params.data_ptr()
