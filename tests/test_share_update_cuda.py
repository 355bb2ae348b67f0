"""The shared policy-value update (cfg.use_share_model): the true gradients written by orl_share_fwdbwd against torch
autograd of the oracle's PolicyValueNetwork on the same minibatch.  At 2*1024 + 37 rows the tape reduction runs three
row blocks, the last one partial; at 5 rows one partial block.  obs_dim 6 gives gemm jobs with N = d = 6 next to the
M = 1 value-head job.  Bar and norm-ratio rescaling of test_ppo_update_cuda.py::test_gradients_match_oracle_autograd."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("rows", [5, 2 * 1024 + 37])
def test_share_gradients_match_oracle_autograd(cuda, rows):
    import torch

    from openrl_b200 import spaces
    from openrl_b200.algorithms.ppo import PPOAlgorithm
    from openrl_b200.buffers.replay_data import ReplayData
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.modules.common import PPONet
    from oracle import loop, nets, ppo as oppo

    d, n = 6, 4
    flags = "--seed 3 --use_share_model true --n_rollout_threads 1 --episode_length " + str(rows)

    class Env:
        agent_num, parallel_env_num = 1, 1
        observation_space, action_space = spaces.Box(-5, 5, (d,), np.float32), spaces.Discrete(n)

        def reset(self, seed=None):
            return np.zeros((1, 1, d), np.float32)

    cfg = create_config_parser().parse_args(flags.split())
    cfg.quiet = True
    net = PPONet(Env(), cfg=cfg, device="cuda:0")
    model = net.module.models["model"]
    trainer = PPOAlgorithm(cfg, net.module, agent_num=1, device=net.device)
    assert trainer.share
    ocfg = loop.cfg_from_flags(flags)
    p = {k: v.detach().cpu().clone() for k, v in model.named_parameters()}
    assert nets.is_shared(p) and sum(v.numel() for v in p.values()) == trainer.share_total

    # a minibatch away from the loss's branch points: ratios within 5% of 1 (clip 0.2), value predictions within 0.1
    # of the values (value clip 0.2), returns ~ N(0, 1) (Huber delta 10), one row in ten inactive
    g = np.random.default_rng(rows)
    obs = torch.from_numpy(g.normal(size=(rows, d)).astype(np.float32))
    actions = torch.from_numpy(g.integers(0, n, size=(rows, 1)).astype(np.float32))
    with torch.no_grad():
        values = nets.critic_forward(p, ocfg, obs)[0]
        logp, _ = nets.policy_eval(p, ocfg, obs, actions)
    f32 = lambda x: torch.from_numpy(np.asarray(x, np.float32))  # noqa: E731
    old_logp = logp + f32(g.uniform(-0.05, 0.05, size=(rows, 1)))
    value_preds = values + f32(g.uniform(-0.1, 0.1, size=(rows, 1)))
    returns, adv = f32(g.normal(size=(rows, 1))), f32(g.normal(size=(rows, 1)))
    active = f32(g.random((rows, 1)) > 0.1)
    # train_ppo normalises the advantages by their mean and std over the active rows (ppo.py:402-409); the kernels take
    # both from the buffer moments gae_stats (ORL_GS_* order)
    a64, r64, act64 = adv.double().view(-1), returns.double().view(-1), active.double().view(-1)
    gae_stats = torch.stack([a64.sum(), (a64 * a64).sum(), torch.tensor(float(rows), dtype=torch.float64), a64 @ act64,
                             (a64 * a64) @ act64, r64.sum(), r64 @ r64, act64.sum()])
    mean = float(gae_stats[3] / gae_stats[7])
    std = float(np.float32(np.sqrt(max(float(gae_stats[4] / gae_stats[7]) - mean * mean, 0.0))))
    adv_n = (adv - float(np.float32(mean))) / float(np.float32(std + 1e-5))

    buf = ReplayData(cfg, 1, Env.observation_space, Env.action_space, episode_length=rows, device="cuda:0")
    for name, v in (("policy_obs", obs), ("actions", actions), ("action_log_probs", old_logp), ("value_preds", value_preds),
                    ("returns", returns), ("active_masks", active), ("advantages", adv)):
        getattr(buf, name).view(-1)[:v.numel()].copy_(v.view(-1))
    buf.gae_stats.copy_(gae_stats)
    perm = torch.from_numpy(g.permutation(rows)).cuda()
    trainer.lrs.copy_(torch.tensor([cfg.lr, cfg.critic_lr]))
    trainer.ppo_update(buf, rows, perm)
    torch.cuda.synchronize()
    got = trainer.share_grads[:trainer.share_total].cpu().numpy()

    ii = torch.from_numpy(perm.cpu().numpy())
    batch = dict(critic_obs=obs[ii], policy_obs=obs[ii], actions=actions[ii], value_preds=value_preds[ii], returns=returns[ii],
                 active_masks=active[ii], old_logp=old_logp[ii], adv=adv_n[ii], action_masks=None)
    opt, _ = oppo.make_optimizers(ocfg, p, p)
    oppo.ppo_update(ocfg, p, p, opt, opt, oppo.ValueNormState(), batch)
    want = np.concatenate([v.grad.numpy().reshape(-1) for v in p.values()])
    # clip_grad_norm_ rescaled the oracle's .grad in place (twice, over the same parameters); undo through the norm ratio
    scale = np.linalg.norm(got) / max(np.linalg.norm(want), 1e-30)
    np.testing.assert_allclose(got, want * scale, rtol=2e-3, atol=2e-6 * np.abs(got).max())
    assert abs(scale - 1.0) < 1e-3 or np.linalg.norm(got) > cfg.max_grad_norm
