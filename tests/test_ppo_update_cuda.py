"""Fused PPO update (orl_ppo_fwdbwd / reduce / apply) against the torch-CPU oracle and the
reference's golden traces.  Tolerance: fp32 losses within 1e-4 relative (north_star), gradients
and parameters compared through the oracle on identical inputs."""
import os

import numpy as np
import pytest

from conftest import GOLDEN

pytestmark = pytest.mark.gpu


def _setup(d, flags_extra=()):
    import torch

    from openrl_b200.algorithms.ppo import PPOAlgorithm
    from openrl_b200.buffers import NormalReplayBuffer
    from test_rollout_cuda import _product

    flags = str(d["meta/flags"]).split() + list(flags_extra)
    cfg, env, net, agent = _product("CartPole-v1", int(d["meta/env_num"]), flags, golden=d)
    trainer = PPOAlgorithm(cfg, net.module, agent_num=1, device=net.device)
    buf = NormalReplayBuffer(cfg, 1, env.observation_space, env.action_space, device=net.device)
    return cfg, net, trainer, buf


def _load_buffer(buf, d, it):
    import torch

    b = buf.data
    g = lambda k: torch.from_numpy(d[f"it{it}/{k}"]).cuda()
    b.policy_obs.copy_(g("policy_obs"))
    b.actions.copy_(g("actions"))
    b.action_log_probs.copy_(g("action_log_probs"))
    b.rewards.copy_(g("rewards"))
    b.masks.copy_(g("masks"))
    b.active_masks.copy_(g("active_masks"))
    b.value_preds.copy_(g("value_preds"))


@pytest.mark.parametrize("tag", ["cartpole", "cartpole_c1"])
def test_first_iteration_updates_match_reference(cuda, tag):
    """Golden rollout buffer of iteration 0 -> GAE kernel -> all updates of the iteration; compare
    the 6 scalars of every update with the reference's (ppo.py:166-176) and the resulting
    parameters / ValueNorm state."""
    import torch

    d = np.load(os.path.join(GOLDEN, f"trace_{tag}.npz"), allow_pickle=True)
    cfg, net, trainer, buf = _setup(d)
    _load_buffer(buf, d, 0)
    vn = net.module.get_critic_value_normalizer()
    buf.data.compute_returns(buf.data.value_preds[-1].clone(), vn)
    torch.cuda.synchronize()
    np.testing.assert_allclose(buf.data.returns.cpu().numpy()[:-1], d["it0/returns"][:-1], rtol=1e-6, atol=1e-6)
    perms = d["it0/perms"]
    T, N = cfg.episode_length, int(d["meta/env_num"])
    total = T * N
    mb = total // cfg.num_mini_batch
    want = d["it0/updates"]
    got = []
    trainer.lrs.copy_(torch.tensor([cfg.lr, cfg.critic_lr]))
    u = 0
    for e in range(cfg.ppo_epoch):
        perm = torch.from_numpy(perms[e]).cuda()
        for i in range(cfg.num_mini_batch):
            trainer.train_info.zero_()
            trainer.ppo_update(buf.data, mb, perm[i * mb:(i + 1) * mb].contiguous())
            got.append(trainer.train_info.cpu().numpy().copy())
            u += 1
    got = np.array(got, np.float64)
    # order of the reference tuple: value_loss, critic_grad_norm, policy_loss, dist_entropy, actor_grad_norm, ratio
    for col, name in enumerate(["value_loss", "critic_grad_norm", "policy_loss", "dist_entropy", "actor_grad_norm", "ratio"]):
        np.testing.assert_allclose(got[:, col], want[:, col], rtol=1e-4, atol=2e-6, err_msg=name)
    for mk in ("policy", "critic"):
        for k, v in net.module.models[mk].state_dict().items():
            gk = f"it0/params/{mk}.{k}"
            if gk in d:
                np.testing.assert_allclose(v.cpu().numpy(), d[gk], rtol=1e-3, atol=0.1 * cfg.lr, err_msg=gk)   # an element whose gradient is at the noise floor may move by a few % of one Adam step
    np.testing.assert_allclose(vn.state.cpu().numpy(), d["it0/vn_after_update"], rtol=1e-5)


def test_gradients_match_oracle_autograd(cuda):
    """True (unfolded) gradients written by orl_ppo_apply vs torch autograd on the oracle nets."""
    import torch

    from oracle import loop, nets, ppo as oppo

    d = np.load(os.path.join(GOLDEN, "trace_cartpole.npz"), allow_pickle=True)
    cfg, net, trainer, buf = _setup(d)
    _load_buffer(buf, d, 0)
    vn = net.module.get_critic_value_normalizer()
    buf.data.compute_returns(buf.data.value_preds[-1].clone(), vn)
    total = cfg.episode_length * int(d["meta/env_num"])
    perm = torch.from_numpy(d["it0/perms"][0]).cuda()
    mb = total // cfg.num_mini_batch
    idx = perm[:mb].contiguous()
    # oracle on the same minibatch
    ocfg = loop.cfg_from_flags(str(d["meta/flags"]))
    pol = {k: torch.from_numpy(d["init/policy." + k]).clone() for k, _ in net.module.models["policy"].named_parameters()}
    cri = {k: torch.from_numpy(d["init/critic." + k]).clone() for k, _ in net.module.models["critic"].named_parameters()}
    opt_p, opt_c = oppo.make_optimizers(ocfg, pol, cri)
    ovn = oppo.ValueNormState()
    flat = lambda x: torch.from_numpy(x.reshape(total, -1))
    ii = torch.from_numpy(d["it0/perms"][0][:mb])
    batch = dict(critic_obs=flat(d["it0/policy_obs"][:-1])[ii], policy_obs=flat(d["it0/policy_obs"][:-1])[ii],
                 actions=flat(d["it0/actions"])[ii], value_preds=flat(d["it0/value_preds"][:-1])[ii],
                 returns=flat(d["it0/returns"][:-1])[ii], active_masks=flat(d["it0/active_masks"][:-1])[ii],
                 old_logp=flat(d["it0/action_log_probs"])[ii], adv=flat(d["it0/advantages"])[ii],
                 action_masks=flat(d["it0/action_masks"][:-1])[ii])
    oppo.ppo_update(ocfg, pol, cri, opt_p, opt_c, ovn, batch)
    trainer.lrs.copy_(torch.tensor([cfg.lr, cfg.critic_lr]))
    trainer.ppo_update(buf.data, mb, idx)
    torch.cuda.synchronize()
    grads = trainer.grads.cpu().numpy()
    for net_i, params in ((0, pol), (1, cri)):
        want = np.concatenate([p.grad.numpy().reshape(-1) for p in params.values()])
        got = grads[net_i, :want.size]
        # clip_grad_norm_ rescaled the oracle's .grad in place; undo through the norm ratio
        scale = np.linalg.norm(got) / max(np.linalg.norm(want), 1e-30)
        if os.environ.get("ORL_DUMP_GRADS"):   # development aid: keep the vectors for offline inspection
            np.savez(os.path.join(os.environ["ORL_DUMP_GRADS"], f"grads_net{net_i}.npz"), got=got, want=want * scale)
        np.testing.assert_allclose(got, want * scale, rtol=2e-3, atol=2e-6 * np.abs(got).max())
        assert abs(scale - 1.0) < 1e-3 or np.linalg.norm(got) > cfg.max_grad_norm


def test_whole_buffer_minibatch_equals_permuted_minibatch(cuda):
    """num_mini_batch == 1: the contiguous (indices=NULL) path gives the same update as any
    permutation of all rows (sum over rows), to fp32 reassociation."""
    import torch

    d = np.load(os.path.join(GOLDEN, "trace_cartpole_c1.npz"), allow_pickle=True)
    res = []
    for use_perm in (False, True):
        cfg, net, trainer, buf = _setup(d)
        _load_buffer(buf, d, 0)
        vn = net.module.get_critic_value_normalizer()
        buf.data.compute_returns(buf.data.value_preds[-1].clone(), vn)
        total = cfg.episode_length * int(d["meta/env_num"])
        trainer.lrs.copy_(torch.tensor([cfg.lr, cfg.critic_lr]))
        trainer.train_info.zero_()
        if use_perm:
            trainer.ppo_update(buf.data, total, torch.from_numpy(d["it0/perms"][0]).cuda())
        else:
            trainer.ppo_update(buf.data, total, None, 0, mb_stats=buf.data.gae_stats[5:8])
        res.append((trainer.train_info.cpu().numpy().copy(), net.module.models["policy"].flat_params.cpu().numpy().copy()))
    np.testing.assert_allclose(res[0][0], res[1][0], rtol=2e-5, atol=1e-7)
    np.testing.assert_allclose(res[0][1], res[1][1], rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("tf32", [False, True])
def test_sharded_minibatch_buckets_sum_to_global_bucket(cuda, tf32):
    """Multi-GPU contract on one GPU: two ranks each process half of the global minibatch with norm_rows = global
    rows and global batch moments; the SUM of their gradient buckets (what the NCCL all-reduce produces) equals the
    bucket of the whole minibatch processed by one rank."""
    import torch

    from openrl_b200 import lib

    d = np.load(os.path.join(GOLDEN, "trace_cartpole_c1.npz"), allow_pickle=True)
    cfg, net, trainer, buf = _setup(d)
    trainer.flags = (trainer.flags | lib.PPO_TENSORCORE) if tf32 else (trainer.flags & ~lib.PPO_TENSORCORE)
    _load_buffer(buf, d, 0)
    vn = net.module.get_critic_value_normalizer()
    buf.data.compute_returns(buf.data.value_preds[-1].clone(), vn)
    total = cfg.episode_length * int(d["meta/env_num"])
    perm = torch.from_numpy(d["it0/perms"][0]).cuda()
    L, s = trainer._lib, lib.current_stream()

    def bucket(indices, norm_rows):
        a = trainer._args(buf.data, indices.numel(), indices.contiguous(), 0)
        a.norm_rows = norm_rows
        a.mb_stats = lib.ptr(buf.data.gae_stats[5:8])       # global moments of the whole minibatch
        lib.check(L.orl_ppo_fwdbwd(a, s), "fwdbwd")
        lib.check(L.orl_ppo_reduce(a, s), "reduce")
        return trainer.folded.clone()

    whole = bucket(perm, 0)
    half = total // 2
    parts = bucket(perm[:half], total) + bucket(perm[half:], total)
    got, want = parts.cpu().numpy(), whole.cpu().numpy()   # folded gradients + 8 tail slots (loss sums in 0..2, rest zero)
    np.testing.assert_allclose(got, want, rtol=2e-4, atol=2e-6 * max(float(np.abs(want).max()), 1.0))


def test_tensor_core_update_matches_fp32_update(cuda):
    """wgmma update (split-fp16 operands, fp32 accumulate) vs the fp32 FFMA update on the same shuffled minibatch
    (gather staging): the six scalars within the 1e-4 parity bar, gradients to fp32-class accuracy."""
    import torch

    from openrl_b200 import lib

    d = np.load(os.path.join(GOLDEN, "trace_cartpole_c1.npz"), allow_pickle=True)
    res = []
    for tf32 in (False, True):
        cfg, net, trainer, buf = _setup(d)
        trainer.flags = (trainer.flags | lib.PPO_TENSORCORE) if tf32 else (trainer.flags & ~lib.PPO_TENSORCORE)
        _load_buffer(buf, d, 0)
        vn = net.module.get_critic_value_normalizer()
        buf.data.compute_returns(buf.data.value_preds[-1].clone(), vn)
        total = cfg.episode_length * int(d["meta/env_num"])
        trainer.lrs.copy_(torch.tensor([cfg.lr, cfg.critic_lr]))
        trainer.train_info.zero_()
        trainer.ppo_update(buf.data, total, torch.from_numpy(d["it0/perms"][0]).cuda())
        torch.cuda.synchronize()
        res.append((trainer.train_info.cpu().numpy().copy(), trainer.grads.cpu().numpy().copy(),
                    net.module.models["policy"].flat_params.cpu().numpy().copy()))
    info32, info_tc = res[0][0], res[1][0]
    np.testing.assert_allclose(info_tc, info32, rtol=1e-4, atol=1e-6)
    for net_i in range(2):
        g32, gtc = res[0][1][net_i], res[1][1][net_i]
        assert np.linalg.norm(gtc - g32) <= 1e-4 * np.linalg.norm(g32), (np.linalg.norm(gtc - g32), np.linalg.norm(g32))
    np.testing.assert_allclose(res[1][2], res[0][2], rtol=0, atol=2e-5)


def test_tensor_core_partial_tile_and_idle_ctas(cuda):
    """Minibatch smaller than one tile (rows < 128) and far fewer tiles than CTAs."""
    import torch

    from openrl_b200 import lib

    d = np.load(os.path.join(GOLDEN, "trace_cartpole.npz"), allow_pickle=True)
    res = []
    for tf32 in (False, True):
        cfg, net, trainer, buf = _setup(d)
        trainer.flags = (trainer.flags | lib.PPO_TENSORCORE) if tf32 else (trainer.flags & ~lib.PPO_TENSORCORE)
        _load_buffer(buf, d, 0)
        vn = net.module.get_critic_value_normalizer()
        buf.data.compute_returns(buf.data.value_preds[-1].clone(), vn)
        trainer.lrs.copy_(torch.tensor([cfg.lr, cfg.critic_lr]))
        trainer.train_info.zero_()
        idx = torch.from_numpy(d["it0/perms"][0][:100]).cuda().contiguous()
        trainer.ppo_update(buf.data, 100, idx)
        torch.cuda.synchronize()
        res.append(trainer.train_info.cpu().numpy().copy())
    np.testing.assert_allclose(res[1], res[0], rtol=1e-4, atol=1e-6)


def test_algorithm_train_accepts_host_numpy_replay_data(cuda, monkeypatch):
    """The reference's algorithm-level seam with a HOST buffer (tests/test_algorithm/test_ppo_algorithm.py:76-82:
    `PPOAlgorithm(cfg, module).train(buffer.data)`, buffer = numpy ReplayData): the golden rollout of iteration 0
    handed over as plain numpy arrays under the reference's attribute names must reproduce the reference's
    updates of that iteration (same minibatch permutations)."""
    import types

    import torch

    d = np.load(os.path.join(GOLDEN, "trace_cartpole.npz"), allow_pickle=True)
    cfg, net, trainer, buf = _setup(d)
    host = types.SimpleNamespace(**{k: d[f"it0/{k}"].copy() for k in
                                    ("policy_obs", "critic_obs", "value_preds", "returns", "masks", "bad_masks", "active_masks",
                                     "actions", "action_log_probs", "rewards", "action_masks")})
    # the golden value_preds were recorded after compute_returns (normalised predictions, as train_ppo sees them)
    perms = [torch.from_numpy(p) for p in d["it0/perms"]]
    monkeypatch.setattr(torch, "randperm", lambda *a, **k: perms.pop(0))
    info = trainer.train(host)
    want = d["it0/updates"].mean(axis=0)
    for col, name in enumerate(["value_loss", "critic_grad_norm", "policy_loss", "dist_entropy", "actor_grad_norm", "ratio"]):
        np.testing.assert_allclose(info[name], want[col], rtol=1e-4, atol=2e-6, err_msg=name)
    assert trainer.h2d_bytes > 0
