"""GRU policies with DiagGaussian heads (cfg.use_recurrent_gaussian_head): the oracle's Gaussian act, eval and update with
the policy's GRU in the path, two envs, and the recurrent oracle loop on them.

TEST INFRASTRUCTURE.  oracle/nets.policy_act_gaussian / policy_eval_gaussian and the Box branch of oracle/ppo.ppo_update
run the feed-forward trunk only.  The functions here are the same maths (ACTLayer continuous branch, act.py:74-77 and
150-158) on `nets.policy_features` with rnn states and masks, and `ppo_update` is oracle/ppo.ppo_update's sequence
(ppo.py:46-176) with that eval, taking the states and masks from the batch.  They run in any dtype (the GPU tests drive
them in float64 as the reference of the kernels).

Envs: `SpreadBoxEnv` has continuous simple_spread's shapes (3 agents, a Dict {"policy": Box(18), "critic": Box(54)}
observation, Box(5) actions) and agents that finish at different steps, so active masks have zeros.  The Box(256) /
Box(8) trace runs tests/wide_gaussian_oracle.py's wide_gaussian_env(256, 8).  `GRUGaussianTrainer` (oracle/loop_ma.
MATrainer with a Box head) is pinned to the unmodified reference by tests/test_gru_gaussian_oracle.py (traces
tests/golden/trace_gru_gaussian_{spread,box_256}.npz, recorded by tools/gen_golden_gru_gaussian.py)."""
import numpy as np
import torch

from oracle import envs as oenvs
from oracle import gae as ogae
from oracle import loop_ma, nets, ppo
from wide_gaussian_oracle import wide_gaussian_vec


def policy_act_gaussian(p, cfg, obs, rnn_states, masks, deterministic=False, normal_noise=None):
    """PolicyNetwork.forward_original with RNNLayer and a DiagGaussian head: (actions, per-dimension log-probs, states)."""
    feat, rnn_states = nets.policy_features(p, cfg, obs, rnn_states, masks)
    mean, std = nets.gaussian_params(p, feat)
    if deterministic:
        actions = mean
    elif normal_noise is None:
        actions = torch.normal(mean, std)
    else:
        actions = normal_noise * std + mean
    return actions, torch.distributions.Normal(mean, std).log_prob(actions), rnn_states


def policy_eval_gaussian(p, cfg, obs, actions, active_masks, rnn_states, masks):
    """PolicyNetwork.eval_actions with RNNLayer and a DiagGaussian head: per-dimension log-probs and the entropy mean over
    rows and dimensions (sum over rows and dimensions / sum(active) with use_policy_active_masks)."""
    feat, _ = nets.policy_features(p, cfg, obs, rnn_states, masks)
    mean, std = nets.gaussian_params(p, feat)
    dist = torch.distributions.Normal(mean, std)
    ent = dist.entropy()
    if active_masks is not None and cfg.use_policy_active_masks:
        ent = (ent * active_masks).sum() / active_masks.sum()
    else:
        ent = ent.mean()
    return dist.log_prob(actions), ent


def ppo_update(cfg, pol, cri, opt_p, opt_c, vn, batch, record=None, evaluate=policy_eval_gaussian, clip_keys=None):
    """One minibatch update of a GRU policy with a DiagGaussian head (oracle/ppo.ppo_update's sequence).  batch carries
    rnn_states / rnn_states_critic (the chunks' initial states) and masks as the recurrent generators give them.
    evaluate: the eval function (a test passes a mistaken one); clip_keys: the policy parameters the clip norm covers
    (None: all of them, as clip_grad_norm_ over the policy's parameters does)."""
    opt_p.zero_grad()
    opt_c.zero_grad()
    active = batch["active_masks"]
    values, _ = nets.critic_forward(cri, cfg, batch["critic_obs"], batch["rnn_states_critic"], batch["masks"])
    logp, ent = evaluate(pol, cfg, batch["policy_obs"], batch["actions"], active, batch["rnn_states"], batch["masks"])
    adv = batch["adv"]
    ratio = torch.exp(logp - batch["old_logp"])
    if getattr(cfg, "dual_clip_ppo", False):
        ratio = torch.min(ratio, torch.tensor(cfg.dual_clip_coeff, dtype=ratio.dtype))
    surr = torch.min(ratio * adv, torch.clamp(ratio, 1.0 - cfg.clip_param, 1.0 + cfg.clip_param) * adv)
    if cfg.use_policy_active_masks:
        policy_loss = (-torch.sum(surr, dim=-1, keepdim=True) * active).sum() / active.sum()
    else:
        policy_loss = -torch.sum(surr, dim=-1, keepdim=True).mean()
    value_loss = ppo.value_loss_fn(cfg, vn, values, batch["value_preds"], batch["returns"], active)
    (policy_loss - ent * cfg.entropy_coef).backward()
    (value_loss * cfg.value_loss_coef).backward()
    if record is not None:
        record.update(grads_policy={k: v.grad.detach().clone() for k, v in pol.items()},
                      grads_critic={k: v.grad.detach().clone() for k, v in cri.items()}, ratio=ratio.detach())
    clipped = [v for k, v in pol.items() if clip_keys is None or k in clip_keys]
    if cfg.use_max_grad_norm:
        agn = torch.nn.utils.clip_grad_norm_(clipped, cfg.max_grad_norm)
        cgn = torch.nn.utils.clip_grad_norm_(list(cri.values()), cfg.max_grad_norm)
    else:
        agn = torch.sqrt(sum(p.grad.norm() ** 2 for p in clipped))
        cgn = torch.sqrt(sum(p.grad.norm() ** 2 for p in cri.values()))
    opt_p.step()
    opt_c.step()
    return (value_loss.item(), float(cgn), policy_loss.item(), ent.item(), float(agn), ratio.mean().item())


# ---------------------------------------------------------------- envs ----------------------------------------------------

class SpreadBoxEnv:
    """Three agents; each sees 18 features in [0, 1) drawn every step, the critic sees all 54.  Box(5) actions, agent i
    rewarded by 1 - mean |target - clip(a, 0, 1)| with the target its first 5 features (float64).  Agent i is done from
    step 3 + i on (done agents keep acting, rewarded 0); the episode ends when all are (step 5).  4-tuple step with the
    agent axis: obs {"policy": (3, 18), "critic": (3, 54)}, rewards (3, 1), dones (3,)."""
    obs_dim, critic_obs_dim, act_dim, agent_num, HORIZON = 18, 54, 5, 3, 5

    def __init__(self):
        self.rng = oenvs.pcg64_np_random(None)
        self.steps = 0
        self._draw()

    def _draw(self):
        self.state = self.rng.random((self.agent_num, self.obs_dim)).astype(np.float32)

    def _obs(self):
        c = np.broadcast_to(self.state.reshape(1, -1), (self.agent_num, self.critic_obs_dim)).copy()
        return {"policy": self.state.copy(), "critic": c}

    def reset(self, seed=None, options=None):
        if seed is not None:
            self.rng = oenvs.pcg64_np_random(seed)
        self.steps = 0
        self._draw()
        return self._obs(), {}

    def step(self, action):
        a = np.asarray(action, dtype=np.float32).reshape(self.agent_num, -1)[:, :self.act_dim].astype(np.float64)
        done_before = np.arange(self.agent_num) + 3 <= self.steps
        target = self.state[:, :self.act_dim].astype(np.float64)
        reward = 1.0 - np.abs(target - np.clip(a, 0.0, 1.0)).mean(-1)
        reward[done_before] = 0.0
        self.steps += 1
        self._draw()
        dones = np.arange(self.agent_num) + 3 <= self.steps
        return self._obs(), reward[:, None], dones, {}


class SpacedSpreadBoxEnv(SpreadBoxEnv):
    """SpreadBoxEnv with the spaces a host vec-env reads (make(..., make_custom_envs=...))."""

    def __init__(self):
        from openrl_b200 import spaces

        super().__init__()
        box = lambda w: spaces.Box(-np.inf, np.inf, (w,), np.float32)  # noqa: E731
        self.observation_space = spaces.Dict({"policy": box(self.obs_dim), "critic": box(self.critic_obs_dim)})
        self.action_space = spaces.Box(-1.0, 1.0, (self.act_dim,), np.float32)


class SpreadBoxVec:
    """SpreadBoxEnv under SyncVectorEnv (seeds seed + i*10086, auto-reset when every agent is done): obs {"policy":
    (N,3,18), "critic": (N,3,54)}, rewards (N,3,1) f64, dones (N,3) bool."""
    obs_dim, critic_obs_dim, act_dim, agent_num = 18, 54, 5, 3
    n_actions = act_dim

    def __init__(self, env_num):
        self.N = env_num
        self.envs = [SpreadBoxEnv() for _ in range(env_num)]

    @staticmethod
    def _stack(obs):
        return {k: np.stack([o[k] for o in obs]) for k in ("policy", "critic")}

    def reset(self, seed=None):
        return self._stack([e.reset(seed=None if seed is None else seed + i * 10086)[0] for i, e in enumerate(self.envs)])

    def step(self, actions):
        obs, rewards, dones = [], np.zeros((self.N, 3, 1), np.float64), np.zeros((self.N, 3), bool)
        for i, e in enumerate(self.envs):
            o, r, d, _ = e.step(actions[i])
            if d.all():
                o, _ = e.reset()
            obs.append(o)
            rewards[i], dones[i] = r, d
        return self._stack(obs), rewards, dones, [{} for _ in range(self.N)]


def _box_vec(env_num):
    v = wide_gaussian_vec(256, 8)(env_num)
    v.n_actions = v.act_dim
    return v


VECS = {"gru_gaussian_spread": SpreadBoxVec, "gru_gaussian_box_256": _box_vec}


class GRUGaussianTrainer(loop_ma.MATrainer):
    """Recurrent PPO / MAPPO (oracle/loop_ma.MATrainer) with a DiagGaussian policy head on VECS[tag]."""

    def __init__(self, cfg, env_num, tag):
        saved = oenvs.ENVS.get("GRUGaussian")
        oenvs.ENVS["GRUGaussian"] = VECS[tag]
        try:
            super().__init__(cfg, "GRUGaussian", env_num)   # builds a Discrete head; replaced below, from the same seed
        finally:
            if saved is None:
                del oenvs.ENVS["GRUGaussian"]
            else:
                oenvs.ENVS["GRUGaussian"] = saved
        import random

        random.seed(cfg.seed)
        np.random.seed(cfg.seed)
        torch.manual_seed(cfg.seed)
        e = self.env
        d, n = e.obs_dim, e.act_dim
        dc = getattr(e, "critic_obs_dim", d)
        self.pol = nets.init_policy(cfg, d, "Box", n)
        self.cri = nets.init_critic(cfg, dc)
        self.opt_p, self.opt_c = ppo.make_optimizers(cfg, self.pol, self.cri)
        T, N, A = cfg.episode_length, env_num, self.A
        self.buf.actions = np.zeros((T, N, A, n), np.float32)
        self.buf.action_log_probs = np.zeros((T, N, A, n), np.float32)

    def rollout(self):
        cfg, b, N, A = self.cfg, self.buf, self.N, self.A
        for step in range(cfg.episode_length):
            with torch.no_grad():
                cat = lambda x: torch.from_numpy(np.concatenate(x))  # noqa: E731
                obs, cobs, masks = cat(b.policy_obs[step]), cat(b.critic_obs[step]), cat(b.masks[step])
                hs, hc = cat(b.rnn_states[step]), cat(b.rnn_states_critic[step])
                actions, logp, hs2 = policy_act_gaussian(self.pol, cfg, obs, hs, masks)
                values, hc2 = nets.critic_forward(self.cri, cfg, cobs, hc, masks)
            actions = actions.numpy().reshape(N, A, -1)
            obs2, rewards, dones, _ = self.env.step(actions)
            dones_env = np.all(dones, axis=1)
            hs2 = hs2.numpy().reshape(N, A, 1, -1).copy()
            hc2 = hc2.numpy().reshape(N, A, 1, -1).copy()
            hs2[dones_env] = 0.0
            hc2[dones_env] = 0.0
            b.rnn_states[step + 1], b.rnn_states_critic[step + 1] = hs2, hc2
            masks_n = np.ones((N, A, 1), np.float32)
            masks_n[dones_env] = 0.0
            active = np.ones((N, A, 1), np.float32)
            active[dones] = 0.0
            active[dones_env] = 1.0
            b.policy_obs[step + 1], b.critic_obs[step + 1] = loop_ma._obs_pair(obs2)
            b.actions[step] = actions
            b.action_log_probs[step] = logp.numpy().reshape(N, A, -1)
            b.value_preds[step] = values.numpy().reshape(N, A, 1)
            b.rewards[step] = rewards
            b.masks[step + 1] = masks_n
            b.active_masks[step + 1] = active

    def train(self):
        cfg, b = self.cfg, self.buf
        vn_state = self.vn.state() if self.vn is not None else None
        _, adv = ogae.advantages(b.returns, b.value_preds, b.active_masks, vn_state, cfg.use_adv_normalize)
        updates, perms = [], []
        for _ in range(cfg.ppo_epoch):
            gen = self._recurrent_batches(adv) if cfg.use_recurrent_policy else self._naive_batches(adv)
            for rand, bt in gen:
                batch = dict(bt, old_logp=bt["action_log_probs"])
                updates.append(ppo_update(cfg, self.pol, self.cri, self.opt_p, self.opt_c, self.vn, batch))
            perms.append(rand.copy())
        return np.array(updates, np.float64), np.stack(perms)
