"""PPOModule: bundle of models {"policy","critic"} + optimizers with the reference's method
surface (openrl/modules/ppo_module.py:32-224, rl_module.py:29-190).

Numeric methods launch CUDA through the C-ABI; optimizers are `FusedAdamState` objects whose
moments the `orl_ppo_apply` kernel updates (torch.optim.Adam semantics, rl_module.py:80-87)."""
import numpy as np
import torch

from .. import lib
from .networks import PolicyNetwork, PolicyValueNetwork, ValueNetwork


class FusedAdamState:
    """State of one Adam optimiser living in flat CUDA buffers (exp_avg, exp_avg_sq, step)."""

    def __init__(self, flat_params, lr, eps, weight_decay, betas=(0.9, 0.999)):
        self.param_groups = [dict(lr=lr, eps=eps, weight_decay=weight_decay, betas=betas)]
        self.exp_avg = torch.zeros_like(flat_params)
        self.exp_avg_sq = torch.zeros_like(flat_params)

    def zero_grad(self):
        pass

    def state_dict(self):
        return dict(param_groups=self.param_groups, exp_avg=self.exp_avg.clone(), exp_avg_sq=self.exp_avg_sq.clone())

    def load_state_dict(self, sd):
        self.param_groups = sd["param_groups"]
        self.exp_avg.copy_(sd["exp_avg"])
        self.exp_avg_sq.copy_(sd["exp_avg_sq"])


class _Roles(dict):
    """{"model": shared net} that also answers the "policy" / "critic" roles with the shared object, so code written
    against the two-net layout (models["policy"], optimizers["critic"], ...) reads the right parameters; iteration,
    `in`, and checkpoints see only the real key, like the reference's dicts (ppo_module.py:60-69)."""

    def __missing__(self, key):
        if key in ("policy", "critic") and "model" in self:
            return self["model"]
        raise KeyError(key)


class PPOModule:
    def __init__(self, cfg, policy_input_space, critic_input_space, act_space, share_model=False, device="cuda:0",
                 rank=0, world_size=1, model_dict=None):
        self.cfg = cfg
        self.device = torch.device(device)
        self.lr, self.critic_lr = cfg.lr, cfg.critic_lr
        self.opti_eps, self.weight_decay = cfg.opti_eps, cfg.weight_decay
        self.act_space = act_space
        self.rank, self.world_size = rank, world_size
        self.share_model = bool(share_model)
        self.models, self.optimizers = _Roles(), _Roles()
        self.adam_steps = torch.zeros(2, dtype=torch.int32, device=self.device)
        self._act_calls = 0   # Philox step of the next stochastic act() call
        self._lib = lib.load()
        if self.share_model:   # ppo_module.py:60-69: one PolicyValueNetwork, one Adam with lr = cfg.lr
            cls = (model_dict or {}).get("model", PolicyValueNetwork)
            self.models["model"] = cls(cfg=cfg, input_space=policy_input_space, action_space=act_space, device=self.device,
                                       use_half=False, extra_args=None)
            self.optimizers["model"] = FusedAdamState(self.models["model"].flat_params, cfg.lr, cfg.opti_eps, cfg.weight_decay)
            return
        # dict order as in the reference: policy first, then critic (ppo_module.py:71-88)
        pol_cls = (model_dict or {}).get("policy", PolicyNetwork)
        cri_cls = (model_dict or {}).get("critic", ValueNetwork)
        self.models["policy"] = pol_cls(cfg=cfg, input_space=policy_input_space, action_space=act_space,
                                        device=self.device, use_half=False, extra_args=None)
        self.optimizers["policy"] = FusedAdamState(self.models["policy"].flat_params, cfg.lr, cfg.opti_eps, cfg.weight_decay)
        self.models["critic"] = cri_cls(cfg=cfg, input_space=critic_input_space, action_space=act_space,
                                        device=self.device, use_half=False, extra_args=None)
        self.optimizers["critic"] = FusedAdamState(self.models["critic"].flat_params, cfg.critic_lr, cfg.opti_eps,
                                                   cfg.weight_decay)

    # `torch.save(module)` / `torch.load` (the reference's checkpoint format, rl_agent.py:187-213): everything is
    # picklable except the ctypes library handle
    def __getstate__(self):
        st = dict(self.__dict__)
        st.pop("_lib", None)
        return st

    def __setstate__(self, st):
        self.__dict__.update(st)
        self._lib = lib.load()

    # -- reference surface -----------------------------------------------------------------
    def lr_decay(self, episode, episodes):
        """update_linear_schedule (openrl/modules/utils/util.py:13-17)."""
        for key, base in ((("model", self.lr),) if self.share_model else (("policy", self.lr), ("critic", self.critic_lr))):
            lr = base - (base * (episode / float(episodes)))
            for g in self.optimizers[key].param_groups:
                g["lr"] = lr

    def get_critic_value_normalizer(self):
        return self.models["critic"].value_normalizer

    def get_values(self, critic_obs, rnn_states_critic=None, masks=None):
        """ValueNetwork.forward on a (rows, d_c) batch -> (rows, 1) CUDA tensor."""
        obs = torch.as_tensor(critic_obs, dtype=torch.float32).to(self.device).contiguous()
        rows = obs.shape[0]
        out = torch.empty(rows, 1, dtype=torch.float32, device=self.device)
        cri = self.models["critic"]
        if self.share_model:
            lib.check(self._lib.orl_share_values(lib.ptr(cri.flat_params), cri.obs_dim, cri.n_actions, cri.activation_id, lib.ptr(obs),
                                                 lib.ptr(out), rows, lib.current_stream()), "orl_share_values")
            return out
        lib.check(self._lib.orl_critic_values(lib.ptr(cri.flat_params), cri.obs_dim, cri.activation_id, lib.ptr(obs),
                                              lib.ptr(out), rows, lib.current_stream()), "orl_critic_values")
        return out

    def get_actions(self, critic_obs, obs, rnn_states_actor=None, rnn_states_critic=None, masks=None, action_masks=None,
                    deterministic=False):
        """ppo_module.py:102-138: (values, actions, action_log_probs, rnn_states_actor, rnn_states_critic) for a batch of
        rows — the policy "original" forward plus the critic forward (feed-forward nets: rnn states pass through)."""
        if getattr(self.models["policy"], "recurrent", False):
            raise NotImplementedError("get_actions for recurrent nets: the recurrent critic runs inside OnPolicyDriver (orl_rnn_critic)")
        actions, logp = self.act(obs, rnn_states_actor, masks, action_masks, deterministic)
        values = self.get_values(critic_obs, rnn_states_critic, masks)
        return values, actions, logp, rnn_states_actor, rnn_states_critic

    def evaluate_actions(self, critic_obs, obs, rnn_states_actor, rnn_states_critic, action, masks, action_masks=None,
                         active_masks=None, critic_masks_batch=None):
        """ppo_module.py:147-193: (values, action_log_probs, dist_entropy, policy_values=None) of given actions; the entropy
        is the active-mask mean when cfg.use_policy_active_masks (act.py:160-168), else the plain mean."""
        pol = self.models["policy"]
        if getattr(pol, "recurrent", False) or self.share_model:
            raise NotImplementedError("evaluate_actions for recurrent / shared nets runs inside the fused update kernels")
        o = torch.as_tensor(obs, dtype=torch.float32).to(self.device).contiguous().view(-1, pol.obs_dim)
        rows = o.shape[0]
        gauss = lib.is_gaussian(pol.head_kind)
        w = pol.n_actions if gauss else 1
        act = torch.as_tensor(action, dtype=torch.float32).to(self.device).contiguous().view(rows, w)
        am = None if (action_masks is None or gauss) else torch.as_tensor(action_masks, dtype=torch.float32).to(self.device).contiguous()
        logp = torch.empty(rows, w, dtype=torch.float32, device=self.device)
        ent = torch.empty(rows, w, dtype=torch.float32, device=self.device)
        lib.check(self._lib.orl_policy_eval(lib.ptr(pol.flat_params), pol.obs_dim, pol.n_actions, pol.activation_id, pol.head_kind,
                                            lib.ptr(o), lib.ptr(act), lib.ptr(am), lib.ptr(logp), lib.ptr(ent), rows,
                                            lib.current_stream()), "orl_policy_eval")
        if active_masks is not None and getattr(self.cfg, "use_policy_active_masks", True):
            m = torch.as_tensor(active_masks, dtype=torch.float32).to(self.device).view(rows, 1)
            dist_entropy = (ent * m).sum() / m.sum() if not gauss else (ent * m).sum() / m.sum()
        else:
            dist_entropy = ent.mean()
        values = self.get_values(critic_obs, rnn_states_critic, critic_masks_batch if critic_masks_batch is not None else masks)
        return values, logp, dist_entropy, None

    def act(self, obs, rnn_states_actor=None, masks=None, action_masks=None, deterministic=False, exp_noise=None,
            rng_seed=None, rng_step=None):
        """PolicyNetwork.forward_original on a (rows, d) batch (ppo_module.py:195-210):
        returns (actions (rows,1) float CUDA tensor, log-probs (rows,1)) and, for a GRU policy, the new rnn states
        (rows, 1, H).  action_masks (rows, n) or None.
        Stochastic calls draw Philox noise keyed by (cfg.seed, call counter, row): every call sees fresh noise
        (the reference samples from torch's advancing global generator)."""
        pol = self.models["policy"]
        if rng_seed is None:
            rng_seed = (int(getattr(self.cfg, "seed", 0)) + 0x51ED270B) & 0xFFFFFFFFFFFF
        if rng_step is None:
            rng_step = self._act_calls
            self._act_calls += 1
        dev = lambda x: None if x is None else torch.as_tensor(x, dtype=torch.float32).to(self.device).contiguous()  # noqa: E731
        obs = dev(obs).view(-1, pol.obs_dim)
        rows = obs.shape[0]
        act_w = pol.n_actions if lib.is_gaussian(pol.head_kind) else 1
        actions = torch.empty(rows, act_w, dtype=torch.float32, device=self.device)
        logp = torch.empty(rows, act_w, dtype=torch.float32, device=self.device)
        if not getattr(pol, "recurrent", False):
            self.act_rows(obs, actions, logp, 0, rows, rng_seed, rng_step, action_masks=dev(action_masks), noise=dev(exp_noise),
                          deterministic=deterministic)
            return actions, logp
        # one GRU step (policy_network.py:130-162 with RNNLayer) on a one-slot buffer: the new states land in slot 1
        H = pol.hidden_size
        states = torch.zeros(2, rows, H, dtype=torch.float32, device=self.device)
        if rnn_states_actor is not None:
            states[0].copy_(dev(rnn_states_actor).reshape(rows, H))
        mk = torch.ones(rows, dtype=torch.float32, device=self.device)
        if masks is not None:
            mk.copy_(dev(masks).reshape(rows))
        self.act_rows(obs, actions, logp, 0, rows, rng_seed, rng_step, action_masks=dev(action_masks), noise=dev(exp_noise),
                      masks=mk, rnn_states=states, deterministic=deterministic)
        return actions, logp, states[1].view(rows, 1, H)

    def act_rows(self, obs, actions, log_probs, r0, r1, rng_seed, rng_step, rng_row_offset=0, action_masks=None, noise=None,
                 masks=None, rnn_states=None, deterministic=False):
        """The policy act on rows [r0, r1) of one slot, with no env step: orl_rollout / orl_share_rollout with
        ORL_ENV_NONE, or orl_rnn_act_rows for a GRU policy.  obs (B, d), actions and log_probs (B, w), action_masks and
        the noise table (B, n) or None are the slot's rows; a GRU policy also reads masks (B,) and rnn_states (2, B, H),
        this slot's states and the next slot's, which it writes.  The noise of row r is keyed by
        (rng_seed, rng_step, r + rng_row_offset)."""
        pol = self.models["policy"]
        recurrent = getattr(pol, "recurrent", False)
        if not recurrent:   # the feed-forward act runs over every row it is handed
            obs, actions, log_probs = obs[r0:r1], actions[r0:r1], log_probs[r0:r1]
            action_masks = None if action_masks is None else action_masks[r0:r1]
            noise = None if noise is None else noise[r0:r1]
            rng_row_offset += r0
        a = lib.OrlRnnArgs() if recurrent else lib.OrlRolloutArgs()
        a.env_kind, a.n_envs, a.n_agents, a.episode_length, a.t_begin, a.t_end = lib.ENV_NONE, obs.shape[0], 1, 1, 0, 1
        a.obs_dim, a.n_actions = pol.obs_dim, pol.n_actions
        a.activation_id, a.deterministic = pol.activation_id, int(bool(deterministic))
        a.policy_params, a.policy_obs = lib.ptr(pol.flat_params), lib.ptr(obs)
        a.actions, a.action_log_probs = lib.ptr(actions), lib.ptr(log_probs)
        a.action_masks, a.exp_noise = lib.ptr(action_masks), lib.ptr(noise)
        a.rng_seed, a.rng_step_base, a.rng_counter, a.rng_row_offset = int(rng_seed), int(rng_step), None, int(rng_row_offset)
        s = lib.current_stream()
        if recurrent:   # reads the noise table by buffer row
            a.critic_obs_dim, a.row_begin, a.row_end = pol.obs_dim, r0, r1
            a.rnn_states, a.masks = lib.ptr(rnn_states), lib.ptr(masks)
            lib.check(self._lib.orl_rnn_act_rows(a, s), "orl_rnn_act_rows")
        else:
            a.head_kind = pol.head_kind
            act_fn = self._lib.orl_share_rollout if self.share_model else self._lib.orl_rollout
            lib.check(act_fn(a, s), "orl_rollout(act)")

    @staticmethod
    def init_rnn_states(rollout_num, agent_num, rnn_layers, hidden_size):
        masks = np.ones((rollout_num * agent_num, 1), dtype=np.float32)
        rnn_state = np.zeros((rollout_num * agent_num, rnn_layers, hidden_size))
        return rnn_state, masks

    def load_policy(self, model_path):
        sd = torch.load(str(model_path), map_location=self.device)
        self.models["policy"].load_state_dict(sd)
