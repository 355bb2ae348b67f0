"""Oracle for joint-action PPO (JRPO, `use_joint_action_loss`) on the recurrent MAPPO update.

TEST INFRASTRUCTURE: the torch-CPU restatement the CUDA path is compared against, pinned to the unmodified
reference by tests/test_jrpo_oracle.py (traces tests/golden/trace_mpe_jrpo*.npz, recorded by
tools/gen_golden_jrpo.py).  Extends oracle/loop_ma.MATrainer; follows, in the reference,
  ReplayData.recurrent_generator_v3   openrl/buffers/replay_data.py:425-551, _cast_v3 in buffers/utils/util.py:100-101
  PPOAlgorithm.prepare_loss (JRPO)    openrl/algorithms/ppo.py:222-224,254-300,306-319,340-360
  PPOAlgorithm.get_data_generator     openrl/algorithms/ppo.py:363-371

A sample of v3 is one (env, step) pair f = n*T + t carrying all A agents; a chunk is L consecutive samples (env
boundaries ignored); rows of a minibatch are ordered (step l, chunk, agent).  The policy is evaluated on every
agent row; the ratio is exp(sum_a logp - sum_a old_logp) per (step, chunk) group with agent 0's advantage and
active mask; the entropy stays per agent row with all agents' active masks; the critic sees agent 0's rows only.
"""
import numpy as np
import torch

from oracle import gae as ogae
from oracle import loop_ma, nets, ppo


def _cast_v3(x):
    """(T, N, A, ...) -> (N*T, A, ...), env-major / time-minor."""
    return x.transpose(1, 0, *range(2, x.ndim)).reshape(-1, *x.shape[2:])


def agent0(x, A):
    """to_single_np (ppo.py:222-224): rows ordered (group, agent) -> agent 0's row of every group."""
    return x.reshape(-1, A, *x.shape[1:])[:, 0]


def ppo_update_joint(cfg, pol, cri, opt_p, opt_c, vn, batch, A):
    """One JRPO minibatch update.  Returns (value_loss, critic_grad_norm, policy_loss, dist_entropy,
    actor_grad_norm, ratio_mean) like oracle.ppo.ppo_update."""
    opt_p.zero_grad()
    opt_c.zero_grad()
    active = batch["active_masks"]
    values, _ = nets.critic_forward(cri, cfg, agent0(batch["critic_obs"], A), agent0(batch["rnn_states_critic"], A),
                                    agent0(batch["masks"], A))
    # entropy from every agent row with every agent's active mask (evaluate_actions runs before the masks are reduced)
    logp, ent = nets.policy_eval(pol, cfg, batch["policy_obs"], batch["actions"], batch.get("action_masks"), active,
                                 batch["rnn_states"], batch["masks"])
    joint = logp.reshape(-1, A, logp.shape[-1]).sum(dim=(1, -1), keepdim=True).reshape(-1, 1)
    joint_old = batch["old_logp"].reshape(-1, A, 1).sum(dim=(1, -1), keepdim=True).reshape(-1, 1)
    adv = agent0(batch["adv"], A)
    act0 = agent0(active, A)
    ratio = torch.exp(joint - joint_old)
    if getattr(cfg, "dual_clip_ppo", False):
        ratio = torch.min(ratio, torch.tensor(cfg.dual_clip_coeff))
    surr = torch.min(ratio * adv, torch.clamp(ratio, 1.0 - cfg.clip_param, 1.0 + cfg.clip_param) * adv)
    if cfg.use_policy_active_masks:
        policy_loss = (-torch.sum(surr, dim=-1, keepdim=True) * act0).sum() / act0.sum()
    else:
        policy_loss = -torch.sum(surr, dim=-1, keepdim=True).mean()
    value_loss = ppo.value_loss_fn(cfg, vn, values, agent0(batch["value_preds"], A), agent0(batch["returns"], A), act0)
    (policy_loss - ent * cfg.entropy_coef).backward()
    (value_loss * cfg.value_loss_coef).backward()
    if cfg.use_max_grad_norm:
        agn = torch.nn.utils.clip_grad_norm_(list(pol.values()), cfg.max_grad_norm)
        cgn = torch.nn.utils.clip_grad_norm_(list(cri.values()), cfg.max_grad_norm)
    else:
        agn = torch.sqrt(sum(p.grad.norm() ** 2 for p in pol.values()))
        cgn = torch.sqrt(sum(p.grad.norm() ** 2 for p in cri.values()))
    opt_p.step()
    opt_c.step()
    return (value_loss.item(), float(cgn), policy_loss.item(), ent.item(), float(agn), ratio.mean().item())


class JointTrainer(loop_ma.MATrainer):
    """MATrainer whose update is JRPO: recurrent_generator_v3 batches and the joint-ratio loss."""

    def __init__(self, cfg, env_id, env_num):
        if not cfg.use_recurrent_policy:
            raise ValueError("JRPO is defined on the chunked recurrent generator (use_recurrent_policy)")
        super().__init__(cfg, env_id, env_num)

    def _v3_batches(self, adv):
        """recurrent_generator_v3 (replay_data.py:425-551)."""
        cfg, b = self.cfg, self.buf
        T, N, A = b.rewards.shape[:3]
        L = cfg.data_chunk_length
        data_chunks = N * T // L
        mb = data_chunks // cfg.num_mini_batch
        rand = torch.randperm(data_chunks).numpy()
        flat = {k: _cast_v3(getattr(b, k)[:T]) for k in ("policy_obs", "critic_obs", "actions", "action_log_probs", "value_preds",
                                                          "returns", "masks", "active_masks", "action_masks")}
        flat["adv"] = _cast_v3(adv)
        hs, hc = _cast_v3(b.rnn_states[:-1]), _cast_v3(b.rnn_states_critic[:-1])   # (N*T, A, 1, H)
        for i in range(cfg.num_mini_batch):
            idx = rand[i * mb:(i + 1) * mb]
            out = {}
            for k, v in flat.items():
                st = np.stack([v[c * L:c * L + L] for c in idx], axis=1)   # (L, n, A, d)
                out[k] = torch.from_numpy(np.ascontiguousarray(st).reshape(L * len(idx) * A, *st.shape[3:]))
            out["rnn_states"] = torch.from_numpy(np.stack([hs[c * L] for c in idx]).reshape(len(idx) * A, *hs.shape[2:]))
            out["rnn_states_critic"] = torch.from_numpy(np.stack([hc[c * L] for c in idx]).reshape(len(idx) * A, *hc.shape[2:]))
            yield rand, out

    def train(self):
        cfg, b = self.cfg, self.buf
        vn_state = self.vn.state() if self.vn is not None else None
        _, adv = ogae.advantages(b.returns, b.value_preds, b.active_masks, vn_state, cfg.use_adv_normalize)
        self.last_adv = adv
        updates, perms = [], []
        for _ in range(cfg.ppo_epoch):
            for rand, bt in self._v3_batches(adv):
                batch = dict(critic_obs=bt["critic_obs"], policy_obs=bt["policy_obs"], actions=bt["actions"],
                             value_preds=bt["value_preds"], returns=bt["returns"], active_masks=bt["active_masks"],
                             old_logp=bt["action_log_probs"], adv=bt["adv"], action_masks=bt["action_masks"],
                             masks=bt["masks"], rnn_states=bt["rnn_states"], rnn_states_critic=bt["rnn_states_critic"])
                updates.append(ppo_update_joint(cfg, self.pol, self.cri, self.opt_p, self.opt_c, self.vn, batch, self.A))
            perms.append(rand.copy())
        return np.array(updates, np.float64), np.stack(perms)
