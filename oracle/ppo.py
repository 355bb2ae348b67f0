"""Oracle: the PPO minibatch update (loss, backward, clip, Adam) on torch-CPU.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Follows
  PPOAlgorithm.ppo_update / prepare_loss / cal_value_loss   openrl/algorithms/ppo.py:46-361
  ValueNorm.update / normalize                               openrl/modules/utils/valuenorm.py:59-90
  huber_loss / mse_loss                                      openrl/modules/utils/util.py:19-27
  Adam(lr, eps=opti_eps, weight_decay)                       openrl/modules/rl_module.py:80-87
"""
import numpy as np
import torch

from . import nets


class ValueNormState:
    """ValueNorm with norm_axes=1, beta=0.99999 (valuenorm.py:6-106) as three scalars: float32 like the reference, or
    float64 (`dtype`) for a high-precision reference of the update; `device` is where the returns it sees live."""

    def __init__(self, state=None, beta=0.99999, dtype=torch.float32, device=None):
        self.beta = beta
        s = [0.0, 0.0, 0.0] if state is None else [float(x) for x in state]
        self.running_mean = torch.tensor([s[0]], dtype=dtype, device=device)
        self.running_mean_sq = torch.tensor([s[1]], dtype=dtype, device=device)
        self.debiasing_term = torch.tensor(s[2], dtype=dtype, device=device)

    def state(self):
        dt = np.float64 if self.running_mean.dtype == torch.float64 else np.float32
        return np.array([self.running_mean.item(), self.running_mean_sq.item(), self.debiasing_term.item()], dt)

    def mean_var(self):
        m = self.running_mean / self.debiasing_term.clamp(min=1e-5)
        msq = self.running_mean_sq / self.debiasing_term.clamp(min=1e-5)
        return m, (msq - m ** 2).clamp(min=1e-2)

    @torch.no_grad()
    def update(self, x):
        w = self.beta
        self.running_mean.mul_(w).add_(x.mean(dim=0) * (1.0 - w))
        self.running_mean_sq.mul_(w).add_((x ** 2).mean(dim=0) * (1.0 - w))
        self.debiasing_term.mul_(w).add_(1.0 * (1.0 - w))

    def normalize(self, x):
        m, v = self.mean_var()
        return (x - m[None]) / torch.sqrt(v)[None]

    def denormalize(self, x):
        m, v = self.mean_var()
        return x * torch.sqrt(v)[None] + m[None]


def huber_loss(e, d):
    a = (abs(e) <= d).float()
    b = (abs(e) > d).float()
    return a * e ** 2 / 2 + b * d * (abs(e) - d / 2)


def make_optimizers(cfg, policy_params, critic_params):
    if policy_params is critic_params:   # cfg.use_share_model: ONE Adam over the shared model, lr = cfg.lr (ppo_module.py:60-69)
        for v in policy_params.values():
            v.requires_grad_(True)
        opt = torch.optim.Adam(list(policy_params.values()), lr=cfg.lr, eps=cfg.opti_eps, weight_decay=cfg.weight_decay)
        return opt, opt
    for v in list(policy_params.values()) + list(critic_params.values()):
        v.requires_grad_(True)
    opt_p = torch.optim.Adam(list(policy_params.values()), lr=cfg.lr, eps=cfg.opti_eps, weight_decay=cfg.weight_decay)
    opt_c = torch.optim.Adam(list(critic_params.values()), lr=cfg.critic_lr, eps=cfg.opti_eps,
                             weight_decay=cfg.weight_decay)
    return opt_p, opt_c


def value_loss_fn(cfg, vn, values, value_preds, returns, active):
    """cal_value_loss (ppo.py:178-220).  vn=None: no normaliser."""
    clipped = value_preds + (values - value_preds).clamp(-cfg.clip_param, cfg.clip_param)
    if vn is not None:
        vn.update(returns)
        target = vn.normalize(returns)
    else:
        target = returns
    e_c, e_o = target - clipped, target - values
    if cfg.use_huber_loss:
        l_c, l_o = huber_loss(e_c, cfg.huber_delta), huber_loss(e_o, cfg.huber_delta)
    else:
        l_c, l_o = e_c ** 2 / 2, e_o ** 2 / 2
    loss = torch.max(l_o, l_c) if cfg.use_clipped_value_loss else l_o
    if cfg.use_value_active_masks:
        return (loss * active).sum() / active.sum()
    return loss.mean()


def ppo_update(cfg, pol, cri, opt_p, opt_c, vn, batch, record=None):
    """One minibatch update.  batch: dict of torch tensors (critic_obs, policy_obs, actions,
    value_preds, returns, masks, active_masks, old_logp, adv, action_masks[, rnn...]).
    Returns (value_loss, critic_grad_norm, policy_loss, dist_entropy, actor_grad_norm, ratio_mean).
    record: a dict that receives what a kernel's intermediate results are compared with: `grads_policy` /
    `grads_critic` ({name: gradient before the clip}), the detached `surr` and `ratio` tensors and the losses."""
    opt_p.zero_grad()
    opt_c.zero_grad()
    active = batch["active_masks"]
    values, _ = nets.critic_forward(cri, cfg, batch["critic_obs"], batch.get("rnn_states_critic"), batch.get("masks"))
    if "act.action_out.fc_mean.weight" in pol:  # Box action space
        logp, ent = nets.policy_eval_gaussian(pol, cfg, batch["policy_obs"], batch["actions"], active)
    else:
        logp, ent = nets.policy_eval(pol, cfg, batch["policy_obs"], batch["actions"], batch.get("action_masks"),
                                     active, batch.get("rnn_states"), batch.get("masks"))
    adv = batch["adv"]
    if getattr(cfg, "a2c", False):          # A2CAlgorithm.prepare_loss (a2c.py:88): -adv * logp, ratio reported 0
        ratio = torch.zeros(1)
        surr = adv.detach() * logp
    else:
        ratio = torch.exp(logp - batch["old_logp"])
        if getattr(cfg, "dual_clip_ppo", False):   # ppo.py:304-305
            ratio = torch.min(ratio, torch.tensor(cfg.dual_clip_coeff))
        surr1 = ratio * adv
        surr2 = torch.clamp(ratio, 1.0 - cfg.clip_param, 1.0 + cfg.clip_param) * adv
        surr = torch.min(surr1, surr2)
    if cfg.use_policy_active_masks:
        policy_loss = (-torch.sum(surr, dim=-1, keepdim=True) * active).sum() / active.sum()
    else:
        policy_loss = -torch.sum(surr, dim=-1, keepdim=True).mean()
    value_loss = value_loss_fn(cfg, vn, values, batch["value_preds"], batch["returns"], active)
    # construct_loss_list + `for loss in loss_list: loss.backward()` (ppo.py:226-236,117-118); with a shared model both
    # losses accumulate into the same .grad, both clip_grad_norm_ calls see ALL parameters (base_value_policy_network.py:
    # 58-62: the second one acts on the already clipped gradients) and the single optimiser steps once
    (policy_loss - ent * cfg.entropy_coef).backward(retain_graph=pol is cri)
    (value_loss * cfg.value_loss_coef).backward()
    if record is not None:
        record.update(grads_policy={k: v.grad.detach().clone() for k, v in pol.items()},
                      grads_critic={k: v.grad.detach().clone() for k, v in cri.items()}, surr=surr.detach(),
                      ratio=ratio.detach(), policy_loss=policy_loss.detach(), entropy=ent.detach(), value_loss=value_loss.detach())
    if cfg.use_max_grad_norm:
        agn = torch.nn.utils.clip_grad_norm_(list(pol.values()), cfg.max_grad_norm)
        cgn = torch.nn.utils.clip_grad_norm_(list(cri.values()), cfg.max_grad_norm)
    else:
        agn = torch.sqrt(sum(p.grad.norm() ** 2 for p in pol.values()))
        cgn = torch.sqrt(sum(p.grad.norm() ** 2 for p in cri.values()))
    opt_p.step()
    if opt_c is not opt_p:
        opt_c.step()
    return (value_loss.item(), float(cgn), policy_loss.item(), ent.item(), float(agn), ratio.mean().item())
