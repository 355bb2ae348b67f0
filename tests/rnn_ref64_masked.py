"""tests/rnn_ref64.py driven with legal-move action masks: the same float64 / float32 reference of one recurrent update
minibatch, with the policy evaluated on masked logits (categorical_logits: -6e4 where the mask is 0, distributions.py:71).

TEST INFRASTRUCTURE.  rnn_ref64 evaluates the policy through `oracle.nets.policy_eval` with no masks; `update` here runs
rnn_ref64.update with that one call given the mask rows of the minibatch (gathered by rnn_ref64.gather, the rows the
policy evaluation itself gathers), so every other line of the reference is the pinned one."""
import types

import torch

import rnn_ref64
from oracle import nets


def update(cfg, buf, state, ids, L, dims, action_masks, dtype=torch.float64):
    """rnn_ref64.update (ordinary chunks) with action_masks (T+1, N, A, n) or (T+1, B, n) applied to the policy."""
    T = buf["actions"].shape[0]
    B = rnn_ref64.rows(buf["actions"]).shape[0] // T
    rp, _ = rnn_ref64.gather(T, B, 1, L, ids, False)
    am = rnn_ref64.rows(action_masks)[rp.reshape(-1)]

    def policy_eval(p, ncfg, obs, actions, masks_arg, *a, **k):
        assert masks_arg is None and obs.shape[0] == am.shape[0]
        return nets.policy_eval(p, ncfg, obs, actions, am.to(device=obs.device, dtype=obs.dtype), *a, **k)

    masked = types.SimpleNamespace(**{k: getattr(nets, k) for k in dir(nets) if not k.startswith("__")})
    masked.policy_eval = policy_eval
    saved = rnn_ref64.nets
    rnn_ref64.nets = masked
    try:
        return rnn_ref64.update(cfg, buf, state, ids, L, dims, joint=False, dtype=dtype)
    finally:
        rnn_ref64.nets = saved
