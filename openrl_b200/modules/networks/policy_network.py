"""PolicyNetwork (reference: openrl/modules/networks/policy_network.py:33): base -> act."""
import torch
import torch.nn as nn

from .base import ACTLayer, FlatParams, MLPBase, RNNLayer, check_obs_shape, recurrent_obs_check


def _policy_shape(space):
    return space["policy"].shape if space.__class__.__name__ == "Dict" else space.shape


class PolicyNetwork(nn.Module):
    def __init__(self, cfg, input_space, action_space, device=torch.device("cpu"), use_half=False, extra_args=None):
        super().__init__()
        # `_use_naive_recurrent_policy or _use_recurrent_policy` (policy_network.py:88-97): same RNNLayer either way
        self.recurrent = bool(cfg.use_recurrent_policy or cfg.use_naive_recurrent_policy)
        self.hidden_size = cfg.hidden_size
        shape = _policy_shape(input_space)
        check_obs_shape(shape, **recurrent_obs_check(cfg, self.recurrent))
        self.obs_dim = shape[0]
        self.activation_id = cfg.activation_id
        self.base = MLPBase(cfg, shape)
        if self.recurrent:   # module order base -> rnn -> act as in the reference (state_dict / flat layout)
            self.rnn = RNNLayer(self.base.output_size, self.base.output_size, cfg.recurrent_N, cfg.use_orthogonal, cfg.rnn_type)
        self.act = ACTLayer(action_space, self.base.output_size, cfg.use_orthogonal, cfg.gain)
        self.head_kind = 1 if self.act.continuous_action else 0          # lib.HEAD_GAUSSIAN / HEAD_CATEGORICAL
        self.n_actions = action_space.shape[0] if self.act.continuous_action else action_space.n  # head width
        # a GRU policy's DiagGaussian head (cfg.use_recurrent_gaussian_head): the 8-row head block of the GRU kernels
        recurrent_gaussian = self.recurrent and self.act.continuous_action
        if recurrent_gaussian and not getattr(cfg, "use_recurrent_gaussian_head", False):
            raise NotImplementedError("recurrent policies are built for Discrete action spaces")
        if recurrent_gaussian and self.n_actions > 8:
            raise NotImplementedError("recurrent policies with DiagGaussian heads are built for Box action spaces of width "
                                      "up to 8 (use_recurrent_gaussian_head)")
        # a feed-forward Categorical head runs up to 64 actions (a logits tile in the kernels); a GRU policy's head runs up
        # to 64 with cfg.use_wide_recurrent_head (a lane-owned 64-vector in the GRU kernels) and up to 8 without; the
        # DiagGaussian heads keep the per-thread head of up to 8 outputs, and run up to 64 with cfg.use_wide_gaussian_head
        # (the 64-wide head tile, lib.HEAD_GAUSSIAN_WIDE, for widths above 8)
        wide_gaussian = self.act.continuous_action and bool(getattr(cfg, "use_wide_gaussian_head", False))
        if wide_gaussian and self.n_actions > 64:
            raise NotImplementedError("DiagGaussian heads are built for Box action spaces of width up to 64 "
                                      "(use_wide_gaussian_head)")
        if self.n_actions > 64:
            raise NotImplementedError("Discrete action spaces of up to 64 actions are built")
        if self.n_actions > 8 and self.recurrent and not getattr(cfg, "use_wide_recurrent_head", False):
            raise NotImplementedError("recurrent policies are built for up to 8 actions (9..64 with use_wide_recurrent_head)")
        if self.n_actions > 8 and self.act.continuous_action and not wide_gaussian:
            raise NotImplementedError("DiagGaussian heads are built for Box action spaces of width up to 8")
        if self.n_actions > 8 and wide_gaussian:
            self.head_kind = 2                                           # lib.HEAD_GAUSSIAN_WIDE
        self.device = torch.device(device)
        self._flat = FlatParams(self, self.device)

    @property
    def flat_params(self):
        return self._flat.flat
