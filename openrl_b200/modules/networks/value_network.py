"""ValueNetwork (reference: openrl/modules/networks/value_network.py:33): base -> v_out,
with the `value_normalizer` attribute the algorithm looks up (ppo_module.py:212-216)."""
import torch
import torch.nn as nn

from .base import FlatParams, MLPBase, PopArt, RNNLayer, ValueNorm, _init, check_obs_shape


def _critic_shape(space):
    return space["critic"].shape if space.__class__.__name__ == "Dict" else space.shape


class ValueNetwork(nn.Module):
    def __init__(self, cfg, input_space, action_space=None, use_half=False, device=torch.device("cpu"), extra_args=None):
        super().__init__()
        self.recurrent = bool(cfg.use_recurrent_policy or cfg.use_naive_recurrent_policy)
        shape = _critic_shape(input_space)
        check_obs_shape(shape, wide=getattr(cfg, "use_wide_observations", False) and not self.recurrent)
        self.obs_dim = shape[0]
        self.activation_id = cfg.activation_id
        self.base = MLPBase(cfg, shape)
        if self.recurrent:
            self.rnn = RNNLayer(self.base.output_size, self.base.output_size, cfg.recurrent_N, cfg.use_orthogonal, cfg.rnn_type)
        head = PopArt(self.base.output_size, 1) if cfg.use_popart else nn.Linear(self.base.output_size, 1)
        self.v_out = _init(head, 1.0, cfg.use_orthogonal)
        self.device = torch.device(device)
        self._flat = FlatParams(self, self.device)
        # registered after flattening: its state is a buffer, not an optimised parameter
        self.value_normalizer = ValueNorm(1, device=self.device) if cfg.use_valuenorm else None

    @property
    def flat_params(self):
        return self._flat.flat
