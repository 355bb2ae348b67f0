"""PolicyValueNetwork for cfg.use_share_model (reference: openrl/modules/networks/policy_value_network.py:33-174):
obs_prep (MLPBase) -> common (MLPLayer(H, H, layer_N=0)) -> {v_out, act}, `critic_obs_prep` aliasing `obs_prep`.
Parameter tree / state_dict names and the initialisation sequence are the reference's; the numeric path is
csrc/orl_share.cu (flat layout = named_parameters order, see orl_deep_core.h).  Discrete action spaces take a
Categorical head, Box spaces of width <= 8 a DiagGaussian head (fc_mean + logstd, as in PolicyNetwork)."""
import torch
import torch.nn as nn

from .base import ACT_NAMES, ACTLayer, FlatParams, MLPBase, ValueNorm, _init, check_obs_shape
from .policy_network import _policy_shape


class CommonLayer(nn.Module):
    """MLPLayer(input, hidden, layer_N=0) (mlp.py:8-46): fc1 = Linear + act + LayerNorm, fc3 = Linear + LayerNorm."""

    def __init__(self, input_dim, hidden_size, use_orthogonal, activation_id):
        super().__init__()
        act = [nn.Tanh(), nn.ReLU(), nn.LeakyReLU(), nn.ELU()][activation_id]
        gain = nn.init.calculate_gain(ACT_NAMES[activation_id])
        self.fc1 = nn.Sequential(_init(nn.Linear(input_dim, hidden_size), gain, use_orthogonal), act, nn.LayerNorm(hidden_size))
        self.fc3 = nn.Sequential(_init(nn.Linear(hidden_size, hidden_size), gain, use_orthogonal), nn.LayerNorm(hidden_size))


class PolicyValueNetwork(nn.Module):
    def __init__(self, cfg, input_space, action_space, device=torch.device("cpu"), use_half=False, extra_args=None):
        super().__init__()
        for name in ("use_recurrent_policy", "use_naive_recurrent_policy", "use_popart"):
            if getattr(cfg, name, False):
                raise NotImplementedError(f"cfg.{name} with use_share_model is not built (feed-forward shared net, ValueNorm)")
        self.recurrent = False
        self.hidden_size = cfg.hidden_size
        shape = _policy_shape(input_space)
        check_obs_shape(shape)
        self.obs_dim = shape[0]
        self.activation_id = cfg.activation_id
        self.obs_prep = MLPBase(cfg, shape)
        self.critic_obs_prep = self.obs_prep                       # policy_value_network.py:75 (same module object)
        self.common = CommonLayer(cfg.hidden_size, cfg.hidden_size, cfg.use_orthogonal, cfg.activation_id)
        self.v_out = _init(nn.Linear(cfg.hidden_size, 1), 1.0, cfg.use_orthogonal)
        self.act = ACTLayer(action_space, cfg.hidden_size, cfg.use_orthogonal, cfg.gain)
        self.head_kind = 1 if self.act.continuous_action else 0          # lib.HEAD_GAUSSIAN / HEAD_CATEGORICAL
        self.n_actions = action_space.shape[0] if self.act.continuous_action else action_space.n  # head width
        if self.n_actions > 8:
            raise NotImplementedError("head widths up to 8 are built")
        self.device = torch.device(device)
        self._flat = FlatParams(self, self.device)
        self.value_normalizer = ValueNorm(1, device=self.device) if cfg.use_valuenorm else None

    @property
    def flat_params(self):
        return self._flat.flat

    def get_actor_para(self):   # base_value_policy_network.py:58-62
        return self.parameters()

    def get_critic_para(self):
        return self.parameters()
