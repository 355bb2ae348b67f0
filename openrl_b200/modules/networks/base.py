"""Building blocks with the reference's module tree / state_dict names
(openrl/modules/networks/utils/mlp.py:8-46,100-176; distributions.py:58-66; valuenorm.py:6-57).

Parameters are created on the CPU with the reference's initialisation sequence (default
nn.Linear init, then orthogonal_/constant_) so that the global torch generator is consumed
identically and a given seed yields the reference's initial weights; `FlatParams` then moves them
into ONE flat float32 CUDA buffer in state_dict order — the layout the kernels read
(orl_mlp.cuh) — and re-points every nn.Parameter at its slice, so `state_dict()`,
`load_state_dict()` and `torch.save(module)` keep working (SURVEY.md §5.4).

These modules carry no torch forward: the numeric path is CUDA only (`orl_rollout`,
`orl_critic_values`, `orl_ppo_*`)."""
import torch
import torch.nn as nn

ACT_NAMES = ["tanh", "relu", "leaky_relu", "selu"]


def _init(module, gain, use_orthogonal=True):
    (nn.init.orthogonal_ if use_orthogonal else nn.init.xavier_uniform_)(module.weight.data, gain=gain)
    nn.init.constant_(module.bias.data, 0)
    return module


def check_obs_shape(shape, wide=False):
    """The observation shapes the kernels take: flat vectors of width 1..64, and of 65..256 when `wide` (a feed-forward
    policy or critic with cfg.use_wide_observations: fc1 runs over 64-wide panels of the observation)."""
    if len(shape) == 1 and shape[0] <= (256 if wide else 64):
        return
    if wide:
        raise NotImplementedError("vector observations of width <= 256 only (the bound of use_wide_observations); "
                                  f"got shape {tuple(shape)}")
    raise NotImplementedError("vector observations of width <= 64 only (65..256: feed-forward policies and critics "
                              f"with use_wide_observations, not GRU policies or use_share_model); got shape {tuple(shape)}")


class MLPLayer(nn.Module):
    def __init__(self, input_dim, hidden_size, layer_N, use_orthogonal, activation_id):
        super().__init__()
        if layer_N != 1:
            raise NotImplementedError("openrl_b200 kernels are built for layer_N == 1 (the reference default)")
        act = [nn.Tanh(), nn.ReLU(), nn.LeakyReLU(), nn.ELU()][activation_id]
        gain = nn.init.calculate_gain(ACT_NAMES[activation_id])
        self.fc1 = nn.Sequential(_init(nn.Linear(input_dim, hidden_size), gain, use_orthogonal), act,
                                 nn.LayerNorm(hidden_size))
        self.fc3 = nn.Sequential(_init(nn.Linear(hidden_size, hidden_size), gain, use_orthogonal),
                                 nn.LayerNorm(hidden_size))


class MLPBase(nn.Module):
    def __init__(self, cfg, obs_shape):
        super().__init__()
        if cfg.use_feature_normalization:
            raise NotImplementedError("use_feature_normalization is not built into the kernels yet")
        if cfg.hidden_size != 64:
            raise NotImplementedError("openrl_b200 kernels are built for hidden_size == 64 (the reference default)")
        self.hidden_size = cfg.hidden_size
        self.mlp = MLPLayer(obs_shape[0], cfg.hidden_size, cfg.layer_N, cfg.use_orthogonal, cfg.activation_id)

    @property
    def output_size(self):
        return self.hidden_size


class RNNLayer(nn.Module):
    """rnn.py:5-28: one-layer nn.GRU (orthogonal weights, zero biases) followed by LayerNorm.  Only the
    parameter tree / initialisation lives here; the forward and the chunked BPTT are orl_rnn.cu."""

    def __init__(self, inputs_dim, outputs_dim, recurrent_N, use_orthogonal, rnn_type="gru"):
        super().__init__()
        if rnn_type != "gru" or recurrent_N != 1:
            raise NotImplementedError("the recurrent kernels are built for rnn_type == 'gru' and recurrent_N == 1 "
                                      "(the reference defaults)")
        self.rnn = nn.GRU(inputs_dim, outputs_dim, num_layers=recurrent_N)
        for name, param in self.rnn.named_parameters():
            if "bias" in name:
                nn.init.constant_(param, 0)
            elif "weight" in name:
                (nn.init.orthogonal_ if use_orthogonal else nn.init.xavier_uniform_)(param)
        self.norm = nn.LayerNorm(outputs_dim)


class Categorical(nn.Module):
    def __init__(self, num_inputs, num_outputs, use_orthogonal=True, gain=0.01):
        super().__init__()
        self.linear = _init(nn.Linear(num_inputs, num_outputs), gain, use_orthogonal)


class AddBias(nn.Module):
    def __init__(self, bias):
        super().__init__()
        self._bias = nn.Parameter(bias.unsqueeze(1))


class DiagGaussian(nn.Module):
    """distributions.py:75-98: mean = fc_mean(x), log-std = a learnable bias initialised to 0."""

    def __init__(self, num_inputs, num_outputs, use_orthogonal=True, gain=0.01):
        super().__init__()
        self.fc_mean = _init(nn.Linear(num_inputs, num_outputs), gain, use_orthogonal)
        self.logstd = AddBias(torch.zeros(num_outputs))


class PopArt(nn.Module):
    """`v_out` under cfg.use_popart (popart.py:9-117).  In the reference's PPO path the PopArt statistics are never
    driven: `value_normalizer` is the ValueNorm object (base_value_network.py:31-34) or None, so `PopArt.update /
    normalize / denormalize` have no caller (ppo.py:190-217, replay_data.py:320-423) and the layer acts as
    `F.linear(x, weight, bias)`.  What differs from nn.Linear is (i) the initialisation sequence — `reset_parameters`
    draws kaiming-uniform weights and a uniform bias from the global generator BEFORE the orthogonal / zero init
    overwrites them (value_network.py:106-109), shifting every later draw — and (ii) four extra checkpoint entries
    (stddev, mean, mean_sq, debiasing_term; buffers here, requires_grad=False parameters there)."""

    def __init__(self, input_shape, output_shape, beta=0.99999, epsilon=1e-5):
        super().__init__()
        import math

        self.beta, self.epsilon = beta, epsilon
        self.weight = nn.Parameter(torch.empty(output_shape, input_shape))
        self.bias = nn.Parameter(torch.empty(output_shape))
        self.register_buffer("stddev", torch.ones(output_shape))
        self.register_buffer("mean", torch.zeros(output_shape))
        self.register_buffer("mean_sq", torch.zeros(output_shape))
        self.register_buffer("debiasing_term", torch.tensor(0.0))
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))          # reset_parameters (popart.py:47-55)
        bound = 1 / math.sqrt(input_shape)
        nn.init.uniform_(self.bias, -bound, bound)


class ACTLayer(nn.Module):
    def __init__(self, action_space, inputs_dim, use_orthogonal, gain):
        super().__init__()
        kind = action_space.__class__.__name__
        if kind == "Discrete":
            self.continuous_action = False
            self.action_out = Categorical(inputs_dim, action_space.n, use_orthogonal, gain)
        elif kind == "Box":
            self.continuous_action = True
            self.action_out = DiagGaussian(inputs_dim, action_space.shape[0], use_orthogonal, gain)
        else:
            raise NotImplementedError(f"action space {kind} has no CUDA head yet (Discrete and Box are built)")


class ValueNorm(nn.Module):
    """Running statistics of the value targets (valuenorm.py:6-57); the three scalars live in one
    float32 CUDA tensor `state` = (running_mean, running_mean_sq, debiasing_term) updated by
    orl_ppo_apply and read by orl_gae / orl_ppo_fwdbwd."""

    def __init__(self, input_shape=1, beta=0.99999, device="cpu"):
        super().__init__()
        self.beta = beta
        self.register_buffer("state", torch.zeros(3, dtype=torch.float32, device=device))

    @property
    def running_mean(self):
        return self.state[0:1]

    @property
    def running_mean_sq(self):
        return self.state[1:2]

    @property
    def debiasing_term(self):
        return self.state[2]

    # checkpoints carry the reference's three entries (valuenorm.py:27-35: running_mean (1,), running_mean_sq (1,),
    # debiasing_term ()), so a critic state_dict saved by either implementation loads into the other
    def _save_to_state_dict(self, destination, prefix, keep_vars):
        destination[prefix + "running_mean"] = self.state[0:1].detach().clone()
        destination[prefix + "running_mean_sq"] = self.state[1:2].detach().clone()
        destination[prefix + "debiasing_term"] = self.state[2].detach().clone()

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        if prefix + "state" in state_dict:                       # round-1 checkpoints
            self.state.copy_(state_dict[prefix + "state"].to(self.state.device).reshape(3))
            return
        for i, name in enumerate(("running_mean", "running_mean_sq", "debiasing_term")):
            if prefix + name in state_dict:
                self.state[i] = state_dict[prefix + name].to(self.state.device).reshape(-1)[0]
            elif strict:
                missing_keys.append(prefix + name)

    def running_mean_var(self):
        d = self.state[2].clamp(min=1e-5)
        m = self.state[0] / d
        var = (self.state[1] / d - m * m).clamp(min=1e-2)
        return m, var


class FlatParams:
    """Flatten a module's parameters (named_parameters order) into one CUDA buffer."""

    def __init__(self, module, device):
        ps = [p for _, p in module.named_parameters()]
        self.numel = sum(p.numel() for p in ps)
        self.flat = torch.empty(self.numel, dtype=torch.float32, device=device)
        off = 0
        for p in ps:
            n = p.numel()
            view = self.flat[off:off + n].view(p.shape)
            view.copy_(p.data.to(torch.float32))
            p.data = view
            off += n
