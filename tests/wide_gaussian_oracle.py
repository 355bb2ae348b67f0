"""Box action spaces of 9..64 dimensions: a target env of the shapes the wide DiagGaussian head is built for, and the
oracle loop on it.

TEST INFRASTRUCTURE.  `wide_gaussian_env(d, n)` is WideBoxTargetEnv (tests/wide_obs_oracle.py) with d observation
features and a Box(n) action whose target is the first n features.  TRACES are the two shapes the traces pin:
dm_control humanoid's (d = 67, Box(21)) and the shared-memory worst case of the update (d = 256, Box(64)).  The
SyncVectorEnv forms and the oracle trainers on them are pinned to the unmodified reference by
tests/test_wide_gaussian_oracle.py (traces tests/golden/trace_wide_gaussian_{21,64}.npz, recorded by
tools/gen_golden_wide_gaussian.py)."""
import numpy as np

from oracle import loop
from wide_obs_oracle import WideBoxTargetEnv, WideBoxTargetVec

# n -> observation width d of the trace trace_wide_gaussian_<n> (both wider than 64: they run with use_wide_observations)
TRACES = {21: 67, 64: 256}


def wide_gaussian_env(d, n):
    """WideBoxTargetEnv with d features in [0, 1) and Box(n) actions rewarded by 1 - mean |target - clip(a, 0, 1)| over
    the first n features."""
    return type(f"WideGaussianTargetEnv{d}x{n}", (WideBoxTargetEnv,), {"obs_dim": d, "act_dim": n})


def spaced_wide_gaussian_env(d, n):
    """wide_gaussian_env(d, n) with the spaces a host vec-env reads (make(..., make_custom_envs=...))."""
    base = wide_gaussian_env(d, n)

    def __init__(self):
        from openrl_b200 import spaces

        base.__init__(self)
        self.observation_space = spaces.Box(-np.inf, np.inf, (d,), np.float32)
        self.action_space = spaces.Box(-1.0, 1.0, (n,), np.float32)
    return type(f"SpacedWideGaussianTargetEnv{d}x{n}", (base,), {"__init__": __init__})


def wide_gaussian_vec(d, n):
    """wide_gaussian_env(d, n) under SyncVectorEnv: obs (N,1,d), rewards (N,1,1) f64, dones (N,1) bool."""
    env = wide_gaussian_env(d, n)

    def __init__(self, env_num):
        self.N = env_num
        self.envs = [env() for _ in range(env_num)]
    return type(f"WideGaussianTargetVec{d}x{n}", (WideBoxTargetVec,), {"obs_dim": d, "act_dim": n, "__init__": __init__})


class WideGaussianTrainer(loop.Trainer):
    """Feed-forward PPO with a DiagGaussian head (oracle/loop.Trainer) on wide_gaussian_vec(d, n)."""

    def __init__(self, cfg, env_num, d, n):
        super().__init__(cfg, "WideGaussianTarget", env_num, env=wide_gaussian_vec(d, n)(env_num))
