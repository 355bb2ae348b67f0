"""Wide Discrete action spaces (9..64 actions): the masked env of tests/masked_oracle.py widened to n actions.

TEST INFRASTRUCTURE.  `wide_target_env(n)` is MaskedTargetEnv with an n-wide one-hot observation and Discrete(n);
`wide_target_vec(n)` its SyncVectorEnv form, and WideMaskedTrainer the feed-forward oracle loop with the reference's mask
ingest on it.  Pinned to the unmodified reference by tests/test_wide_actions_oracle.py (traces
tests/golden/trace_wide_actions_{9,64}.npz, recorded by tools/gen_golden_wide_actions.py)."""
from masked_oracle import MaskedTargetEnv, MaskedTargetVec, _MaskIngest
from oracle import loop

WIDTHS = (9, 64)


def wide_target_env(n):
    """MaskedTargetEnv with n actions and an n-wide observation."""
    return type(f"WideMaskedTargetEnv{n}", (MaskedTargetEnv,), {"obs_dim": n, "n_actions": n})


def wide_target_vec(n):
    """MaskedTargetVec over wide_target_env(n)."""
    env = wide_target_env(n)

    class WideMaskedTargetVec(MaskedTargetVec):
        obs_dim = n_actions = n

        def __init__(self, env_num, report=None):
            super().__init__(env_num, report)
            self.envs = [env() for _ in range(env_num)]

    return WideMaskedTargetVec


class WideMaskedTrainer(_MaskIngest, loop.Trainer):
    """Feed-forward PPO (oracle/loop.Trainer) on wide_target_vec(n)."""

    def __init__(self, cfg, env_num, n):
        super().__init__(cfg, "MaskedTarget", env_num, env=wide_target_vec(n)(env_num))
        self._ingest_masks(1)
