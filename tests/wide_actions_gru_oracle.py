"""Wide Discrete action spaces (9..64 actions) with a GRU policy: the recurrent oracle loop on the widened masked env.

TEST INFRASTRUCTURE.  WideMaskedMATrainer is the recurrent oracle loop (oracle/loop_ma.MATrainer) with the reference's mask
ingest on wide_target_vec(n) of tests/wide_actions_oracle.py.  Pinned to the unmodified reference by
tests/test_wide_actions_gru_oracle.py (traces tests/golden/trace_wide_actions_gru_{9,64}.npz, recorded by
tools/gen_golden_wide_actions_gru.py)."""
from masked_oracle import _MaskIngest
from oracle import envs as oenvs
from oracle import loop_ma
from wide_actions_oracle import wide_target_vec


class WideMaskedMATrainer(_MaskIngest, loop_ma.MATrainer):
    """Recurrent PPO (oracle/loop_ma.MATrainer) on wide_target_vec(n)."""

    def __init__(self, cfg, env_num, n):
        saved = oenvs.ENVS.get("MaskedTarget")
        oenvs.ENVS["MaskedTarget"] = lambda k: wide_target_vec(n)(k)
        try:
            super().__init__(cfg, "MaskedTarget", env_num)
        finally:
            if saved is None:
                del oenvs.ENVS["MaskedTarget"]
            else:
                oenvs.ENVS["MaskedTarget"] = saved
        self._ingest_masks(self.A)
