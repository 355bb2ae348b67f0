"""openrl_b200 — H100-native (sm_90a) implementation of OpenRL's rollout-collection +
PPO/MAPPO-update hot path behind OpenRL's own Python surface (`make`, `PPONet`, `PPOAgent`).

Host code is Python (as the reference's is); all numeric inner loops are hand-written CUDA in
`openrl_b200/csrc`, reached through the C-ABI of `include/openrl_b200.h` via ctypes.
"""
__version__ = "0.1.0"
