#!/usr/bin/env python
"""Record the wide-action GRU traces by executing the unmodified reference on the masked env widened to 9 and 64 actions.

TEST INFRASTRUCTURE, run where the reference source is present; the outputs are committed under tests/golden/.

    PYTHONPATH=oracle/refstubs:oracle:<reference checkout> python tools/gen_golden_wide_actions_gru.py

The recipe of tools/gen_golden_wide_actions.py (`gen_trace` of oracle/gen_golden.py unchanged, MaskedTargetEnv of
tests/masked_oracle.py with `obs_dim = n_actions = n`) with a recurrent policy, as trace_masked_gru is to trace_masked_ff:

  trace_wide_actions_gru_9    GRU PPO (--use_recurrent_policy true --data_chunk_length 3), Discrete(9), 4 envs, T = 16,
                              2 epochs, 2 minibatches, 2 iterations
  trace_wide_actions_gru_64   the same with Discrete(64)
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

import gen_golden as gg  # noqa: E402
import gen_golden_masked as gm  # noqa: E402
from masked_oracle import MaskedTargetEnv  # noqa: E402
from wide_actions_oracle import WIDTHS  # noqa: E402

ENV_NUM, ITERS = 4, 2
FLAGS = gm.TRACES["masked_gru"]


def main():
    torch.set_num_threads(8)   # the thread count every other trace was recorded with (tests/test_oracle_loop.py)
    make = gg.make
    gg.make = lambda id, env_num=1, **kw: make(id, env_num=env_num, make_custom_envs=gm.make_masked_envs, **kw)
    saved = MaskedTargetEnv.obs_dim, MaskedTargetEnv.n_actions
    try:
        for n in WIDTHS:
            # GymMaskedTarget builds MaskedTargetEnv() and reads its class attributes for the spaces
            MaskedTargetEnv.obs_dim = MaskedTargetEnv.n_actions = n
            gg.gen_trace("MaskedTarget", ENV_NUM, FLAGS, ITERS, f"wide_actions_gru_{n}")
    finally:
        gg.make = make
        MaskedTargetEnv.obs_dim, MaskedTargetEnv.n_actions = saved


if __name__ == "__main__":
    main()
