#!/usr/bin/env python
"""Record the joint-action PPO (JRPO, `--use_joint_action_loss true`) traces by executing the unmodified reference.

TEST INFRASTRUCTURE, run where the reference source is present; the outputs are committed under tests/golden/.

    PYTHONPATH=oracle/refstubs:oracle:<reference checkout> python tools/gen_golden_jrpo.py

Uses `gen_trace` of oracle/gen_golden.py unchanged.  JRPO draws its minibatches from
ReplayData.recurrent_generator_v3 (replay_data.py:425-551), which gen_trace does not wrap, so this script wraps
it to record the advantages it is handed (first call of every iteration, one call per epoch) and adds them to
the written trace as `it<i>/advantages`, the key the other recurrent traces carry.

  trace_mpe_jrpo     simple_spread, 4 envs, the examples/mpe/mpe_jrpo.yaml flags, ppo_epoch 2, 2 iterations,
                     data_chunk_length 2, one minibatch (25 steps: chunks straddle env boundaries)
  trace_mpe_jrpo_mb  the same with --num_mini_batch 2 --data_chunk_length 4
"""
import os

import numpy as np
import torch

import gen_golden as gg
from openrl.buffers.replay_data import ReplayData

JRPO = ["--seed", "0", "--episode_length", "25", "--ppo_epoch", "2", "--lr", "7e-4", "--critic_lr", "7e-4",
        "--use_recurrent_policy", "true", "--use_joint_action_loss", "true", "--use_valuenorm", "true",
        "--use_adv_normalize", "true", "--log_interval", "1000"]
TRACES = {"mpe_jrpo": JRPO, "mpe_jrpo_mb": JRPO + ["--num_mini_batch", "2", "--data_chunk_length", "4"]}
EPOCHS, ITERS = 2, 2


def record(tag, flags):
    advs = []
    orig_v3 = ReplayData.recurrent_generator_v3

    def v3(self, advantages, *a, **k):
        advs.append(advantages.copy())
        return orig_v3(self, advantages, *a, **k)

    ReplayData.recurrent_generator_v3 = v3
    try:
        gg.gen_trace("simple_spread", 4, flags, ITERS, tag)
    finally:
        ReplayData.recurrent_generator_v3 = orig_v3
    assert len(advs) == EPOCHS * ITERS, len(advs)
    path = os.path.join(gg.OUT, f"trace_{tag}.npz")
    with np.load(path, allow_pickle=True) as d:
        rec = {k: d[k] for k in d.files}
    for it in range(ITERS):
        rec[f"it{it}/advantages"] = advs[it * EPOCHS]
    np.savez_compressed(path, **rec)


def main():
    torch.set_num_threads(8)   # the thread count every other trace was recorded with (tests/test_oracle_loop.py)
    for tag, flags in TRACES.items():
        record(tag, flags)


if __name__ == "__main__":
    main()
