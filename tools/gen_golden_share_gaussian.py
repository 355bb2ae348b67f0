#!/usr/bin/env python
"""Record the shared-model DiagGaussian trace by executing the unmodified reference.

TEST INFRASTRUCTURE, run where the reference source is present; the output is committed under tests/golden/.

    PYTHONPATH=oracle/refstubs:oracle:<reference checkout> python tools/gen_golden_share_gaussian.py

Uses `gen_trace` of oracle/gen_golden.py unchanged: IdentityEnvcontinuous (Box(1) actions), 4 envs, seed 0,
T = 16, 2 epochs, 2 minibatches, 2 iterations, with --use_share_model true, so the reference builds one
PolicyValueNetwork whose ACTLayer carries a DiagGaussian head (act.action_out.fc_mean + act.action_out.logstd).
Eight torch threads, as the other traces were recorded with.

  trace_share_gaussian
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]

import gen_golden as gg  # noqa: E402

FLAGS = ["--seed", "0", "--episode_length", "16", "--ppo_epoch", "2", "--num_mini_batch", "2", "--use_share_model", "true",
         "--log_interval", "1000"]


def main():
    torch.set_num_threads(8)
    gg.gen_trace("IdentityEnvcontinuous", 4, FLAGS, 2, "share_gaussian")


if __name__ == "__main__":
    main()
