"""Host side of joint-action PPO (JRPO) without a GPU: the v3 row-index helper against the oracle's
recurrent_generator_v3 gather, and the flag value shared by the C header and the Python mirror."""
import os
import re

import numpy as np
import torch

from conftest import ROOT


def test_v3_row_indices_match_the_v3_gather():
    """Every step of a v3 chunk addresses the (T, N*A) buffer rows that recurrent_generator_v3 stacks: agent 0's rows
    for the critic / minibatch moments, all agent rows in (chunk, step, agent) order for the policy."""
    import jrpo_oracle
    from openrl_b200.buffers.replay_data import v3_row_indices

    T, N, A, L = 25, 4, 3, 2
    ids_buf = np.arange(T * N * A, dtype=np.float32).reshape(T, N, A, 1)   # value = buffer row t*B + n*A + a
    flat = jrpo_oracle._cast_v3(ids_buf)                                   # (N*T, A, 1)
    chunks = torch.tensor([12, 0, 49, 31])                                 # chunk 12 straddles env 0 and env 1
    want = np.stack([flat[c * L:c * L + L] for c in chunks.numpy()], axis=0)   # (chunks, L, A, 1)
    got_all = v3_row_indices(chunks, L, T, A, N * A, all_agents=True).numpy()
    got_0 = v3_row_indices(chunks, L, T, A, N * A).numpy()
    np.testing.assert_array_equal(got_all, want.reshape(-1))
    np.testing.assert_array_equal(got_0, want[:, :, 0, 0].reshape(-1))
    assert got_0[0:2].tolist() == [24 * N * A, 1 * A]   # t = 24 of env 0, then t = 0 of env 1


def test_joint_action_flag_matches_header():
    from openrl_b200 import lib

    text = open(os.path.join(ROOT, "include", "openrl_b200.h")).read()
    defs = dict((k, int(v)) for k, v in re.findall(r"#define (ORL_[A-Z0-9_]+) (\d+)\b", text))
    assert defs["ORL_PPO_JOINT_ACTION"] == lib.PPO_JOINT_ACTION
    others = [v for k, v in defs.items() if k.startswith("ORL_PPO_") and k != "ORL_PPO_JOINT_ACTION"]
    assert all(v & lib.PPO_JOINT_ACTION == 0 for v in others)   # a bit of its own
