"""The host-stepped rollout (`HostVecEnv`, ORL_ENV_NONE): one loop over one group or two groups in ping-pong, one act
launcher, one staged step per env range.

GPU: on an env whose observations do not depend on the actions, the synchronous and the two-group loop write the same
bits and train to the same policy over consecutive `PPOAgent.train` calls, so both keep drawing fresh noise from the
second call on.  CPU: the staged step of the whole range goes through `env.step`, that of a sub-range through
`env.step_range`, and the uploaded block has the staged length with and without action masks."""
import numpy as np
import pytest

from helpers import CountEnv


def _train_twice(recurrent, grouped, T, N):
    """Two `PPOAgent.train(T * N)` calls on a fresh env and net; per call the buffers and the policy parameters."""
    import torch

    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.envs.common import make
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.logger import Logger

    flags = ["--seed", "5", "--episode_length", str(T), "--ppo_epoch", "1", "--num_mini_batch", "2",
             "--host_env_groups", grouped]
    if recurrent:
        flags += ["--use_recurrent_policy", "true", "--data_chunk_length", "4"]
    cfg = create_config_parser().parse_args(flags)
    cfg.quiet = True
    env = make("Count-v0", env_num=N,
               make_custom_envs=lambda id, env_num, render_mode=None, **kw: [(lambda i=i: CountEnv(i, horizon=5)) for i in range(env_num)])
    assert env.supports_groups
    net = PPONet(env, cfg=cfg, device="cuda:0")     # re-seeds torch: the same initial weights and minibatch permutations
    agent = PPOAgent(net)
    out = []
    for _ in range(2):
        agent.train(total_time_steps=T * N, logger=Logger(quiet=True))
        torch.cuda.synchronize()
        b = agent.driver.buffer.data
        keys = ("actions", "action_log_probs") + (("rnn_states",) if recurrent else ())
        out.append({k: getattr(b, k).cpu().numpy().copy() for k in keys}
                   | {"policy": net.module.models["policy"].flat_params.cpu().numpy().copy()})
    assert agent.driver.host_act_steps == 2 * T      # the second call's slots took Philox steps T .. 2T - 1
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("recurrent", [False, True])
def test_host_loops_agree_across_train_calls(cuda, recurrent):
    T, N = 16, 64
    sync, grouped = _train_twice(recurrent, "false", T, N), _train_twice(recurrent, "true", T, N)
    for call in range(2):
        for k in sync[call]:
            assert np.array_equal(sync[call][k], grouped[call][k]), (call, k)


class _RecordingHost:
    """A host vec-env that records which step entry point was called; obs = [action, env index], reward = action."""

    def __init__(self, n, masks):
        from openrl_b200 import spaces

        self.parallel_env_num, self.agent_num, self.masks = n, 1, masks
        self.observation_space = spaces.Box(-np.inf, np.inf, (2,), np.float32)
        self.action_space = spaces.Discrete(3)
        self.calls = []

    def reset(self, seed=None):
        return np.zeros((self.parallel_env_num, 1, 2), np.float32)

    def step(self, actions):
        self.calls.append(("step", 0, self.parallel_env_num))
        return self._step(0, self.parallel_env_num, actions)

    def step_range(self, lo, hi, actions):
        self.calls.append(("step_range", lo, hi))
        return self._step(lo, hi, actions)

    def _step(self, lo, hi, actions):
        assert actions.dtype == np.int64 and actions.shape == (hi - lo, 1, 1)
        a = actions[:, 0, 0].astype(np.float32)
        obs = np.stack([a, np.arange(lo, hi, dtype=np.float32)], -1)[:, None, :]
        infos = [{"action_masks": np.array([1, e % 2, 1])} if self.masks else {} for e in range(lo, hi)]
        return obs, a[:, None, None], (np.arange(lo, hi) % 3 == 0)[:, None], infos


@pytest.mark.parametrize("masks", [False, True])
def test_staged_step_steps_the_range_and_returns_the_staged_block(masks):
    import torch

    from openrl_b200.envs.vec_env.host_venv import HostVecEnv

    N = 6
    env = HostVecEnv(_RecordingHost(N, masks), device="cpu")
    w = 2 + 2 + (3 if masks else 0)
    for lo, hi, call in ((0, N, "step"), (2, 5, "step_range"), (0, N, "step")):
        n = hi - lo
        acts = torch.arange(lo, hi, dtype=torch.float32).remainder(3).view(n, 1)
        env.fetch_actions(lo, hi, acts)
        dev, obs, rewards, dones, infos, has_masks = env.step_staged(lo, hi)
        assert env.env.calls[-1] == (call, lo, hi)
        assert has_masks == masks and len(infos) == n
        blk = dev.numpy()
        assert blk.shape == (n * w,)
        assert np.array_equal(blk[:n * 2].reshape(n, 2), np.stack([acts[:, 0].numpy(), np.arange(lo, hi)], -1))
        assert np.array_equal(blk[n * 2:n * 3], acts[:, 0].numpy())
        assert np.array_equal(blk[n * 3:n * 4], (np.arange(lo, hi) % 3 == 0).astype(np.float32))
        if masks:
            want = np.stack([[1, e % 2, 1] for e in range(lo, hi)]).astype(np.float32)
            assert np.array_equal(blk[n * 4:].reshape(n, 3), want)
    assert len(env.env.calls) == 3
