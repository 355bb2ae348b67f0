"""CartPole tensor-core rollout (R envs per CTA) at env counts that leave the last CTA ragged, through `orl_rollout` with
device sampling (Philox noise), T = 128.

Bars: observations, rewards and masks bit-exact against the numpy oracle env stepped with the kernel's own sampled
actions; log-probs within 1e-5 of `orl_policy_eval` on the recorded observations and actions; one launch over [0, T)
identical to T one-step launches."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

T = 128
SEED = 11


@pytest.fixture(scope="module")
def device():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _driver(n_envs):
    from openrl_b200.algorithms.ppo import PPOAlgorithm
    from openrl_b200.buffers import NormalReplayBuffer
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.drivers.onpolicy_driver import OnPolicyDriver
    from openrl_b200.envs.common import make
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent

    cfg = create_config_parser().parse_args(["--seed", "3", "--episode_length", str(T), "--log_interval", "1000000"])
    cfg.quiet = True
    env = make("CartPole-v1", env_num=n_envs)
    net = PPONet(env, cfg=cfg, device="cuda:0")
    agent = PPOAgent(net)
    trainer = PPOAlgorithm(cfg, net.module, agent_num=1, device=net.device)
    buf = NormalReplayBuffer(cfg, 1, env.observation_space, env.action_space, device=net.device)
    drv = OnPolicyDriver({"cfg": cfg, "num_agents": 1, "run_dir": None, "envs": env, "device": net.device}, trainer, buf, agent)
    env._seed_streams(SEED)   # the same per-env PCG64 streams as CartPoleVec.reset(seed=SEED)
    drv.reset_and_buffer_init()
    drv.trainer.prep_rollout()
    return drv


def _launch(drv, t_begin, t_end, counter=True):
    """counter=False keys the noise of step t by t alone (no device counter, which advances by t_end - t_begin per launch)."""
    from openrl_b200 import lib

    a = drv._rollout_args(t_begin, t_end, None)
    if not counter:
        a.rng_counter = None
    lib.check(drv._lib.orl_rollout(a, lib.current_stream()), "orl_rollout")


def _buffers(drv):
    import torch

    torch.cuda.synchronize()
    b = drv.buffer.data
    return {k: getattr(b, k).cpu().numpy().copy() for k in ("actions", "policy_obs", "rewards", "masks", "action_log_probs")}


@pytest.mark.parametrize("n_envs", [4096 + 17, 100])
def test_rollout_rows_matches_oracle_env_and_policy_eval(device, n_envs):
    import torch

    from openrl_b200 import lib
    from oracle.envs import CartPoleVec

    drv = _driver(n_envs)
    _launch(drv, 0, T)
    got = _buffers(drv)
    ref = CartPoleVec(n_envs)
    assert np.array_equal(got["policy_obs"][0], ref.reset(seed=SEED))
    acts = got["actions"]
    assert set(np.unique(acts)) <= {0.0, 1.0}
    for t in range(T):
        o, r, d, _ = ref.step(acts[t].astype(np.int64))
        assert np.array_equal(got["policy_obs"][t + 1], o), t
        assert np.array_equal(got["rewards"][t], r.astype(np.float32)), t
        assert np.array_equal(got["masks"][t + 1][..., 0], (~d).astype(np.float32)), t

    pol = drv.trainer.algo_module.models["policy"]
    rows = T * n_envs
    obs = torch.from_numpy(got["policy_obs"][:T].reshape(rows, 4)).to(device)
    act = torch.from_numpy(acts.reshape(rows, 1)).to(device)
    logp = torch.empty(rows, 1, dtype=torch.float32, device=device)
    ent = torch.empty(rows, 1, dtype=torch.float32, device=device)
    lib.check(drv._lib.orl_policy_eval(lib.ptr(pol.flat_params), pol.obs_dim, pol.n_actions, pol.activation_id, pol.head_kind,
                                       lib.ptr(obs), lib.ptr(act), None, lib.ptr(logp), lib.ptr(ent), rows,
                                       lib.current_stream()), "orl_policy_eval")
    torch.cuda.synchronize()
    np.testing.assert_allclose(got["action_log_probs"].reshape(rows, 1), logp.cpu().numpy(), rtol=0, atol=1e-5)


def test_rollout_rows_single_launch_equals_per_step_launches(device):
    n_envs = 4096 + 17
    one = _driver(n_envs)
    _launch(one, 0, T, counter=False)
    per = _driver(n_envs)
    for t in range(T):
        _launch(per, t, t + 1, counter=False)
    a, b = _buffers(one), _buffers(per)
    for k in a:
        assert np.array_equal(a[k], b[k]), k
