"""Key layout of the device action noise, on one GPU.

Every rollout kernel draws the Exp(1) noise of (step, row) from Philox4x32-10 keyed by the seed, with counter
(step lo, step hi, row + rng_row_offset, lane), lanes 0 / 1 giving the 8 draws -log U.  That layout is what makes an
env-sharded run draw the noise of the unsharded one.  Here the same table is built on the host (numpy Philox, a step
base above 2^32 and a non-zero row offset) and each acting path runs twice on the same inputs: once with device
Philox, once with that table.  Actions must agree and log-probs be bit-equal; a disagreement passes only at a near-tie
of argmax(p / q), because the host -log may differ from the device logf in the last bit.  For device-env paths each env
is compared up to its first such tie (the trajectories part there)."""
import numpy as np
import pytest

from helpers import philox_units

pytestmark = pytest.mark.gpu

SEED = 0x1234_5678_9ABC
STEP_BASE = (1 << 32) + 77      # the high step word must reach the counter
ROW_OFFSET = 1000               # and so must rng_row_offset


def noise_table(T, rows, n, seed, step_base, row_offset):
    """(T, rows, n) float32 Exp(1) noise exactly as the device keys it: step = step_base + t, row = row + row_offset."""
    return (-np.log(philox_units(T, rows, seed, step_base, row_offset, (0, 1))[..., :n])).astype(np.float32)


def assert_same_draws(act_a, lp_a, act_b, lp_b, q, per_env_trajectory=False, valid=None):
    """act/lp: (T, rows); q: (T, rows, n).  Actions agree with bit-equal log-probs, or the rows are at a near-tie.
    `valid` (T, rows) leaves out the entries it marks False."""
    act_a, act_b = act_a.astype(np.int64), act_b.astype(np.int64)
    T, rows = act_a.shape
    live = np.ones(rows, bool)
    compared = 0
    for t in range(T):
        cur = live & (valid[t] if valid is not None else True)
        same = act_a[t] == act_b[t]
        chk = cur & same
        assert np.array_equal(lp_a[t][chk].view(np.int32), lp_b[t][chk].view(np.int32)), f"log-probs differ at step {t}"
        compared += int(chk.sum())
        diff = np.nonzero(cur & ~same)[0]
        if diff.size:
            ra = np.exp(lp_a[t, diff].astype(np.float64)) / q[t, diff, act_a[t, diff]]
            rb = np.exp(lp_b[t, diff].astype(np.float64)) / q[t, diff, act_b[t, diff]]
            assert np.all(np.abs(ra - rb) <= 1e-6 * np.maximum(ra, rb)), f"{diff.size} rows pick different actions at step {t}"
            if per_env_trajectory:
                live[diff] = False
    assert compared >= act_a.size // 2, "too few rows compared"


@pytest.fixture(scope="module")
def device():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _policy(n_actions, obs_dim, extra=()):
    from openrl_b200 import spaces
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.modules.common import PPONet

    class Env:
        agent_num, parallel_env_num = 1, 1
        observation_space, action_space = spaces.Box(-5, 5, (obs_dim,), np.float32), spaces.Discrete(n_actions)

        def reset(self, seed=None):
            return np.zeros((1, 1, obs_dim), np.float32)

    cfg = create_config_parser().parse_args(["--seed", "5", *extra])
    cfg.quiet = True
    net = PPONet(Env(), cfg=cfg, device="cuda:0")
    sd = net.module.models["policy"].state_dict()
    for k in sd:
        if k.endswith("action_out.linear.weight"):
            sd[k].mul_(8.0)   # probabilities far from uniform
    return net.module


def _act_ff(module, obs, noise):
    """PPOModule.act's launch with the step base and row offset under test."""
    import torch

    from openrl_b200 import lib

    pol = module.models["policy"]
    rows = obs.shape[0]
    actions = torch.empty(rows, 1, dtype=torch.float32, device=obs.device)
    logp = torch.empty(rows, 1, dtype=torch.float32, device=obs.device)
    a = lib.OrlRolloutArgs()
    a.env_kind, a.n_envs, a.n_agents, a.episode_length = lib.ENV_NONE, rows, 1, 1
    a.t_begin, a.t_end = 0, 1
    a.obs_dim, a.critic_obs_dim, a.n_actions = pol.obs_dim, 0, pol.n_actions
    a.activation_id, a.deterministic, a.head_kind = pol.activation_id, 0, pol.head_kind
    a.policy_params, a.policy_obs = lib.ptr(pol.flat_params), lib.ptr(obs)
    a.actions, a.action_log_probs, a.exp_noise = lib.ptr(actions), lib.ptr(logp), lib.ptr(noise)
    a.rng_seed, a.rng_step_base, a.rng_row_offset = SEED, STEP_BASE, ROW_OFFSET
    fn = module._lib.orl_share_rollout if module.share_model else module._lib.orl_rollout
    lib.check(fn(a, lib.current_stream()), "act")
    torch.cuda.synchronize()
    return actions.cpu().numpy()[None, :, 0], logp.cpu().numpy()[None, :, 0]


@pytest.mark.parametrize("share", [False, True])
def test_act_feed_forward_noise_key(device, share):
    import torch

    n, rows = 5, 20_000
    module = _policy(n, 6, ["--use_share_model", "true"] if share else [])
    assert module.share_model == share
    obs = torch.from_numpy(np.random.default_rng(1).normal(size=(rows, 6)).astype(np.float32)).to(device)
    q = noise_table(1, rows, n, SEED, STEP_BASE, ROW_OFFSET)
    a0, l0 = _act_ff(module, obs, None)
    a1, l1 = _act_ff(module, obs, torch.from_numpy(q).to(device))
    assert_same_draws(a0, l0, a1, l1, q)


def test_act_recurrent_noise_key(device):
    """The recurrent act (orl_rnn_act_rows on rows [0, rows), rng_row_offset 0) keys by the local row."""
    import torch

    n, rows = 5, 20_000
    module = _policy(n, 6, ["--use_recurrent_policy", "true"])
    obs = np.random.default_rng(2).normal(size=(rows, 6)).astype(np.float32)
    q = noise_table(1, rows, n, SEED, STEP_BASE, 0)
    a0, l0, _ = module.act(obs, deterministic=False, rng_seed=SEED, rng_step=STEP_BASE)
    a1, l1, _ = module.act(obs, deterministic=False, exp_noise=q, rng_seed=SEED, rng_step=STEP_BASE)
    torch.cuda.synchronize()
    assert_same_draws(a0.cpu().numpy().T, l0.cpu().numpy().T, a1.cpu().numpy().T, l1.cpu().numpy().T, q)


def _driver(env_name, n_envs, T, extra=()):
    from openrl_b200.algorithms.ppo import PPOAlgorithm
    from openrl_b200.buffers import NormalReplayBuffer
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.drivers.onpolicy_driver import OnPolicyDriver
    from openrl_b200.envs.common import make
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent

    cfg = create_config_parser().parse_args(["--seed", "3", "--episode_length", str(T), "--log_interval", "1000000", *extra])
    cfg.quiet = True
    env = make(env_name, env_num=n_envs)
    net = PPONet(env, cfg=cfg, device="cuda:0")
    agent = PPOAgent(net)
    trainer = PPOAlgorithm(cfg, net.module, agent_num=env.agent_num, device=net.device)
    buf = NormalReplayBuffer(cfg, env.agent_num, env.observation_space, env.action_space, device=net.device)
    drv = OnPolicyDriver({"cfg": cfg, "num_agents": env.agent_num, "run_dir": None, "envs": env, "device": net.device},
                         trainer, buf, agent)
    drv.reset_and_buffer_init()
    drv.trainer.prep_rollout()
    return drv


def _device_env_rollout(env_name, n_envs, T, table):
    import torch

    from openrl_b200 import lib

    drv = _driver(env_name, n_envs, T)
    noise = None if table is None else torch.from_numpy(table).to(drv.device)
    a = drv._rollout_args(0, T, noise)
    a.rng_seed, a.rng_step_base, a.rng_counter, a.rng_row_offset = SEED, STEP_BASE, None, ROW_OFFSET * a.n_agents
    lib.check(drv._lib.orl_rollout(a, lib.current_stream()), "orl_rollout")
    torch.cuda.synchronize()
    d = drv.buffer.data
    B = n_envs * drv.envs.agent_num
    return d.actions.cpu().numpy().reshape(T, B), d.action_log_probs.cpu().numpy().reshape(T, B)


@pytest.mark.parametrize("env_name,n_actions,n_envs", [("CartPole-v1", 2, 1000), ("GridWorldEnv", 5, 1000),
                                                       ("simple_spread", 5, 300)])
def test_device_env_rollout_noise_key(device, env_name, n_actions, n_envs):
    """CartPole: the rows kernel (noise drawn one step ahead on the env threads); GridWorld: rollout_tc_kernel;
    simple_spread: the FFMA rollout_kernel with three agent rows per env."""
    T = 6
    a0, l0 = _device_env_rollout(env_name, n_envs, T, None)
    q = noise_table(T, a0.shape[1], n_actions, SEED, STEP_BASE, ROW_OFFSET * (a0.shape[1] // n_envs))
    a1, l1 = _device_env_rollout(env_name, n_envs, T, q)
    valid = None
    if env_name == "simple_spread":   # the agents of one env share a trajectory: a tie on one agent ends the env's comparison
        env_same = (a0 == a1).reshape(T, n_envs, 3).all(-1)
        env_live = np.cumprod(np.vstack([np.ones((1, n_envs), bool), env_same[:-1]]), 0).astype(bool)
        valid = np.repeat(env_live, 3, axis=1)
    assert_same_draws(a0, l0, a1, l1, q, per_env_trajectory=True, valid=valid)


def test_rng_counter_advances_per_launch(device):
    import torch

    from openrl_b200 import lib

    T = 4
    drv = _driver("CartPole-v1", 64, T)
    drv.rng_counter.zero_()
    for t0, t1 in ((0, 1), (1, 4)):
        lib.check(drv._lib.orl_rollout(drv._rollout_args(t0, t1, None), lib.current_stream()), "orl_rollout")
        torch.cuda.synchronize()
        assert int(drv.rng_counter.item()) == t1, (t0, t1)


def _selfplay_launch(env, params, buf, t_begin, t_end, counter):
    from openrl_b200 import lib

    T, N = buf["act"].shape
    a = lib.OrlRolloutArgs()
    a.env_kind, a.n_envs, a.n_agents, a.episode_length = env.kind, N, 1, T
    a.t_begin, a.t_end, a.obs_dim, a.n_actions, a.activation_id, a.deterministic = t_begin, t_end, 4, 5, 1, 0
    a.policy_params, a.policy_obs = lib.ptr(params), lib.ptr(buf["obs"])
    a.actions, a.action_log_probs, a.rewards = lib.ptr(buf["act"]), lib.ptr(buf["logp"]), lib.ptr(buf["rew"])
    a.masks, a.active_masks = lib.ptr(buf["masks"]), lib.ptr(buf["active"])
    a.rng_seed, a.rng_step_base, a.rng_row_offset, a.rng_counter = SEED, STEP_BASE, ROW_OFFSET, lib.ptr(counter)
    a.env_i32, a.env_table, a.env_table_len = lib.ptr(env.env_i32), lib.ptr(env.env_table), env.env_table_len
    a.ep_return, a.ep_length, a.episode_stats = lib.ptr(env.ep_return), lib.ptr(env.ep_length), lib.ptr(env.episode_stats)
    lib.check(lib.load().orl_selfplay_rollout(env.selfplay_args(a), lib.current_stream()), "orl_selfplay_rollout")


def test_selfplay_learner_noise_key(device):
    """The self-play rollout has no table mode: its learner actions are checked against host argmax(p / q), p from
    orl_policy_eval on the recorded observations, q from the host table (row = env + rng_row_offset, lanes 0 / 1).
    The device counter advances by t_end - t_begin per launch."""
    import torch

    from openrl_b200 import lib
    from openrl_b200.envs.common import make

    N, T, n = 2000, 8, 5
    env = make("GridWorldSelfPlay", env_num=N)
    obs0, _ = env.reset(seed=0)
    z = lambda *sh: torch.zeros(*sh, dtype=torch.float32, device=device)   # noqa: E731
    buf = dict(obs=z(T + 1, N, 4), act=z(T, N), logp=z(T, N), rew=z(T, N), masks=torch.ones(T + 1, N, device=device),
               active=torch.ones(T + 1, N, device=device))
    buf["obs"][0].copy_(torch.from_numpy(obs0[:, 0, :]))
    L = lib.load()
    gen = torch.Generator().manual_seed(7)
    params = (torch.randn(int(L.orl_net_param_count(4, n)), generator=gen) * 0.4).to(device)
    counter = torch.zeros(1, dtype=torch.int64, device=device)
    _selfplay_launch(env, params, buf, 0, T, counter)
    torch.cuda.synchronize()
    assert int(counter.item()) == T

    rows = T * N
    obs = buf["obs"][:T].reshape(rows, 4).contiguous()
    logp_all = np.zeros((rows, n), np.float32)
    ent = torch.empty(rows, 1, dtype=torch.float32, device=device)
    for j in range(n):   # log-prob of every action from the policy itself
        act = torch.full((rows, 1), float(j), device=device)
        lp = torch.empty(rows, 1, dtype=torch.float32, device=device)
        lib.check(L.orl_policy_eval(lib.ptr(params), 4, n, 1, lib.HEAD_CATEGORICAL, lib.ptr(obs), lib.ptr(act), None, lib.ptr(lp),
                                    lib.ptr(ent), rows, lib.current_stream()), "orl_policy_eval")
        torch.cuda.synchronize()
        logp_all[:, j] = lp.cpu().numpy()[:, 0]
    got = buf["act"].cpu().numpy().reshape(rows).astype(np.int64)
    q = noise_table(T, N, n, SEED, STEP_BASE, ROW_OFFSET).reshape(rows, n).astype(np.float64)
    ratio = np.exp(logp_all.astype(np.float64)) / q
    want = ratio.argmax(1)
    r_got, r_want = ratio[np.arange(rows), got], ratio[np.arange(rows), want]
    # policy_eval's forward is a different kernel from the self-play one, so its probabilities differ in the last bits
    tie = np.abs(r_got - r_want) <= 1e-5 * r_want
    assert np.all((got == want) | tie), f"{int(((got != want) & ~tie).sum())} of {rows} learner actions differ"
    assert (got == want).mean() > 0.99
    np.testing.assert_allclose(buf["logp"].cpu().numpy().reshape(rows), logp_all[np.arange(rows), got], rtol=0, atol=1e-5)

    _selfplay_launch(env, params, buf, 2, 5, counter)
    torch.cuda.synchronize()
    assert int(counter.item()) == T + 3
