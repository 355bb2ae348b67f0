"""DiagGaussian head (Box action spaces) and the FFMA row-batch forward against the float64 oracle (oracle/nets.py), at
obs / action widths (17, 6) and (3, 1).

- PPOModule.act (rollout_kernel, ORL_ENV_NONE) at row counts that make orl_rollout pick each of its 8, 16 and 32 rows per
  CTA: with a normal-noise table, deterministic, and with device Philox noise, whose eps = (action - mean) / std must be
  the host Box-Muller of Philox lanes 2..5 (u1 from lanes 2 and 4, u2 from lanes 3 and 5).
- orl_policy_eval with HEAD_GAUSSIAN and orl_critic_values with obs_dim > 8 at 37 rows and at 2 * SMs * 128 + 37 rows,
  where CTAs walk two 128-row tiles and the last tile is partial.

Bars: 1e-5 absolute (the categorical eval bar of test_rollout_rows_cuda.py); deterministic log-probs and the entropies
bit for bit against their float32 closed forms."""
import numpy as np
import pytest

from helpers import philox_units

pytestmark = pytest.mark.gpu

SHAPES = [(17, 6), (3, 1)]
SEED, STEP = 0x2468_ACE0_1357, (1 << 32) + 5
LOG_SQRT_2PI = np.float32(0.9189385332046727)
ENTROPY_CONST = np.float32(1.4189385332046727)   # 0.5 + 0.5 log(2 pi)


def _sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _act_rows(rows_per_cta):
    """orl_rollout wants >= 4 CTAs per SM: 32 rows per CTA from 128 * SMs rows, 16 from 64 * SMs, else 8"""
    sm = _sm_count()
    return {8: 37, 16: 64 * sm + 5, 32: 128 * sm + 37}[rows_per_cta]


def _tile_rows(tiles):
    """grid = min(tiles, 2 * SMs) CTAs of 128 rows"""
    return 37 if tiles == 1 else 2 * _sm_count() * 128 + 37


def _module(d, n):
    import torch

    from openrl_b200 import spaces
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.modules.common import PPONet
    from oracle import loop

    class Env:
        agent_num, parallel_env_num = 1, 1
        observation_space, action_space = spaces.Box(-5, 5, (d,), np.float32), spaces.Box(-1, 1, (n,), np.float32)

        def reset(self, seed=None):
            return np.zeros((1, 1, d), np.float32)

    flags = "--seed 7"
    cfg = create_config_parser().parse_args(flags.split())
    cfg.quiet = True
    module = PPONet(Env(), cfg=cfg, device="cuda:0").module
    sd = module.models["policy"].state_dict()
    sd["act.action_out.fc_mean.weight"].mul_(5.0)   # means of order 0.5
    sd["act.action_out.logstd._bias"].copy_(torch.linspace(-0.5, 0.5, n).view(n, 1))
    return module, loop.cfg_from_flags(flags)


def _params64(model):
    return {k: v.detach().cpu().double() for k, v in model.named_parameters()}


def _logstd(module):
    return module.models["policy"].state_dict()["act.action_out.logstd._bias"].cpu().numpy()[:, 0]


def _obs(rows, d, seed):
    return np.random.default_rng(seed).normal(size=(rows, d)).astype(np.float32)


@pytest.mark.parametrize("rows_per_cta", [8, 16, 32])
@pytest.mark.parametrize("d,n", SHAPES)
def test_act_normal_noise_table_matches_oracle(cuda, d, n, rows_per_cta):
    import torch

    from oracle import nets

    module, ocfg = _module(d, n)
    rows = _act_rows(rows_per_cta)
    obs = _obs(rows, d, rows)
    noise = np.random.default_rng(rows + 1).normal(size=(rows, n)).astype(np.float32)
    act, logp = module.act(obs, exp_noise=noise)
    torch.cuda.synchronize()
    with torch.no_grad():
        want_act, want_logp = nets.policy_act_gaussian(_params64(module.models["policy"]), ocfg, torch.from_numpy(obs).double(),
                                                       normal_noise=torch.from_numpy(noise).double())
    np.testing.assert_allclose(act.cpu().numpy(), want_act.numpy(), rtol=0, atol=1e-5)
    np.testing.assert_allclose(logp.cpu().numpy(), want_logp.numpy(), rtol=0, atol=1e-5)


@pytest.mark.parametrize("d,n", SHAPES)
def test_act_deterministic_is_the_mean(cuda, d, n):
    import torch

    from oracle import nets

    module, ocfg = _module(d, n)
    rows = _act_rows(8)
    obs = _obs(rows, d, 3)
    act, logp = module.act(obs, deterministic=True)
    torch.cuda.synchronize()
    with torch.no_grad():
        mean, _ = nets.policy_act_gaussian(_params64(module.models["policy"]), ocfg, torch.from_numpy(obs).double(),
                                           deterministic=True)
    np.testing.assert_allclose(act.cpu().numpy(), mean.numpy(), rtol=0, atol=1e-5)
    want = np.broadcast_to(-_logstd(module) - LOG_SQRT_2PI, (rows, n))   # float32, as the kernel rounds it
    assert np.array_equal(logp.cpu().numpy().view(np.int32), want.view(np.int32))


@pytest.mark.parametrize("rows_per_cta", [8, 32])
@pytest.mark.parametrize("d,n", SHAPES)
def test_act_philox_noise_is_box_muller_of_lanes_2_to_5(cuda, d, n, rows_per_cta):
    import torch

    module, _ = _module(d, n)
    rows = _act_rows(rows_per_cta)
    obs = _obs(rows, d, 5)
    mean, _ = module.act(obs, deterministic=True)
    act, _ = module.act(obs, rng_seed=SEED, rng_step=STEP)
    torch.cuda.synchronize()
    std = np.exp(_logstd(module).astype(np.float64))
    eps = (act.cpu().numpy().astype(np.float64) - mean.cpu().numpy()) / std
    u = philox_units(1, rows, SEED, STEP, 0, (2, 3, 4, 5))[0].astype(np.float64)   # (rows, 16): lanes 2, 3, 4, 5
    u1 = np.concatenate([u[:, 0:4], u[:, 8:12]], 1)
    u2 = np.concatenate([u[:, 4:8], u[:, 12:16]], 1)
    want = np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)
    np.testing.assert_allclose(eps, want[:, :n], rtol=0, atol=1e-5)


@pytest.mark.parametrize("tiles", [1, 2])
@pytest.mark.parametrize("d,n", SHAPES)
def test_policy_eval_matches_oracle(cuda, d, n, tiles):
    import torch

    from openrl_b200 import lib
    from oracle import nets

    module, ocfg = _module(d, n)
    pol = module.models["policy"]
    rows = _tile_rows(tiles)
    obs = _obs(rows, d, 7)
    p = _params64(pol)
    with torch.no_grad():
        mean, _ = nets.policy_act_gaussian(p, ocfg, torch.from_numpy(obs).double(), deterministic=True)
    # actions one to three standard deviations from the mean
    g = np.random.default_rng(rows)
    actions = (mean.numpy() + np.exp(_logstd(module)) * g.normal(size=(rows, n))).astype(np.float32)
    o, a = torch.from_numpy(obs).to(cuda), torch.from_numpy(actions).to(cuda)
    logp = torch.empty(rows, n, dtype=torch.float32, device=cuda)
    ent = torch.empty(rows, n, dtype=torch.float32, device=cuda)
    lib.check(module._lib.orl_policy_eval(lib.ptr(pol.flat_params), d, n, pol.activation_id, lib.HEAD_GAUSSIAN, lib.ptr(o),
                                          lib.ptr(a), None, lib.ptr(logp), lib.ptr(ent), rows, lib.current_stream()),
              "orl_policy_eval")
    torch.cuda.synchronize()
    with torch.no_grad():
        want_logp, want_ent = nets.policy_eval_gaussian(p, ocfg, torch.from_numpy(obs).double(), torch.from_numpy(actions).double())
    np.testing.assert_allclose(logp.cpu().numpy(), want_logp.numpy(), rtol=0, atol=1e-5)
    want = np.broadcast_to(ENTROPY_CONST + _logstd(module), (rows, n))   # float32, as the kernel rounds it
    got_ent = ent.cpu().numpy()
    assert np.array_equal(got_ent.view(np.int32), want.view(np.int32))
    np.testing.assert_allclose(got_ent.astype(np.float64).mean(), float(want_ent), rtol=1e-6)


@pytest.mark.parametrize("tiles", [1, 2])
@pytest.mark.parametrize("d", [17, 54])
def test_critic_values_matches_oracle(cuda, d, tiles):
    """obs_dim > 8: the FFMA critic forward (obs_dim <= 8 runs the tensor-core one)"""
    import torch

    from oracle import nets

    module, ocfg = _module(d, 1)
    rows = _tile_rows(tiles)
    obs = _obs(rows, d, 11)
    values = module.get_values(obs)
    torch.cuda.synchronize()
    with torch.no_grad():
        want = nets.critic_forward(_params64(module.models["critic"]), ocfg, torch.from_numpy(obs).double())[0]
    np.testing.assert_allclose(values.cpu().numpy(), want.numpy(), rtol=0, atol=1e-5)
