"""Helpers several test modules share: agents built through the product API, host-stepped stand-in envs, the host
Philox of the device action noise, golden-trace drivers, g++ shims of the device cores and the oracle-trace thread
count.  Not a test module: nothing here is collected."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from openrl_b200 import spaces

# the train_info columns of a recorded update, in the reference's order
KEYS = ["value_loss", "critic_grad_norm", "policy_loss", "dist_entropy", "actor_grad_norm", "ratio"]
# The reference traces were recorded on an 8-core host with torch's default of 8 intra-op threads, and the oracle
# reproduces them bit for bit only under comparable threading: with 1 thread the QR of the orthogonal init differs
# (init parameters off by up to ~2e-7); on a 16-core host running 16 threads the first update's CPU reductions differ
# in their last bits, which moves a continuous action of iteration 1 by one ulp.  Running the oracle with the
# recording count makes these bit-exact checks independent of the host.
TRACE_THREADS = 8
M32 = np.uint64(0xFFFFFFFF)


@pytest.fixture(autouse=True)
def trace_threads():
    """Runs every test of a module that imports it at TRACE_THREADS torch threads."""
    before = torch.get_num_threads()
    torch.set_num_threads(TRACE_THREADS)
    yield
    torch.set_num_threads(before)


# ---------------------------------------------------------------- g++ shims ---------------------------------------------

def gxx_shim(tmp_path_factory, name, source):
    """tests/<source> compiled with g++ against openrl_b200/csrc into a shared library <name>, loaded."""
    out = tmp_path_factory.mktemp(name) / f"lib{name}.so"
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-I", os.path.join(ROOT, "openrl_b200", "csrc"),
                    os.path.join(ROOT, "tests", source), "-o", str(out)], check=True)
    return ctypes.CDLL(str(out))


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


TP_DZ1, TP_DZ3, TP_DZ5, TP_DZ7, TP_DLOG, TP_DV = 0, 64, 128, 192, 256, 264
TQ_X, TQ_Y1, TQ_Y3, TQ_Y5, TQ_Y7 = 272, 336, 400, 464, 528
TS = dict(DY1N1=592, DY1=656, DY3N3=720, DY3=784, DY5N5=848, DY5=912, DY7N7=976, DY7=1040)


def grads_from_tape(tape, d, n):
    g = {}
    P = lambda off, m: tape[:, off:off + m]   # noqa: E731
    g["obs_prep.mlp.fc1.0.weight"] = P(TP_DZ1, 64).T @ P(TQ_X, d)
    g["obs_prep.mlp.fc1.0.bias"] = P(TP_DZ1, 64).sum(0)
    g["obs_prep.mlp.fc1.2.weight"], g["obs_prep.mlp.fc1.2.bias"] = P(TS["DY1N1"], 64).sum(0), P(TS["DY1"], 64).sum(0)
    g["obs_prep.mlp.fc3.0.weight"] = P(TP_DZ3, 64).T @ P(TQ_Y1, 64)
    g["obs_prep.mlp.fc3.0.bias"] = P(TP_DZ3, 64).sum(0)
    g["obs_prep.mlp.fc3.1.weight"], g["obs_prep.mlp.fc3.1.bias"] = P(TS["DY3N3"], 64).sum(0), P(TS["DY3"], 64).sum(0)
    g["common.fc1.0.weight"] = P(TP_DZ5, 64).T @ P(TQ_Y3, 64)
    g["common.fc1.0.bias"] = P(TP_DZ5, 64).sum(0)
    g["common.fc1.2.weight"], g["common.fc1.2.bias"] = P(TS["DY5N5"], 64).sum(0), P(TS["DY5"], 64).sum(0)
    g["common.fc3.0.weight"] = P(TP_DZ7, 64).T @ P(TQ_Y5, 64)
    g["common.fc3.0.bias"] = P(TP_DZ7, 64).sum(0)
    g["common.fc3.1.weight"], g["common.fc3.1.bias"] = P(TS["DY7N7"], 64).sum(0), P(TS["DY7"], 64).sum(0)
    g["v_out.weight"] = P(TP_DV, 1).T @ P(TQ_Y7, 64)
    g["v_out.bias"] = P(TP_DV, 1).sum(0)
    g["act.action_out.linear.weight"] = P(TP_DLOG, n).T @ P(TQ_Y7, 64)
    g["act.action_out.linear.bias"] = P(TP_DLOG, n).sum(0)
    return g


# ---------------------------------------------------------------- agents and envs ---------------------------------------

def make_agent(env, flags, golden=None, like=None, start=True):
    """PPONet and PPOAgent on a ready vec env, under the parsed flags (quiet).
    golden: the reference's initial weights init/<net>.<key>, for each net of the module ("policy" and "critic", or the
      shared "model"); like: {net: state_dict} of weights to start from where golden has none.  A ValueNorm's
      state_dict entries are copies, so its state is never pinned.
    start: run agent.train(total_time_steps=0), which builds the trainer, buffer and driver and resets the envs."""
    from openrl_b200.configs.config import create_config_parser
    from openrl_b200.modules.common import PPONet
    from openrl_b200.runners.common import PPOAgent
    from openrl_b200.utils.logger import Logger

    cfg = create_config_parser().parse_args(flags)
    cfg.quiet = True
    net = PPONet(env, cfg=cfg, device="cuda:0")
    for mk, model in net.module.models.items():
        sd = model.state_dict()
        for k in sd:
            if golden is not None and f"init/{mk}.{k}" in golden and "value_normalizer" not in k:
                sd[k].copy_(torch.from_numpy(golden[f"init/{mk}.{k}"]))
            elif like is not None:
                sd[k].copy_(like[mk][k])
    agent = PPOAgent(net)
    if start:
        agent.train(total_time_steps=0, logger=Logger(quiet=True))
    return cfg, net, agent


def product(env_id, env_num, flags, golden=None, **env_kw):
    """make_agent on a device env from make(), in parity mode, not started: (cfg, env, net, agent)."""
    from openrl_b200.envs.common import make

    env = make(env_id, env_num=env_num, **env_kw)
    cfg, net, agent = make_agent(env, flags + ["--parity_mode", "true", "--log_interval", "1"], golden=golden, start=False)
    return cfg, env, net, agent


class SyntheticHost:
    """BASELINE.md config 5 stand-in (mujoco is absent): obs ~ N(0,1) (N,1,17), reward ~ N(0,1),
    done ~ Bernoulli(1/1000), Box(6) actions."""

    def __init__(self, n, obs_dim=17, act_dim=6, seed=0):
        self.parallel_env_num, self.agent_num = n, 1
        self.observation_space = spaces.Box(-np.inf, np.inf, (obs_dim,), np.float32)
        self.action_space = spaces.Box(-1, 1, (act_dim,), np.float32)
        self.rng = np.random.default_rng(seed)
        self.obs_dim = obs_dim

    def reset(self, seed=None):
        if seed is not None:
            self.rng = np.random.default_rng(seed)
        return self.rng.standard_normal((self.parallel_env_num, 1, self.obs_dim)).astype(np.float32)

    def step(self, actions):
        assert actions.shape == (self.parallel_env_num, 1, 6) and np.isfinite(actions).all()
        n = self.parallel_env_num
        return (self.rng.standard_normal((n, 1, self.obs_dim)).astype(np.float32), self.rng.standard_normal((n, 1, 1)),
                self.rng.random((n, 1)) < 1e-3, [{} for _ in range(n)])


class CountEnv:
    """5-tuple API, episode ends after `horizon` steps; obs = [t, id]."""

    def __init__(self, ident, horizon=3):
        self.observation_space = spaces.Box(-np.inf, np.inf, (2,), np.float32)
        self.action_space = spaces.Discrete(3)
        self.ident, self.horizon, self.t, self.seed_seen, self.tag = ident, horizon, 0, None, "x"
        self.actions = []

    def reset(self, seed=None, options=None):
        self.t = 0
        if seed is not None:
            self.seed_seen = seed
        return np.array([0, self.ident], np.float32), {"reset": True}

    def step(self, a):
        assert isinstance(a, (int, np.integer)) or np.asarray(a).shape == ()
        self.actions.append(int(a))
        self.t += 1
        return np.array([self.t, self.ident], np.float32), float(a), self.t >= self.horizon, False, {"t": self.t}


# ---------------------------------------------------------------- host Philox -------------------------------------------

def philox4x32_10(c0, c1, c2, c3, seed):
    """Philox4x32-10 on uint64 arrays holding 32-bit words (the device's philox4x32_10)."""
    c = [np.asarray(x, np.uint64) & M32 for x in np.broadcast_arrays(c0, c1, c2, c3)]
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64((seed >> 32) & 0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & M32]
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & M32, (k1 + np.uint64(0xBB67AE85)) & M32
    return c


def philox_units(T, rows, seed, step_base, row_offset, lanes):
    """(T, rows, 4 * len(lanes)) float32 uniforms in (0, 1): the four words of each Philox lane in `lanes`, keyed as the
    device's action_philox keys them (step = step_base + t, row = row + row_offset) and mapped by u32_to_unit_open."""
    step = np.uint64(step_base) + np.arange(T, dtype=np.uint64)[:, None]
    row = np.uint64(row_offset) + np.arange(rows, dtype=np.uint64)[None, :]
    words = []
    for lane in lanes:
        words += philox4x32_10(step & M32, step >> np.uint64(32), row, np.uint64(lane), seed)
    u = np.stack(words, -1)
    return ((u >> np.uint64(8)).astype(np.float32) + np.float32(0.5)) * np.float32(1.0 / 16777216.0)


# ---------------------------------------------------------------- golden traces -----------------------------------------

def check_recurrent_trace(tag, env_id, golden_dir=GOLDEN):
    """Drive rollout -> returns -> update by hand for every recorded iteration and compare each stage with the
    unmodified reference's trace (trace_<tag>.npz under golden_dir)."""
    from openrl_b200.utils.logger import Logger

    d = np.load(os.path.join(golden_dir, f"trace_{tag}.npz"), allow_pickle=True)
    iters, N = int(d["meta/iters"]), int(d["meta/env_num"])
    cfg, env, net, agent = product(env_id, N, str(d["meta/flags"]).split(), golden=d)
    agent.train(total_time_steps=0, logger=Logger(quiet=True))   # builds trainer / buffer / driver, resets the envs
    drv = agent.driver
    b = drv.buffer.data
    assert b.rnn_states.shape == d["it0/rnn_states"].shape
    for it in range(iters):
        tag_i = f"it{it}"
        drv.episode = it
        drv.actor_rollout()
        assert np.array_equal(b.actions.cpu().numpy(), d[f"{tag_i}/actions"]), tag_i
        np.testing.assert_allclose(b.action_log_probs.cpu().numpy(), d[f"{tag_i}/action_log_probs"], rtol=0, atol=2e-5)
        np.testing.assert_allclose(b.rnn_states.cpu().numpy(), d[f"{tag_i}/rnn_states"], rtol=0, atol=2e-5)
        assert np.array_equal(b.masks.cpu().numpy(), d[f"{tag_i}/masks"])
        np.testing.assert_allclose(b.policy_obs.cpu().numpy(), d[f"{tag_i}/policy_obs"], rtol=0, atol=2e-6)
        np.testing.assert_allclose(b.rewards.cpu().numpy(), d[f"{tag_i}/rewards"], rtol=1e-6, atol=1e-5)
        drv.compute_returns()
        np.testing.assert_allclose(b.rnn_states_critic.cpu().numpy(), d[f"{tag_i}/rnn_states_critic"], rtol=0, atol=2e-5)
        np.testing.assert_allclose(b.value_preds.cpu().numpy()[:-1], d[f"{tag_i}/value_preds"][:-1], rtol=0, atol=2e-5)
        np.testing.assert_allclose(b.returns.cpu().numpy()[:-1], d[f"{tag_i}/returns"][:-1], rtol=1e-4, atol=2e-4)
        info = drv.trainer.train(b)
        want = d[f"{tag_i}/updates"].mean(axis=0)
        for col, name in enumerate(KEYS):
            np.testing.assert_allclose(info[name], want[col], rtol=2e-4, atol=1e-5, err_msg=f"{tag_i} {name}")
        for mk in ("policy", "critic"):
            for k, v in net.module.models[mk].state_dict().items():
                gk = f"{tag_i}/params/{mk}.{k}"
                if gk in d and "value_normalizer" not in k:
                    np.testing.assert_allclose(v.cpu().numpy(), d[gk], rtol=2e-3, atol=2e-5, err_msg=gk)
        vn = net.module.models["critic"].value_normalizer
        if vn is not None:
            np.testing.assert_allclose(vn.state.cpu().numpy(), d[f"{tag_i}/vn_after_update"], rtol=1e-5, atol=1e-7)
        b.after_update()


def ppo_update_setup(d, flags_extra=()):
    from openrl_b200.algorithms.ppo import PPOAlgorithm
    from openrl_b200.buffers import NormalReplayBuffer

    flags = str(d["meta/flags"]).split() + list(flags_extra)
    cfg, env, net, agent = product("CartPole-v1", int(d["meta/env_num"]), flags, golden=d)
    trainer = PPOAlgorithm(cfg, net.module, agent_num=1, device=net.device)
    buf = NormalReplayBuffer(cfg, 1, env.observation_space, env.action_space, device=net.device)
    return cfg, net, trainer, buf


def load_buffer(buf, d, it):
    b = buf.data
    g = lambda k: torch.from_numpy(d[f"it{it}/{k}"]).cuda()
    b.policy_obs.copy_(g("policy_obs"))
    b.actions.copy_(g("actions"))
    b.action_log_probs.copy_(g("action_log_probs"))
    b.rewards.copy_(g("rewards"))
    b.masks.copy_(g("masks"))
    b.active_masks.copy_(g("active_masks"))
    b.value_preds.copy_(g("value_preds"))
