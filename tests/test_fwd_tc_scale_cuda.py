"""The tensor-core forward passes of orl_fwd_tc.cu at C2 scale against float64, row by row: the critic pass
(`critic_values_tc_kernel`, `orl_critic_values` for observation widths up to 8), the CartPole rollout
(`rollout_cartpole_rows_kernel`, 32 envs per CTA) and the GridWorld rollout (`rollout_tc_kernel`, 128 envs per CTA).

C2 (CartPole, 4096 envs, T = 128) runs a critic pass over (T + 1) x 4096 = 528 384 rows each iteration: on an H100 SXM
its 4128 tiles of 128 rows spread over 2 x 132 CTAs, 15 or 16 per CTA.  Every case runs three nets: the initial nets of
the C2 config, random nets (LayerNorm gains 1 +- 0.2, biases 0.1: a wrong LayerNorm fold shows), and the nets after three
C2 training iterations through PPOAgent.train.  The critic pass runs every activation (ReLU is a compiled-in template;
tanh, LeakyReLU and ELU share the runtime path), the rollouts ReLU, tanh and ELU.

Bars.  The reference is tests/fwd_tc_ref64.py: the oracle's float64 forward and, per row r and output j, the error scale
S_rj of a forward whose fc3 products and head sums are rounded at a relative size e, and the absolute floor D_rj of n1's
subnormal split halves (rows whose LayerNorm-1 variance is far below eps: there the error is no relative one, and err / S
grows without bound as the observation shrinks).
  * Critic values: |v - v64| <= TAU S_r + D_r on every row.
  * Log-probs of the sampled action a: |lp - nl64_a| <= TAU (S_ra + max_j S_rj) + D_ra + max_j D_rj + FLOOR_r,
    FLOOR_r = FLOOR_ULPS float32 ulps of (1 + |log-sum-exp|), for the kernel's own log-softmax.  The float64 logits are
    computed on the recorded observations, so a near-tie never makes the trajectories part.
  * Actions: a == argmax_j p64_j / q_j (first index wins; argmax p64 when deterministic), q the Exp(1) noise: the host
    table the kernel read, or the device Philox draws rebuilt on the host (tests/helpers.py philox_units).  The only
    exception is a near-tie, where the float64 log-ratio margin between the kernel's pick and the float64 argmax is at
    most TAU (S_ra + S_r,argmax) + D_ra + D_r,argmax + 2 FLOOR_r (+ 2^-21 with Philox noise, whose host and device -log may differ in the last
    bit).  Near-ties must stay under NEAR_TIE_SHARE of the rows.
Without a bar: a permuted observation array gives exactly the permuted values (a row's value does not depend on its tile,
CTA or place in the tile), observation rows past `rows` set to NaN change nothing and the values past `rows` stay
untouched; the GridWorld rollout's observations, rewards and masks are bit-exact against oracle.envs.GridWorldVec
stepped with the kernel's actions from a reset table.

TAU and the mutants.  TAU is measured on an H100 (see its comment).  Each mutant of tests/fwd_tc_ref64.py is shown to be
caught; measured on the H100, in units of TAU (the worst row's error beyond the floors, against the mutant), for the
initial / random / trained net with ReLU:
  * C2 critic buffer: fc3-hi-only 519 / 538 / 402, fc3-no-Al 477 / 386 / 350, ln1-bias-fold-dropped - / 1.0e5 / 3300
    (the initial net's be1 is 0), stale-tile (CTA 0's 16th tile) 9e5 or more.  The checks ask for >= 2 TAU (stale-tile:
    outside the bar).
  * C2 rollout log-probs, CartPole / GridWorld: fc3-hi-only 159 / 188 / 211 and 113 / 144 / 134, fc3-no-Al 112 / 130 /
    183 and 85 / 110 / 117, ln1-bias-fold-dropped - / 11700 / 4760 and - / 21200 / 1390; >= 2 TAU asked.
  * ln-eps-dropped (printed): 148 / 30 / 2210 on the C2 critic buffer, 15 / 12 / 4460 on the CartPole rollout, below 1 on
    GridWorld's; on fc1 outputs of small spread (var ~ 1e-3) 4000 (ReLU) and 290 (tanh), where it must reach 2 TAU.
  * noise-row-shifted: 47 % (CartPole) and 79 % (GridWorld) of the C2 rollout's actions fail the action check, none with
    the right noise.

LayerNorm statistics.  The kernels compute a LayerNorm's variance in one pass, as E[x^2] - mu^2 in float32, which loses
digits as |mu| / sigma of the row grows.  The C2 runs reach LN1 |mu| / sigma 1.03 and LN3 0.38 (printed); a synthetic
critic case puts LN1 at 4x that (4.1, from an fc1 bias offset), where the kernel measured 2.3e-8 S, inside TAU: no limit
of the one-pass statistics shows at these ratios.

Small n1.  The floor D is what keeps rows near zero inside the bar: the width test scales 128 rows down to 10^-10, which
with an initial net (b1 = 0) puts LayerNorm-1's variance far below eps and n1 far below fp16's normal range.  Against S
alone such rows reach any err / S (the split's absolute error of 2^-25 per element against an n1 that shrinks with the
observation); beyond D they stay at the level of every other row."""
import types

import numpy as np
import pytest
import torch

import ffma_ref64
import fwd_tc_ref64 as ref
from helpers import philox_units
from scale_harness import no_tf32, random_net, rel  # noqa: F401  (no_tf32: pytest fixture)

pytestmark = pytest.mark.gpu

# TAU, measured on an H100 SXM (NVIDIA H100 80GB HBM3, 132 SMs, 700 W power limit; 264 CTAs in the critic pass): the
# worst kernel error beyond the floors is 4.5e-8 S, in the critic pass at observation width 8 (trained net, ELU, one row
# past a full wave); C2's 528 384 rows reach 3.7e-8 (trained net, tanh), width 1 (whose test scales rows towards 0) 3.5e-8, and
# the rollouts' log-prob errors all lie inside their float32 floor.  TAU is that worst value x 1.57.
TAU = 7e-8
FLOOR_ULPS = 4
NEAR_TIE_SHARE = 1e-4
T, C2_ENVS, T_M = 128, 4096, 128
C2_ROWS = (T + 1) * C2_ENVS   # the critic pass of one C2 iteration: 528 384 rows
FLAGS = ["--seed", "0", "--episode_length", str(T), "--ppo_epoch", "4", "--num_mini_batch", "1", "--log_interval", "1000000",
         "--log_each_episode", "false"]
ACTS = {"tanh": 0, "relu": 1, "leaky_relu": 2, "elu": 3}
ROLLOUT_ACTS = ("relu", "tanh", "elu")
NETS = ("init", "random", "trained")
SEED, STEP_BASE, ROW_OFFSET = 0x1234_5678_9ABC, (1 << 32) + 77, 1000


@pytest.fixture(autouse=True)
def _needs_cuda(cuda):
    pass


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def noise_table(T_, rows, n, seed, step_base, row_offset):
    """(T, rows, n) float32 Exp(1) noise as the device keys it (step = step_base + t, row = row + row_offset)."""
    return (-np.log(philox_units(T_, rows, seed, step_base, row_offset, (0, 1))[..., :n])).astype(np.float32)


class Worst:
    """The worst err/S of a test's cases, printed per case and at the end."""

    def __init__(self, name):
        self.name, self.val, self.where, self.bad = name, 0.0, "", []

    def add(self, case, es, extra=""):
        print(f"  {self.name} {case:56s} worst err/S {es:9.2e} = {es / TAU:5.2f} TAU {extra}")
        if es > self.val:
            self.val, self.where = es, case
        if not es <= TAU:
            self.bad.append(f"{case}: err/S {es:.3e} > TAU {TAU:.1e}")

    def done(self):
        print(f"  {self.name}: worst err/S {self.val:.2e} = {self.val / TAU:.2f} TAU ({self.where})")
        assert not self.bad, "\n".join(self.bad)


# ---------------------------------------------------------------- nets ------------------------------------------------

def _trained_agent(env_id):
    """The C2 config on `env_id` with 4096 envs: its initial nets, its nets after three PPOAgent.train iterations, and the
    agent, whose buffer then holds the critic observations of a rollout by the trained policy."""
    from helpers import make_agent
    from openrl_b200.envs.common import make
    from openrl_b200.utils.logger import Logger

    torch.manual_seed(0)
    _, _, agent = make_agent(make(env_id, env_num=C2_ENVS), FLAGS)
    m = agent.driver.trainer.algo_module
    flat = lambda: {k: m.models[mk].flat_params.detach().clone() for k, mk in (("pol", "policy"), ("cri", "critic"))}  # noqa: E731
    init = flat()
    agent.train(total_time_steps=3 * T * C2_ENVS, logger=Logger(quiet=True))
    trained = flat()
    assert not torch.equal(init["pol"], trained["pol"]) and not torch.equal(init["cri"], trained["cri"])
    agent.driver.actor_rollout()
    torch.cuda.synchronize()
    return init, trained, agent


@pytest.fixture(scope="module")
def c2():
    init, trained, agent = _trained_agent("CartPole-v1")
    obs = agent.driver.buffer.data.critic_obs.reshape(-1, 4).clone()
    assert obs.shape[0] == C2_ROWS
    g = torch.Generator(device="cuda").manual_seed(21)
    nets = {"pol": dict(init=init["pol"], trained=trained["pol"], random=random_net(g, ffma_ref64.param_shapes(4, 2, "categorical"))),
            "cri": dict(init=init["cri"], trained=trained["cri"], random=random_net(g, ffma_ref64.param_shapes(4, 1, "critic")))}
    # the largest LayerNorm |mu| / sigma of the C2 forwards (critic and policy over the C2 observations, ReLU)
    ms = [0.0, 0.0]
    for key, n, head in (("cri", 1, "critic"), ("pol", 2, "categorical")):
        for name in NETS:
            r = ref.folded(nets[key][name], 4, n, head, obs, 1)
            ms = [max(ms[0], float(r["mu_sigma1"].max())), max(ms[1], float(r["mu_sigma3"].max()))]
    print(f"\n  C2 nets: largest LN1 |mu|/sigma {ms[0]:.2f}, LN3 {ms[1]:.2f} (C2 critic buffer)")
    yield types.SimpleNamespace(obs=obs, nets=nets, mu_sigma=ms)
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def grid_nets():
    init, trained, _ = _trained_agent("GridWorldEnv")
    g = torch.Generator(device="cuda").manual_seed(22)
    return dict(init=init["pol"], trained=trained["pol"], random=random_net(g, ffma_ref64.param_shapes(4, 5, "categorical")))


def _width_nets(c2, d):
    """Critic nets of observation width d: the C2 nets for d = 4; otherwise the oracle's initial critic of width d, a
    random net, and the trained C2 critic with its fc1 columns repeated over the d inputs (scaled by sqrt(4 / d))."""
    if d == 4:
        return c2.nets["cri"]
    from oracle import nets

    shapes = ffma_ref64.param_shapes(d, 1, "critic")
    torch.manual_seed(d)
    cfg = types.SimpleNamespace(hidden_size=64, layer_N=1, activation_id=1, use_feature_normalization=False,
                                use_recurrent_policy=False, use_popart=False)
    init = nets.init_critic(cfg, d)
    p = ffma_ref64.unflatten(c2.nets["cri"]["trained"], 4, 1, "critic")
    p["base.mlp.fc1.0.weight"] = p["base.mlp.fc1.0.weight"][:, [k % 4 for k in range(d)]] * (4 / d) ** 0.5
    flat = lambda q: torch.cat([q[name].reshape(-1) for name, _ in shapes]).float().cuda()  # noqa: E731
    g = torch.Generator(device="cuda").manual_seed(100 + d)
    return dict(init=flat(init), random=random_net(g, shapes), trained=flat(p))


# ---------------------------------------------------------------- the critic pass -------------------------------------

def _values(flat, d, act_id, obs, rows, out=None):
    from openrl_b200 import lib

    v = torch.empty(rows, device="cuda") if out is None else out
    lib.check(lib.load().orl_critic_values(lib.ptr(flat), d, act_id, lib.ptr(obs), lib.ptr(v), rows, lib.current_stream()),
              "orl_critic_values")
    torch.cuda.synchronize()
    return v


def excess(err, S, D):
    """max over rows of (err - D) / S where err exceeds the subnormal floor D: the error in units of S that TAU bounds."""
    over = (err - D).clamp(min=0)
    return float(torch.where(over > 0, over / S, torch.zeros_like(over)).max())


def _critic_err(flat, d, act_id, obs, v, r=None):
    r = r or ref.reference(flat, d, 1, "critic", obs, act_id)
    return excess((v.double() - r["out"][:, 0]).abs(), r["S"][:, 0], r["D"][:, 0]), r


def _vs_critic_mutant(v, vm, r):
    """Where the kernel's values sit against a mutant's, in units of TAU (worst row)."""
    return excess((v.double() - vm).abs(), r["S"][:, 0], r["D"][:, 0]) / TAU


def _grid():
    return 2 * _sms()


def _row_count(label):
    G = _grid()
    return {"1": 1, "127": 127, "128": 128, "129": 129, "128G-1": 128 * G - 1, "128G": 128 * G, "128G+1": 128 * G + 1,
            "c2": C2_ROWS, "c2+37": C2_ROWS + 37}[label]


def _c2_obs(c2, rows):
    """The first `rows` rows of the C2 critic buffer, N(0, 1) rows past its end."""
    if rows <= C2_ROWS:
        return c2.obs[:rows].contiguous()
    g = torch.Generator(device="cuda").manual_seed(rows)
    return torch.cat([c2.obs, torch.randn(rows - C2_ROWS, 4, generator=g, device="cuda")])


ROW_LABELS = ["1", "127", "128", "129", "128G-1", "128G", "128G+1", "c2", "c2+37"]


@pytest.mark.parametrize("label", ROW_LABELS)
def test_critic_row_counts(c2, no_tf32, label):
    """The C2 critic observations over row counts at the edges of a tile, of one wave of 2 x SMs CTAs and of C2's
    528 384 rows (4128 tiles, 15 or 16 per CTA on 264 CTAs)."""
    rows = _row_count(label)
    tiles = -(-rows // T_M)
    G = min(tiles, _grid())
    if label.startswith("c2"):
        assert tiles // G >= 15, (tiles, G)
    obs = _c2_obs(c2, rows)
    w = Worst(f"critic rows={rows} ({tiles} tiles, G={G})")
    for net in NETS:
        for act, act_id in ACTS.items():
            flat = c2.nets["cri"][net]
            v = _values(flat, 4, act_id, obs, rows)
            es, r = _critic_err(flat, 4, act_id, obs, v)
            w.add(f"{net}/{act}", es, f"rel L2 {rel(v, r['out'][:, 0]):.2e}")
    w.done()


@pytest.mark.parametrize("d", [1, 3, 4, 5, 8])
def test_critic_obs_widths(c2, no_tf32, d):
    """N(0, 1) observations of width d (fc1's K zero-padded to 8), at 129 rows and one row past a full wave.  Their first
    128 rows are scaled down by 10^0 ... 10^-10: with an initial net (b1 = 0) such rows have a LayerNorm-1 variance far
    below eps and subnormal split halves of n1, which the floor D bounds (tests/fwd_tc_ref64.py)."""
    nets = _width_nets(c2, d)
    w = Worst(f"critic d={d}")
    for rows in (129, 128 * _grid() + 1):
        obs = torch.randn(rows, d, generator=torch.Generator(device="cuda").manual_seed(rows + d), device="cuda")
        obs[:T_M] *= torch.logspace(0, -10, T_M, device="cuda")[:, None]
        for net in NETS:
            for act, act_id in ACTS.items():
                v = _values(nets[net], d, act_id, obs, rows)
                es, _ = _critic_err(nets[net], d, act_id, obs, v)
                w.add(f"rows={rows} {net}/{act}", es)
    w.done()


@pytest.mark.parametrize("label", ["129", "128G+1", "c2+37"])
def test_critic_rows_are_independent_of_their_place(c2, label):
    """Values of a permuted observation array are exactly the permuted values; NaN observation rows past `rows` change
    nothing, and the values buffer past `rows` keeps its sentinel."""
    rows = _row_count(label)
    obs = _c2_obs(c2, rows)
    perm = torch.randperm(rows, generator=torch.Generator(device="cuda").manual_seed(5), device="cuda")
    pad = 2 * T_M + 3
    poisoned = torch.cat([obs, torch.full((pad, 4), float("nan"), device="cuda")])
    for net in ("random", "trained"):
        for act in ("relu", "tanh"):
            flat = c2.nets["cri"][net]
            v = _values(flat, 4, ACTS[act], obs, rows)
            vp = _values(flat, 4, ACTS[act], obs[perm].contiguous(), rows)
            assert torch.equal(vp, v[perm]), (net, act, int((vp != v[perm]).sum()))
            out = torch.full((rows + pad,), -12345.0, device="cuda")
            _values(flat, 4, ACTS[act], poisoned, rows, out)
            assert torch.equal(out[:rows], v), (net, act)
            assert bool((out[rows:] == -12345.0).all()), (net, act)


def _mutant_sizes(v, flat, obs, act_id, r):
    """{mutant: worst |v - v_mutant| / S in units of TAU} for the forward mutants."""
    out = {}
    for m in ref.FORWARD_MUTANTS:
        out[m] = _vs_critic_mutant(v, ref.folded(flat, 4, 1, "critic", obs, act_id, mutant=m)["out"][:, 0], r)
    return out


def test_critic_mutants_are_caught_on_c2(c2, no_tf32):
    obs, G = c2.obs, _grid()
    bad = []
    for net in NETS:
        flat = c2.nets["cri"][net]
        v = _values(flat, 4, 1, obs, C2_ROWS)
        es, r = _critic_err(flat, 4, 1, obs, v)
        sizes = _mutant_sizes(v, flat, obs, 1, r)
        # stale-tile: the last tile of CTA 0 (its 16th) carries its 15th tile's values
        k = (-(-C2_ROWS // T_M) - 1) // G
        vm, changed = ref.stale_tile(r["out"][:, 0], C2_ROWS, G, 0, k)
        sizes["stale-tile"] = _vs_critic_mutant(v, vm, r)
        print(f"  c2 critic {net:8s} kernel {es / TAU:.2f} TAU; against the mutants: "
              + ", ".join(f"{m} {s:.1f} TAU" for m, s in sizes.items()))
        need = ["fc3-hi-only", "fc3-no-Al", "stale-tile"] + (["ln1-bias-fold-dropped"] if net != "init" else [])
        bad += [f"{net}: {m} at {sizes[m]:.2f} TAU" for m in need if not sizes[m] >= (2.0 if m != "stale-tile" else 1.0)]
    assert not bad, bad


def test_critic_ln_eps_small_spread(c2, no_tf32):
    """fc1 outputs of small spread (random net, fc1 weight and bias x 0.055: var ~ 1e-3), where LayerNorm-1's eps is 1 %
    of the variance: the kernel stays within TAU, and the mutant without eps is caught."""
    g = torch.Generator(device="cuda").manual_seed(31)
    flat = random_net(g, ffma_ref64.param_shapes(4, 1, "critic"))
    s = ffma_ref64.blocks(4, 1, "critic")
    flat[s["base.mlp.fc1.0.weight"]] *= 0.055
    flat[s["base.mlp.fc1.0.bias"]] *= 0.055
    rows = 128 * _grid() + 1
    obs = torch.randn(rows, 4, generator=g, device="cuda")
    w = Worst("critic small fc1 spread")
    for act in ("relu", "tanh"):
        v = _values(flat, 4, ACTS[act], obs, rows)
        es, r = _critic_err(flat, 4, ACTS[act], obs, v)
        p = ref.params(flat, 4, 1, "critic")
        var1 = torch.relu(obs.double() @ p["base.mlp.fc1.0.weight"].t() + p["base.mlp.fc1.0.bias"]).var(-1).median()
        eps_m = ref.folded(flat, 4, 1, "critic", obs, ACTS[act], mutant="ln-eps-dropped")["out"][:, 0]
        caught = _vs_critic_mutant(v, eps_m, r)
        w.add(act, es, f"(median fc1 var {float(var1):.1e}); ln-eps-dropped at {caught:.1f} TAU")
        assert caught >= 2.0, (act, caught)
    w.done()


def test_critic_ln1_far_from_zero(c2, no_tf32):
    """LN1 rows at 4x the largest |mu| / sigma of the C2 runs, from an fc1 bias offset on a random net (ReLU)."""
    target = 4 * c2.mu_sigma[0]
    g = torch.Generator(device="cuda").manual_seed(41)
    base = random_net(g, ffma_ref64.param_shapes(4, 1, "critic"))
    sb = ffma_ref64.blocks(4, 1, "critic")["base.mlp.fc1.0.bias"]
    rows = 128 * _grid() + 1
    obs = torch.randn(rows, 4, generator=g, device="cuda")
    c = 1.0
    for _ in range(8):   # rescale the offset by target / reached until the largest ratio is on target
        flat = base.clone()
        flat[sb] += c
        got = float(ref.folded(flat, 4, 1, "critic", obs, 1)["mu_sigma1"].max())
        if abs(got / target - 1) < 0.01:
            break
        c *= target / got
    v = _values(flat, 4, 1, obs, rows)
    es, r = _critic_err(flat, 4, 1, obs, v)
    assert abs(float(r["mu_sigma1"].max()) / target - 1) < 0.01, (float(r["mu_sigma1"].max()), target)
    w = Worst("critic LN1 far from zero")
    w.add(f"LN1 |mu|/sigma up to {float(r['mu_sigma1'].max()):.1f} (C2 max {c2.mu_sigma[0]:.2f}, offset {c:.2f})", es)
    w.done()


# ---------------------------------------------------------------- the rollouts ----------------------------------------

_DRIVERS = {}


def _driver(env_id, n_envs, **env_kw):
    """A started agent's driver for `env_id` with n_envs envs (cached unless env_kw are given)."""
    from helpers import make_agent
    from openrl_b200.envs.common import make

    key = (env_id, n_envs)
    if env_kw or key not in _DRIVERS:
        _, _, agent = make_agent(make(env_id, env_num=n_envs, **env_kw), FLAGS)
        if env_kw:
            return agent.driver
        _DRIVERS[key] = agent.driver
    return _DRIVERS[key]


def _rollout(drv, flat, act_id, mode, table=None):
    """One launch over [0, T) with the given policy; the recorded (obs, actions, log-probs) as (T N, ...) rows."""
    from openrl_b200 import lib

    b = drv.buffer.data
    a = drv._rollout_args(0, T, table if mode == "table" else None)
    a.policy_params, a.activation_id, a.deterministic = lib.ptr(flat), act_id, int(mode == "deterministic")
    a.rng_seed, a.rng_step_base, a.rng_counter, a.rng_row_offset = SEED, STEP_BASE, None, ROW_OFFSET
    lib.check(drv._lib.orl_rollout(a, lib.current_stream()), "orl_rollout")
    torch.cuda.synchronize()
    N = drv.envs.parallel_env_num
    out = dict(obs=b.policy_obs[:T].reshape(T * N, 4).clone(), act=b.actions[:T].reshape(T * N).clone(),
               lp=b.action_log_probs[:T].reshape(T * N).clone(), all_obs=b.policy_obs.reshape(T + 1, N, 4).clone(),
               rewards=b.rewards.reshape(T, N).clone(), masks=b.masks.reshape(T + 1, N).clone())
    b.after_update()
    return out


def _check_rollout(flat, n, act_id, run, q, mode, mutant=None):
    """Log-probs and actions of one rollout against the float64 forward of its recorded observations (against a forward
    mutant's logits, with the clean forward's S and D, when `mutant` is given)."""
    r = ref.reference(flat, 4, n, "categorical", run["obs"], act_id)
    S, D = r["S"], r["D"]
    l64 = r["out"] if mutant is None else ref.folded(flat, 4, n, "categorical", run["obs"], act_id, mutant=mutant)["out"]
    lse = l64.logsumexp(-1)
    nl = l64 - lse[:, None]
    floor = FLOOR_ULPS * 2.0 ** -24 * (1 + lse.abs())
    a = run["act"].long()
    assert bool(((a >= 0) & (a < n)).all())
    pick = lambda x, i: x.gather(1, i[:, None])[:, 0]   # noqa: E731
    sa, smax = pick(S, a), S.max(-1).values
    fa = floor + pick(D, a) + D.max(-1).values
    err = (run["lp"].double() - pick(nl, a)).abs()
    es = excess(err, sa + smax, fa)
    lp_bar = TAU * (sa + smax) + fa
    lp_bad = int((err > lp_bar).sum())
    score = nl if mode == "deterministic" else nl - q.double().log()
    want = score.argmax(-1)
    margin = pick(score, want) - pick(score, a)
    tie_bar = (TAU * (sa + pick(S, want)) + pick(D, a) + pick(D, want) + 2 * floor
               + (2.0 ** -21 if mode == "philox" else 0.0))
    differ = want != a
    ties, wrong = int((differ & (margin <= tie_bar)).sum()), int((differ & (margin > tie_bar)).sum())
    return dict(es=es, of_bar=float((err / lp_bar).max()), lp_bad=lp_bad, ties=ties, wrong=wrong, rows=a.numel(),
                ms1=float(r["mu_sigma1"].max()),
                ms3=float(r["mu_sigma3"].max()))


_Q = {}


def _noise(N, n, mode):
    """(T, N, n) noise on the device: the table a table-mode run reads, or the host rebuild of the device Philox draws."""
    key = (N, n, mode)
    if key not in _Q:
        q = (noise_table(T, N, n, SEED, STEP_BASE, ROW_OFFSET) if mode == "philox"
             else noise_table(T, N, n, SEED + 1, 3, 0))
        _Q[key] = torch.from_numpy(q).cuda()
    return _Q[key]


def _rollout_case(env_id, n, nets, n_envs, mode):
    drv = _driver(env_id, n_envs)
    q = None if mode == "deterministic" else _noise(n_envs, n, mode)
    w = Worst(f"{env_id} N={n_envs} {mode}")
    bad, ms = [], [0.0, 0.0]
    for net in NETS:
        for act in ROLLOUT_ACTS:
            run = _rollout(drv, nets[net], ACTS[act], mode, q)
            c = _check_rollout(nets[net], n, ACTS[act], run, None if q is None else q.reshape(T * n_envs, n), mode)
            w.add(f"{net}/{act}", c["es"], f"log-probs at {c['of_bar']:.2f} of their bar, near-ties {c['ties']} of "
                                           f"{c['rows']}, LN1/LN3 |mu|/sigma "
                                           f"{c['ms1']:.2f}/{c['ms3']:.2f}")
            if c["lp_bad"] or c["wrong"] or c["ties"] > NEAR_TIE_SHARE * c["rows"]:
                bad.append(f"{net}/{act}: {c['lp_bad']} log-probs off the bar, {c['wrong']} wrong actions, "
                           f"{c['ties']} near-ties")
    w.done()
    assert not bad, bad


MODES = ["table", "philox", "deterministic"]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("n_envs", [C2_ENVS, C2_ENVS + 17, 20])
def test_cartpole_rollout(c2, no_tf32, n_envs, mode):
    _rollout_case("CartPole-v1", 2, c2.nets["pol"], n_envs, mode)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("n_envs", [C2_ENVS, C2_ENVS + 17, 20])
def test_gridworld_rollout(grid_nets, no_tf32, n_envs, mode):
    _rollout_case("GridWorldEnv", 5, grid_nets, n_envs, mode)


@pytest.mark.parametrize("n_envs", [C2_ENVS, C2_ENVS + 17, 20])
def test_gridworld_env_matches_oracle(grid_nets, n_envs):
    """The fused GridWorld rollout's observations, rewards and masks against oracle.envs.GridWorldVec stepped with the
    kernel's actions, both resetting from the same per-env table."""
    from oracle.envs import GridWorldVec

    K = 8
    rng = np.random.default_rng(n_envs)
    table = rng.integers(0, 10, size=(n_envs, K, 2))
    goal = (table == 1).all(-1)
    table[goal] = [5, 5]

    class PerEnvTable(GridWorldVec):
        def __init__(self, n, table):
            super().__init__(n)
            self.table, self.count = table, np.zeros(n, np.int64)

        def _reset_one(self, i):
            self.steps[i] = 0
            self.pos[i] = self.table[i, min(self.count[i], K - 1)]
            self.count[i] += 1

    drv = _driver("GridWorldEnv", n_envs, reset_table=table)
    run = _rollout(drv, grid_nets["trained"], 1, "philox")
    # starting an agent resets its envs, maybe more than once: the oracle starts from the table entry slot 0 shows
    start = run["all_obs"][0].cpu().numpy()
    used = [k for k in range(K) if np.array_equal(start[:, :2], table[:, k].astype(np.float32))]
    assert used, "slot 0 holds no reset of the table"
    oracle = PerEnvTable(n_envs, table)
    oracle.reset()
    oracle.pos[:], oracle.count[:] = table[:, used[0]], used[0] + 1
    assert np.array_equal(start, oracle._obs()[:, 0].astype(np.float32))
    acts = run["act"].reshape(T, n_envs).cpu().numpy().astype(np.int64)
    all_obs, rew, masks = run["all_obs"].cpu().numpy(), run["rewards"].cpu().numpy(), run["masks"].cpu().numpy()
    resets = 0
    for t in range(T):
        o, r, d, _ = oracle.step(acts[t][:, None, None])
        assert np.array_equal(all_obs[t + 1], o[:, 0].astype(np.float32)), t
        assert np.array_equal(rew[t], r[:, 0, 0].astype(np.float32)), t
        assert np.array_equal(masks[t + 1], (~d[:, 0]).astype(np.float32)), t
        resets += int(d.sum())
    c = _check_rollout(grid_nets["trained"], 5, 1, run, _noise(n_envs, 5, "philox").reshape(T * n_envs, 5), "philox")
    print(f"  GridWorld N={n_envs}: {resets} resets, err/S {c['es']:.2e}, near-ties {c['ties']}")
    assert resets > 0 and c["lp_bad"] == 0 and c["wrong"] == 0


@pytest.mark.parametrize("env_id,n", [("CartPole-v1", 2), ("GridWorldEnv", 5)])
def test_rollout_mutants_are_caught(c2, grid_nets, env_id, n):
    """A C2-sized rollout (ReLU, Philox noise) against the mutants: the log-probs' bar against the forward mutants' logits
    (fc3-hi-only, fc3-no-Al and ln1-bias-fold-dropped at >= 2 TAU on the random and trained nets; ln-eps-dropped printed),
    the action check against the noise of the next row."""
    nets = c2.nets["pol"] if env_id == "CartPole-v1" else grid_nets
    drv = _driver(env_id, C2_ENVS)
    q = _noise(C2_ENVS, n, "philox").reshape(-1, n)
    qs = ref.noise_row_shifted(_noise(C2_ENVS, n, "philox")).reshape(-1, n)
    bad = []
    for net in NETS:
        run = _rollout(drv, nets[net], 1, "philox")
        ok = _check_rollout(nets[net], n, 1, run, q, "philox")
        shifted = _check_rollout(nets[net], n, 1, run, qs, "philox")
        sizes = {m: _check_rollout(nets[net], n, 1, run, q, "philox", mutant=m)["es"] / TAU for m in ref.FORWARD_MUTANTS}
        print(f"  {env_id} {net:8s} log-probs {ok['es'] / TAU:.2f} TAU; against the mutants: "
              + ", ".join(f"{m} {s:.1f} TAU" for m, s in sizes.items())
              + f"; wrong actions {ok['wrong']} with the right noise, {shifted['wrong']} of {shifted['rows']} with the "
              f"next row's")
        need = ["fc3-hi-only", "fc3-no-Al", "ln1-bias-fold-dropped"] if net != "init" else []
        bad += [f"{net}: {m} at {sizes[m]:.2f} TAU" for m in need if not sizes[m] >= 2.0]
        if not (ok["wrong"] == 0 and shifted["wrong"] > 0.1 * shifted["rows"]):
            bad.append(f"{net}: noise-row-shifted, {ok['wrong']} / {shifted['wrong']} wrong actions")
    assert not bad, bad
