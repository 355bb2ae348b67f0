"""The float64 reference of the tensor-core forward passes (tests/fwd_tc_ref64.py) on the CPU: its folded forward, which S,
D and the mutants are built on, is the oracle's forward; its split-fp16 emulation is as close to the exact fc3 product as
the kernels' three passes must be, also where n1's split halves are subnormal (within the floor D); and every forward
mutant moves an output by at least 1e-5 of that output's error scale S.  The GPU test
(tests/test_fwd_tc_scale_cuda.py) measures the kernels in units of S, at a TAU of ~1e-7, so a mutant that moves
an output by 1e-5 S sits well outside it."""
import types

import pytest
import torch

import ffma_ref64
import fwd_tc_ref64 as ref
from oracle import nets

ROWS = 4096


def _net(seed, d, n, head, fc1_scale=1.0):
    """A random_net-style flat vector (tests/scale_harness.py) on the CPU in float64: weights at 1 / sqrt(fan-in) (0.3
    of that in the heads), LayerNorm gains 1 +- 0.2, biases 0.1 N(0, 1); fc1_scale scales fc1's weight and bias."""
    g = torch.Generator().manual_seed(seed)
    parts = []
    for name, shp in ffma_ref64.param_shapes(d, n, head):
        x = torch.randn(shp, generator=g, dtype=torch.float64)
        if len(shp) == 2:
            x *= (0.3 if name.startswith(("act.", "v_out")) else 1.0) / shp[1] ** 0.5
        elif name.endswith("weight"):
            x = 1.0 + 0.2 * x
        else:
            x *= 0.1
        if name.startswith("base.mlp.fc1.0."):
            x *= fc1_scale
        parts.append(x.reshape(-1))
    return torch.cat(parts)


def _obs(seed, d, rows=ROWS):
    return torch.randn(rows, d, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


@pytest.mark.parametrize("activation_id", [0, 1, 2, 3], ids=["tanh", "relu", "leaky_relu", "elu"])
@pytest.mark.parametrize("head,d,n", [("critic", 4, 1), ("critic", 1, 1), ("critic", 8, 1), ("categorical", 4, 2),
                                      ("categorical", 4, 5)])
def test_folded_forward_is_the_oracle(head, d, n, activation_id):
    """The folded forward against the oracle's unfolded one: nets.critic_forward for a critic (ref.forward is that call
    itself), nets.categorical_logits for a Categorical head, of whose log-softmax ref.forward's raw logits must be the
    input.  The LayerNorm gains and biases of a random net are far from 1 and 0, so a wrong fold shows."""
    flat, obs = _net(1, d, n, head), _obs(2, d)
    p = ffma_ref64.unflatten(flat, d, n, head)
    cfg = types.SimpleNamespace(layer_N=1, activation_id=activation_id, use_recurrent_policy=False)
    fo = ref.folded(flat, d, n, head, obs, activation_id)
    if head == "critic":
        want = nets.critic_forward(p, cfg, obs)[0]
        assert _rel(fo["out"], want) <= 1e-12
    else:
        want = nets.categorical_logits(p, nets.mlp_base(p, "base", obs, 1, activation_id))
        assert _rel(ref.forward(flat, d, n, head, obs, activation_id).log_softmax(-1), want) <= 1e-12
        assert _rel(fo["out"].log_softmax(-1), want) <= 1e-12
    assert bool((fo["S"] > 0).all())


def test_split_emulation_is_within_the_three_pass_bound():
    """Each of the three passes is exact in float64; what is left out, Al.Bl, and the roundings of hi and lo are of
    relative size 2^-22 per product, inside 2^-20 A3."""
    flat, obs = _net(3, 4, 1, "critic"), _obs(4, 4)
    p = ref.params(flat, 4, 1, "critic")
    f = ref.fold(p, "critic")
    n1, _, _ = ref._ln(nets.activation(obs @ f["W1"].t() + f["b1"], 1), ref.LN_EPS)
    exact = n1 @ f["W3f"].t()
    emul = ref.fc3_split(n1, f["W3f"])
    A3 = n1.abs() @ f["W3f"].abs().t() + f["b3f"].abs()
    worst = float(((emul - exact).abs() / A3).max())
    hi_only = float(((ref.fc3_split(n1, f["W3f"], ("hh",)) - exact).abs() / A3).max())
    print(f"\n  split emulation: max |emulated - exact| = {worst:.2e} A3 (bound 2^-20 = {2 ** -20:.2e}); Ah.Bh alone "
          f"{hi_only:.2e} A3")
    assert 0 < worst <= 2 ** -20
    assert hi_only > 16 * worst


@pytest.mark.parametrize("activation_id", [0, 1, 2], ids=["tanh", "relu", "leaky_relu"])
@pytest.mark.parametrize("d", [1, 4])
def test_subnormal_floor_bounds_the_emulation_near_zero(d, activation_id):
    """The oracle's initial critic (b1 = 0) on observations from 10^-12 to 10: as they shrink, LayerNorm-1's variance falls
    far below eps and n1's split halves turn subnormal.  Against S alone the emulated split's error then grows without
    bound; within the floor D it stays at the split's relative size."""
    torch.manual_seed(d)
    cfg = types.SimpleNamespace(hidden_size=64, layer_N=1, activation_id=activation_id, use_feature_normalization=False,
                                use_recurrent_policy=False, use_popart=False)
    p = nets.init_critic(cfg, d)
    flat = torch.cat([p[name].reshape(-1) for name, _ in ffma_ref64.param_shapes(d, 1, "critic")]).double()
    scale = torch.logspace(-12, 1, 500, dtype=torch.float64)[:, None]
    obs = torch.cat([scale * _obs(7, d, 500), -scale * _obs(8, d, 500)])
    exact = ref.folded(flat, d, 1, "critic", obs, activation_id)
    err = (ref.folded(flat, d, 1, "critic", obs, activation_id, split=True)["out"] - exact["out"]).abs()
    raw = float((err / exact["S"]).max())
    within = float(((err - exact["D"]).clamp(min=0) / exact["S"]).max())
    print(f"\n  d={d}: emulated split error up to {raw:.2e} S; beyond the floor D {within:.2e} S")
    assert raw > 1e-4 and within <= 2 ** -22


# the nets each mutant needs to show: ln-eps-dropped on fc1 outputs of small spread (var ~ 1e-3), as in the GPU test
MUTANT_NETS = {"fc3-hi-only": {}, "fc3-no-Al": {}, "ln1-bias-fold-dropped": {}, "ln-eps-dropped": dict(fc1_scale=0.055)}


@pytest.mark.parametrize("head,n", [("critic", 1), ("categorical", 2), ("categorical", 5)])
@pytest.mark.parametrize("mutant", ref.FORWARD_MUTANTS)
def test_every_forward_mutant_moves_an_output(mutant, head, n):
    flat, obs = _net(5, 4, n, head, **MUTANT_NETS[mutant]), _obs(6, 4)
    clean = ref.folded(flat, 4, n, head, obs, 1)
    bad = ref.folded(flat, 4, n, head, obs, 1, mutant=mutant)
    moved = float(((bad["out"] - clean["out"]).abs() / clean["S"]).max())
    print(f"\n  {mutant:24s} {head:12s} n={n}: moves an output by {moved:.2e} S")
    assert moved >= 1e-5, (mutant, moved)


def test_row_mutants():
    v = torch.arange(1000, dtype=torch.float64)
    bad, rows = ref.stale_tile(v, 1000, grid=3, cta=1, k=2)
    assert rows.tolist() == list(range(7 * 128, 1000))
    assert torch.equal(bad[rows], v[4 * 128:4 * 128 + rows.numel()])
    assert torch.equal(bad[:7 * 128], v[:7 * 128])
    q = torch.rand(3, 5, 2, dtype=torch.float64)
    s = ref.noise_row_shifted(q)
    assert torch.equal(s[:, :4], q[:, 1:]) and torch.equal(s[:, 4], q[:, 4])
