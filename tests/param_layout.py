"""The flat parameter layout the float64 references share: (state_dict name, shape) lists in the order of a kernel's flat
parameter buffer, and the slices and tensors of one such buffer.

TEST INFRASTRUCTURE.  Every 64-wide MLP trunk (orl_mlp.cuh net_offsets, orl_rnn_core.h rnn_offsets, orl_deep_core.h
deep_offsets) is fc1 (linear, LayerNorm) then fc3 (linear, LayerNorm); a head follows it."""
import math

H = 64


def mlp_trunk(d, prefix="base.mlp."):
    """The trunk on d-wide inputs, its names under `prefix`."""
    return [(prefix + "fc1.0.weight", (H, d)), (prefix + "fc1.0.bias", (H,)),
            (prefix + "fc1.2.weight", (H,)), (prefix + "fc1.2.bias", (H,)),
            (prefix + "fc3.0.weight", (H, H)), (prefix + "fc3.0.bias", (H,)),
            (prefix + "fc3.1.weight", (H,)), (prefix + "fc3.1.bias", (H,))]


def head(n, kind):
    """The head of width n on the trunk's H features; kind: "categorical", "gaussian" or "critic"."""
    if kind == "critic":
        return [("v_out.weight", (1, H)), ("v_out.bias", (1,))]
    if kind == "gaussian":
        return [("act.action_out.fc_mean.weight", (n, H)), ("act.action_out.fc_mean.bias", (n,)),
                ("act.action_out.logstd._bias", (n, 1))]
    return [("act.action_out.linear.weight", (n, H)), ("act.action_out.linear.bias", (n,))]


def blocks(shapes):
    """{name: slice of the flat buffer} in flat order."""
    out, off = {}, 0
    for name, shp in shapes:
        k = math.prod(shp)
        out[name] = slice(off, off + k)
        off += k
    return out


def unflatten(flat, shapes):
    """{name: a copy of its block of the flat tensor, in its shape}."""
    return {name: flat[s].reshape(shp).clone() for (name, shp), s in zip(shapes, blocks(shapes).values())}
