// Sequential (one row at a time) restatement of the SHARED policy-value network of cfg.use_share_model
// (reference: PolicyValueNetwork, openrl/modules/networks/policy_value_network.py:33-174), compiled BOTH by nvcc
// (device functions used by orl_share.cu, one thread per row) and by g++ (tests/test_deep_core_cpu.py drives it through a
// C shim and checks forward, backward and every parameter gradient against torch autograd of the oracle).
//
// Network:  x(d) -> obs_prep = MLPBase: fc1 -> act -> LN1 -> fc3 -> LN3          (mlp.py:100-176, layer_N = 1)
//                -> common   = MLPLayer(64, 64, layer_N = 0): fc5 -> act -> LN5 -> fc7 -> LN7   (mlp.py:8-46)
//                -> { v_out: Linear(64, 1),  act: Categorical linear / DiagGaussian fc_mean Linear(64, n) }
// Flat parameter layout (named_parameters order of the reference; `critic_obs_prep` aliases `obs_prep`):
//   W1[64][d] b1 g1 be1 | W3[64][64] b3 g3 be3 | W5[64][64] b5 g5 be5 | W7[64][64] b7 g7 be7 | Wv[1][64] bv | Wa[n][64] ba
//   and, for a DiagGaussian head (Box(n) actions), logstd[n] (act.action_out.logstd._bias, shape (n, 1)) after ba.
// The head output is the logits of a Categorical head and the mean of a DiagGaussian one; the dL/dlogstd of a row is
// the loss's business (orl_loss.cuh gaussian_row), kept in the tape field TS_DLS of the Gaussian tape.
// The backward writes a per-row "tape" of local gradients and forward activations; the parameter gradients are tape
// reductions dW = sum_rows P^T Q / column sums, done by orl::reduce_tape (orl_tape.cu).
// The widths, activations, LayerNorm and the obs_prep trunk are those of the recurrent core (orl_rnn_core.h).
#pragma once
#include "orl_rnn_core.h"

#ifdef __CUDACC__
// Real calls on the device (own stack frames): with a whole sequential step inlined into its kernel, nvcc 12.9 once
// merged the stack slots of the caller's observation row and the callee's outputs (observed in SASS as a corrupted
// tape of the recurrent core), i.e. wrong gradients.  `inline`: one definition however many files include this header.
#define ORLD_STEP inline __host__ __device__ __noinline__
#else
#define ORLD_STEP static inline
#endif

namespace orl_deep {

using orl_rnn::H;
using orl_rnn::MAXN;
using orl_rnn::MAXD;
using orl_rnn::act_fwd;
using orl_rnn::act_bwd_from_out;
using orl_rnn::layernorm64;
using orl_rnn::layernorm64_bwd;
using orl_rnn::linear64;
using orl_rnn::linear64_bwd_data;

struct Offsets {
    int d, n;
    int w1, b1, g1, be1, w3, b3, g3, be3, w5, b5, g5, be5, w7, b7, g7, be7, wv, bv, wa, ba, total;
};
ORL_HD Offsets deep_offsets(int d, int n, bool gaussian = false) {
    Offsets o; o.d = d; o.n = n; int p = 0;
    o.w1 = p; p += H * d; o.b1 = p; p += H; o.g1 = p; p += H; o.be1 = p; p += H;
    o.w3 = p; p += H * H; o.b3 = p; p += H; o.g3 = p; p += H; o.be3 = p; p += H;
    o.w5 = p; p += H * H; o.b5 = p; p += H; o.g5 = p; p += H; o.be5 = p; p += H;
    o.w7 = p; p += H * H; o.b7 = p; p += H; o.g7 = p; p += H; o.be7 = p; p += H;
    o.wv = p; p += H; o.bv = p; p += 1;
    o.wa = p; p += n * H; o.ba = p; p += n;
    if (gaussian) p += n;   // logstd
    o.total = p;
    return o;
}
// logstd[n] of a DiagGaussian head: right after ba
ORL_HD int logstd_offset(const Offsets& o) { return o.ba + o.n; }

// tape layout of one row (floats).  P operands (local gradients), Q operands (layer inputs), S column-sum fields.
constexpr int TP_DZ1 = 0, TP_DZ3 = 64, TP_DZ5 = 128, TP_DZ7 = 192, TP_DLOG = 256, TP_DV = 264;
constexpr int TQ_X = 272, TQ_Y1 = 336, TQ_Y3 = 400, TQ_Y5 = 464, TQ_Y7 = 528;
constexpr int TS_DY1N1 = 592, TS_DY1 = 656, TS_DY3N3 = 720, TS_DY3 = 784, TS_DY5N5 = 848, TS_DY5 = 912, TS_DY7N7 = 976, TS_DY7 = 1040;
constexpr int TAPE = 1104;
// DiagGaussian head: the same fields, then the row's dL/dlogstd[8] (zero beyond n), column-summed into logstd
constexpr int TS_DLS = 1104, TAPE_GAUSSIAN = 1112;
ORL_HD constexpr int tape_width(bool gaussian) { return gaussian ? TAPE_GAUSSIAN : TAPE; }

// what the backward needs from the forward of one row
struct Save {
    float a1[H], n1[H], n3[H], a5[H], n5[H], n7[H];
    float rstd1, rstd3, rstd5, rstd7;
};

// forward of one row: x[d] -> value, logits[n].  `sv` / `tape` may be NULL (rollout / value passes).
ORLD_STEP void deep_forward(const float* P, const Offsets& o, int act_id, const float* x, float* value, float* logits, Save* sv,
                            float* tape) {
    float a[H], nrm[H], y[H], z[H];
    // obs_prep
    orl_rnn::trunk_forward(P, o, act_id, x, y, sv ? sv->a1 : nullptr, sv ? sv->n1 : nullptr, tape ? tape + TQ_Y1 : nullptr,
                           sv ? sv->n3 : nullptr, sv ? &sv->rstd1 : nullptr, sv ? &sv->rstd3 : nullptr);
    if (tape) { for (int k = 0; k < MAXD; ++k) tape[TQ_X + k] = k < o.d ? x[k] : 0.f; for (int j = 0; j < H; ++j) tape[TQ_Y3 + j] = y[j]; }
    // common.fc1 -> act -> LN5
    linear64(P + o.w5, P + o.b5, y, H, z);
    for (int j = 0; j < H; ++j) a[j] = act_fwd(z[j], act_id);
    float r = layernorm64(a, nrm);
    if (sv) { for (int j = 0; j < H; ++j) { sv->a5[j] = a[j]; sv->n5[j] = nrm[j]; } sv->rstd5 = r; }
    for (int j = 0; j < H; ++j) y[j] = nrm[j] * P[o.g5 + j] + P[o.be5 + j];
    if (tape) for (int j = 0; j < H; ++j) tape[TQ_Y5 + j] = y[j];
    // common.fc3 -> LN7
    linear64(P + o.w7, P + o.b7, y, H, z);
    r = layernorm64(z, nrm);
    if (sv) { for (int j = 0; j < H; ++j) sv->n7[j] = nrm[j]; sv->rstd7 = r; }
    for (int j = 0; j < H; ++j) y[j] = nrm[j] * P[o.g7 + j] + P[o.be7 + j];
    if (tape) for (int j = 0; j < H; ++j) tape[TQ_Y7 + j] = y[j];
    // heads
    if (value) {
        float s = P[o.bv];
        for (int k = 0; k < H; ++k) s = fmaf(P[o.wv + k], y[k], s);
        *value = s;
    }
    if (logits) {
        for (int j = 0; j < o.n; ++j) {
            float s = P[o.ba + j];
            for (int k = 0; k < H; ++k) s = fmaf(P[o.wa + j * H + k], y[k], s);
            logits[j] = s;
        }
    }
}

// backward of one row given dL/dvalue and dL/dlogits: fills the P and S fields of the tape row
ORLD_STEP void deep_backward(const float* P, const Offsets& o, int act_id, const Save& sv, float dvalue, const float* dlogits,
                             float* tape) {
    float dy[H], dn[H], dz[H];
    for (int j = 0; j < MAXN; ++j) tape[TP_DLOG + j] = j < o.n ? dlogits[j] : 0.f;
    for (int j = 0; j < 8; ++j) tape[TP_DV + j] = j == 0 ? dvalue : 0.f;
    // heads -> y7
    for (int k = 0; k < H; ++k) {
        float s = P[o.wv + k] * dvalue;
        for (int j = 0; j < o.n; ++j) s = fmaf(P[o.wa + j * H + k], dlogits[j], s);
        dy[k] = s;
    }
    // LN7 affine + norm -> dz7
    for (int j = 0; j < H; ++j) { tape[TS_DY7N7 + j] = dy[j] * sv.n7[j]; tape[TS_DY7 + j] = dy[j]; dn[j] = dy[j] * P[o.g7 + j]; }
    layernorm64_bwd(dn, sv.n7, sv.rstd7, dz);
    for (int j = 0; j < H; ++j) tape[TP_DZ7 + j] = dz[j];
    // fc7 -> y5 -> LN5 -> act
    linear64_bwd_data(P + o.w7, dz, dy);
    for (int j = 0; j < H; ++j) { tape[TS_DY5N5 + j] = dy[j] * sv.n5[j]; tape[TS_DY5 + j] = dy[j]; dn[j] = dy[j] * P[o.g5 + j]; }
    layernorm64_bwd(dn, sv.n5, sv.rstd5, dz);
    for (int j = 0; j < H; ++j) { dz[j] *= act_bwd_from_out(sv.a5[j], act_id); tape[TP_DZ5 + j] = dz[j]; }
    // fc5 -> y3 -> obs_prep
    linear64_bwd_data(P + o.w5, dz, dy);
    orl_rnn::trunk_backward<TP_DZ1, TP_DZ3, TS_DY1N1, TS_DY1, TS_DY3N3, TS_DY3>(P, o, act_id, sv, dy, tape);
}

}  // namespace orl_deep
