// Sequential (one row at a time) restatement of the recurrent policy / value network of the PPO hot
// path.  The step functions are host code: g++ compiles them for the CPU tests (tests/test_rnn_core_cpu.py
// drives them through a tiny C shim and checks them against the torch oracle) and they are the element-wise
// reference of the warp-cooperative step of orl_rnn_warp.cuh — so the numerics of the GRU path are verified
// without a GPU.  The parameter offsets, the tape layout and the helpers are __host__ __device__: the warp path
// and the shared-model core (orl_deep_core.h) use them, and the MLPBase trunk (trunk_forward / trunk_backward) is
// also that of the shared-model core and of the self-play forward (orl_selfplay.cu).
//
// Network (reference: MLPBase mlp.py:100-176 -> RNNLayer rnn.py:5-99 (nn.GRU 64->64, 1 layer, then
// LayerNorm) -> head: Categorical.linear act.py / v_out value_network.py:106-109):
//   x(d) -> fc1 -> act -> LN1 -> fc3 -> LN3 -> GRU(h*mask) -> LNr -> head(n)
// Flat parameter layout (state_dict order of the reference, see rnn_offsets):
//   W1[64][d] b1 g1 be1 | W3[64][64] b3 g3 be3 | Wih[192][64] Whh[192][64] bih[192] bhh[192] | gr ber | Wh[n][64] bh[n]
// and, for a DiagGaussian head, | logstd[n] (act.action_out.fc_mean.*, then act.action_out.logstd._bias)
// GRU gate order r, z, n (torch.nn.GRU).  The chunk backward writes a per-row "tape" of local gradients
// and forward activations; the parameter gradients are tape reductions  dW = sum_rows P^T Q.
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define ORL_HD __host__ __device__ __forceinline__
#else
#define ORL_HD static inline
#endif

namespace orl_rnn {

constexpr int H = 64, G3 = 192, MAXN = 8, MAXD = 64;
constexpr float LN_EPS = 1e-5f;

struct Offsets {
    int d, n;
    int w1, b1, g1, be1, w3, b3, g3, be3, wih, whh, bih, bhh, gr, ber, wh, bh, ls, total;
};
ORL_HD Offsets rnn_offsets(int d, int n, bool gaussian = false) {
    Offsets o; o.d = d; o.n = n; int p = 0;
    o.w1 = p; p += H * d; o.b1 = p; p += H; o.g1 = p; p += H; o.be1 = p; p += H;
    o.w3 = p; p += H * H; o.b3 = p; p += H; o.g3 = p; p += H; o.be3 = p; p += H;
    o.wih = p; p += G3 * H; o.whh = p; p += G3 * H; o.bih = p; p += G3; o.bhh = p; p += G3;
    o.gr = p; p += H; o.ber = p; p += H;
    o.wh = p; p += n * H; o.bh = p; p += n;
    o.ls = p; if (gaussian) p += n;   // logstd
    o.total = p;
    return o;
}

// tape layout of one row-step (floats)
constexpr int TP_DZ1 = 0, TP_DZ3 = 64, TP_DGI = 128, TP_DGH = 320, TP_DLOG = 512;            // P operands
constexpr int TQ_X = 520, TQ_Y1 = 584, TQ_Y3 = 648, TQ_HM = 712, TQ_O = 776;                   // Q operands
constexpr int TS_DY1N1 = 840, TS_DY1 = 904, TS_DY3N3 = 968, TS_DY3 = 1032, TS_DONO = 1096, TS_DO = 1160;  // column sums
constexpr int TAPE = 1224;

ORL_HD float act_fwd(float z, int id) {
    switch (id) { case 0: return tanhf(z); case 1: return z > 0.f ? z : 0.f; case 2: return z > 0.f ? z : 0.01f * z; default: return z > 0.f ? z : expm1f(z); }
}
ORL_HD float act_bwd_from_out(float a, int id) {   // derivative given the OUTPUT a (a == 0 only where relu clipped)
    switch (id) { case 0: return 1.f - a * a; case 1: return a > 0.f ? 1.f : 0.f; case 2: return a > 0.f ? 1.f : 0.01f; default: return a > 0.f ? 1.f : a + 1.f; }
}
ORL_HD float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// y = LN(v) without affine; returns rstd; n_out = normalised
ORL_HD float layernorm64(const float* v, float* n_out) {
    float s = 0.f;
    for (int i = 0; i < H; ++i) s += v[i];
    const float m = s * (1.f / H);
    float q = 0.f;
    for (int i = 0; i < H; ++i) { const float dlt = v[i] - m; n_out[i] = dlt; q += dlt * dlt; }
    const float r = 1.f / sqrtf(q * (1.f / H) + LN_EPS);
    for (int i = 0; i < H; ++i) n_out[i] *= r;
    return r;
}
// dv = rstd * (dn - mean(dn) - n * mean(dn*n))
ORL_HD void layernorm64_bwd(const float* dn, const float* n, float rstd, float* dv) {
    float s1 = 0.f, s2 = 0.f;
    for (int i = 0; i < H; ++i) { s1 += dn[i]; s2 += dn[i] * n[i]; }
    s1 *= (1.f / H); s2 *= (1.f / H);
    for (int i = 0; i < H; ++i) dv[i] = rstd * (dn[i] - s1 - n[i] * s2);
}
// y[j] = b[j] + sum_k W[j][k] x[k]   (64 x K, row-major)
ORL_HD void linear64(const float* W, const float* b, const float* x, int K, float* y) {
    for (int j = 0; j < H; ++j) {
        float s = b[j];
        for (int k = 0; k < K; ++k) s = fmaf(W[j * K + k], x[k], s);
        y[j] = s;
    }
}
// dx[k] = sum_j W[j][k] dz[j]
ORL_HD void linear64_bwd_data(const float* W, const float* dz, float* dx) {
    for (int k = 0; k < H; ++k) dx[k] = 0.f;
    for (int j = 0; j < H; ++j) {
        const float g = dz[j];
        for (int k = 0; k < H; ++k) dx[k] = fmaf(W[j * H + k], g, dx[k]);
    }
}

// The MLPBase trunk of one row, x(d) -> fc1 -> act -> LN1 -> fc3 -> LN3 -> y3[64], of every sequential core and of the
// self-play forward.  O: any offsets struct with d, w1, b1, g1, be1, w3, b3, g3, be3.  Writes a1 (the activation), n1,
// y1 (= LN1 with affine), n3, rstd1 and rstd3 where the caller passes them.
template <class O>
ORL_HD void trunk_forward(const float* P, const O& o, int act_id, const float* x, float* y3, float* a1 = nullptr,
                          float* n1 = nullptr, float* y1 = nullptr, float* n3 = nullptr, float* rstd1 = nullptr,
                          float* rstd3 = nullptr) {
    float a[H], nrm[H];
    for (int j = 0; j < H; ++j) {
        float s = P[o.b1 + j];
        for (int k = 0; k < o.d; ++k) s = fmaf(P[o.w1 + j * o.d + k], x[k], s);
        a[j] = act_fwd(s, act_id);
    }
    const float r1 = layernorm64(a, nrm);
    if (a1) for (int j = 0; j < H; ++j) a1[j] = a[j];
    if (n1) for (int j = 0; j < H; ++j) n1[j] = nrm[j];
    if (rstd1) *rstd1 = r1;
    for (int j = 0; j < H; ++j) y3[j] = nrm[j] * P[o.g1 + j] + P[o.be1 + j];   // y1, until fc3 has read it
    if (y1) for (int j = 0; j < H; ++j) y1[j] = y3[j];
    linear64(P + o.w3, P + o.b3, y3, H, a);
    const float r3 = layernorm64(a, nrm);
    if (n3) for (int j = 0; j < H; ++j) n3[j] = nrm[j];
    if (rstd3) *rstd3 = r3;
    for (int j = 0; j < H; ++j) y3[j] = nrm[j] * P[o.g3 + j] + P[o.be3 + j];
}

// Backward of the trunk from dy3 = dL/dy3, given the forward's saved a1, n1, n3, rstd1, rstd3 (fields of S).  Writes the
// trunk's tape fields, whose offsets each core passes at compile time.
template <int DZ1, int DZ3, int DY1N1, int DY1, int DY3N3, int DY3, class O, class S>
ORL_HD void trunk_backward(const float* P, const O& o, int act_id, const S& sv, const float* dy3, float* tape) {
    float dn[H], dz[H], dy[H];
    for (int j = 0; j < H; ++j) { tape[DY3N3 + j] = dy3[j] * sv.n3[j]; tape[DY3 + j] = dy3[j]; dn[j] = dy3[j] * P[o.g3 + j]; }
    layernorm64_bwd(dn, sv.n3, sv.rstd3, dz);
    for (int j = 0; j < H; ++j) tape[DZ3 + j] = dz[j];
    linear64_bwd_data(P + o.w3, dz, dy);
    for (int j = 0; j < H; ++j) { tape[DY1N1 + j] = dy[j] * sv.n1[j]; tape[DY1 + j] = dy[j]; dn[j] = dy[j] * P[o.g1 + j]; }
    layernorm64_bwd(dn, sv.n1, sv.rstd1, dz);
    for (int j = 0; j < H; ++j) tape[DZ1 + j] = dz[j] * act_bwd_from_out(sv.a1[j], act_id);
}

// Saved forward state of one row-step (what the backward needs)
struct StepSave {
    float a1[H], n1[H], n3[H], y3[H], hm[H], r[H], z[H], nn[H], ghn[H], no[H];
    float rstd1, rstd3, rstdr;
};

// One forward step of a recurrent net.  x[d], h_in[64], mask -> h_out[64], head out[n].
// `sv` may be NULL (rollout).  Also returns y1 / o through the tape pointer when given.
static inline void rnn_step_forward(const float* P, const Offsets& o, int act_id, const float* x, const float* h_in, float mask,
                             float* h_out, float* out, StepSave* sv, float* tape) {
    float a1[H], n1[H], y1[H], n3[H], y3[H], rstd1, rstd3;
    if (tape) for (int k = 0; k < MAXD; ++k) tape[TQ_X + k] = k < o.d ? x[k] : 0.f;
    trunk_forward(P, o, act_id, x, y3, a1, n1, y1, n3, &rstd1, &rstd3);
    float hm[H];
    for (int j = 0; j < H; ++j) hm[j] = h_in[j] * mask;
    float hraw[H], rr[H], zz[H], nn[H], ghn[H];
    for (int j = 0; j < H; ++j) {
        float gir = P[o.bih + j], giz = P[o.bih + H + j], gin = P[o.bih + 2 * H + j];
        float ghr = P[o.bhh + j], ghz = P[o.bhh + H + j], ghnv = P[o.bhh + 2 * H + j];
        for (int k = 0; k < H; ++k) {
            const float yv = y3[k], hv = hm[k];
            gir = fmaf(P[o.wih + j * H + k], yv, gir);
            giz = fmaf(P[o.wih + (H + j) * H + k], yv, giz);
            gin = fmaf(P[o.wih + (2 * H + j) * H + k], yv, gin);
            ghr = fmaf(P[o.whh + j * H + k], hv, ghr);
            ghz = fmaf(P[o.whh + (H + j) * H + k], hv, ghz);
            ghnv = fmaf(P[o.whh + (2 * H + j) * H + k], hv, ghnv);
        }
        const float r = sigmoidf_(gir + ghr), z = sigmoidf_(giz + ghz);
        const float nv = tanhf(gin + r * ghnv);
        rr[j] = r; zz[j] = z; nn[j] = nv; ghn[j] = ghnv;
        hraw[j] = (1.f - z) * nv + z * hm[j];
    }
    float no[H];
    const float rstdr = layernorm64(hraw, no);
    float ov[H];
    for (int j = 0; j < H; ++j) { ov[j] = no[j] * P[o.gr + j] + P[o.ber + j]; h_out[j] = hraw[j]; }
    for (int j = 0; j < o.n; ++j) {
        float s = P[o.bh + j];
        for (int k = 0; k < H; ++k) s = fmaf(P[o.wh + j * H + k], ov[k], s);
        out[j] = s;
    }
    if (sv) {
        for (int j = 0; j < H; ++j) {
            sv->a1[j] = a1[j]; sv->n1[j] = n1[j]; sv->n3[j] = n3[j]; sv->y3[j] = y3[j]; sv->hm[j] = hm[j];
            sv->r[j] = rr[j]; sv->z[j] = zz[j]; sv->nn[j] = nn[j]; sv->ghn[j] = ghn[j]; sv->no[j] = no[j];
        }
        sv->rstd1 = rstd1; sv->rstd3 = rstd3; sv->rstdr = rstdr;
    }
    if (tape) {
        for (int j = 0; j < H; ++j) { tape[TQ_Y1 + j] = y1[j]; tape[TQ_Y3 + j] = y3[j]; tape[TQ_HM + j] = hm[j]; tape[TQ_O + j] = ov[j]; }
    }
}

// Backward of one row-step.  dlogit[n]: dL/d head output; dh_from_next[64]: dL/d h_out arriving from the
// following step of the chunk (zero for the last step).  Writes the P / S parts of the tape and returns
// dL/d h_in (already multiplied by the mask) in dh_prev.
static inline void rnn_step_backward(const float* P, const Offsets& o, int act_id, const StepSave& sv, float mask, const float* dlogit,
                              const float* dh_from_next, float* dh_prev, float* tape) {
    float dov[H], dno[H], dh[H];
    for (int k = 0; k < H; ++k) {
        float s = 0.f;
        for (int j = 0; j < o.n; ++j) s = fmaf(P[o.wh + j * H + k], dlogit[j], s);
        dov[k] = s;
        dno[k] = s * P[o.gr + k];
        tape[TS_DONO + k] = s * sv.no[k];
        tape[TS_DO + k] = s;
    }
    layernorm64_bwd(dno, sv.no, sv.rstdr, dh);
    for (int k = 0; k < H; ++k) dh[k] += dh_from_next[k];
    float dgi[G3], dgh[G3], dhm[H];
    for (int j = 0; j < H; ++j) {
        const float r = sv.r[j], z = sv.z[j], nv = sv.nn[j];
        const float dnn = dh[j] * (1.f - z), dz = dh[j] * (sv.hm[j] - nv);
        dhm[j] = dh[j] * z;
        const float dnpre = dnn * (1.f - nv * nv);
        const float dr = dnpre * sv.ghn[j];
        const float dzpre = dz * z * (1.f - z), drpre = dr * r * (1.f - r);
        dgi[j] = drpre; dgi[H + j] = dzpre; dgi[2 * H + j] = dnpre;
        dgh[j] = drpre; dgh[H + j] = dzpre; dgh[2 * H + j] = dnpre * r;
    }
    float dy3[H];
    for (int k = 0; k < H; ++k) {
        float s = 0.f, t = 0.f;
        for (int g = 0; g < G3; ++g) { s = fmaf(P[o.wih + g * H + k], dgi[g], s); t = fmaf(P[o.whh + g * H + k], dgh[g], t); }
        dy3[k] = s;
        dh_prev[k] = (dhm[k] + t) * mask;
    }
    for (int g = 0; g < G3; ++g) { tape[TP_DGI + g] = dgi[g]; tape[TP_DGH + g] = dgh[g]; }
    trunk_backward<TP_DZ1, TP_DZ3, TS_DY1N1, TS_DY1, TS_DY3N3, TS_DY3>(P, o, act_id, sv, dy3, tape);
    for (int j = 0; j < MAXN; ++j) tape[TP_DLOG + j] = j < o.n ? dlogit[j] : 0.f;
}

}  // namespace orl_rnn
