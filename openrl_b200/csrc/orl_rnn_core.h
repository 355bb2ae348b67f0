// Sequential (one row at a time) restatement of the recurrent policy / value network of the PPO hot
// path, compiled BOTH by nvcc (device functions used by orl_rnn.cu, one thread per row / chunk) and by
// g++ (tests/test_rnn_core_cpu.py drives it through a tiny C shim and checks it against the torch
// oracle) — so the numerics of the GRU path are verified without a GPU.
//
// Network (reference: MLPBase mlp.py:100-176 -> RNNLayer rnn.py:5-99 (nn.GRU 64->64, 1 layer, then
// LayerNorm) -> head: Categorical.linear act.py / v_out value_network.py:106-109):
//   x(d) -> fc1 -> act -> LN1 -> fc3 -> LN3 -> GRU(h*mask) -> LNr -> head(n)
// Flat parameter layout (state_dict order of the reference, see rnn_offsets):
//   W1[64][d] b1 g1 be1 | W3[64][64] b3 g3 be3 | Wih[192][64] Whh[192][64] bih[192] bhh[192] | gr ber | Wh[n][64] bh[n]
// GRU gate order r, z, n (torch.nn.GRU).  The chunk backward writes a per-row "tape" of local gradients
// and forward activations; the parameter gradients are tape reductions  dW = sum_rows P^T Q.
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define ORL_HD __host__ __device__ __forceinline__
// The two step functions are real calls on the device (own stack frames): with everything inlined into the
// per-chunk kernel nvcc 12.9 merged the stack slots of the caller's observation row and the callee's GRU
// output (observed in SASS and as a corrupted tape), i.e. wrong gradients.
#define ORL_HD_STEP __host__ __device__ __noinline__
#else
#define ORL_HD static inline
#define ORL_HD_STEP static inline
#endif

namespace orl_rnn {

constexpr int H = 64, G3 = 192, MAXN = 8, MAXD = 64;
constexpr float LN_EPS = 1e-5f;

struct Offsets {
    int d, n;
    int w1, b1, g1, be1, w3, b3, g3, be3, wih, whh, bih, bhh, gr, ber, wh, bh, total;
};
ORL_HD Offsets rnn_offsets(int d, int n) {
    Offsets o; o.d = d; o.n = n; int p = 0;
    o.w1 = p; p += H * d; o.b1 = p; p += H; o.g1 = p; p += H; o.be1 = p; p += H;
    o.w3 = p; p += H * H; o.b3 = p; p += H; o.g3 = p; p += H; o.be3 = p; p += H;
    o.wih = p; p += G3 * H; o.whh = p; p += G3 * H; o.bih = p; p += G3; o.bhh = p; p += G3;
    o.gr = p; p += H; o.ber = p; p += H;
    o.wh = p; p += n * H; o.bh = p; p += n;
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

// Saved forward state of one row-step (what the backward needs)
struct StepSave {
    float a1[H], n1[H], n3[H], y3[H], hm[H], r[H], z[H], nn[H], ghn[H], no[H];
    float rstd1, rstd3, rstdr;
};

// One forward step of a recurrent net.  x[d], h_in[64], mask -> h_out[64], head out[n].
// `sv` may be NULL (rollout).  Also returns y1 / o through the tape pointer when given.
ORL_HD_STEP void rnn_step_forward(const float* P, const Offsets& o, int act_id, const float* x, const float* h_in, float mask,
                             float* h_out, float* out, StepSave* sv, float* tape) {
    float a1[H], n1[H], y1[H], z3[H], n3[H], y3[H];
    if (tape) for (int k = 0; k < MAXD; ++k) tape[TQ_X + k] = k < o.d ? x[k] : 0.f;
    for (int j = 0; j < H; ++j) {
        float s = P[o.b1 + j];
        for (int k = 0; k < o.d; ++k) s = fmaf(P[o.w1 + j * o.d + k], x[k], s);
        a1[j] = act_fwd(s, act_id);
    }
    const float rstd1 = layernorm64(a1, n1);
    for (int j = 0; j < H; ++j) y1[j] = n1[j] * P[o.g1 + j] + P[o.be1 + j];
    for (int j = 0; j < H; ++j) {
        float s = P[o.b3 + j];
        for (int k = 0; k < H; ++k) s = fmaf(P[o.w3 + j * H + k], y1[k], s);
        z3[j] = s;
    }
    const float rstd3 = layernorm64(z3, n3);
    for (int j = 0; j < H; ++j) y3[j] = n3[j] * P[o.g3 + j] + P[o.be3 + j];
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
ORL_HD_STEP void rnn_step_backward(const float* P, const Offsets& o, int act_id, const StepSave& sv, float mask, const float* dlogit,
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
    float dn3[H], dz3[H];
    for (int k = 0; k < H; ++k) { dn3[k] = dy3[k] * P[o.g3 + k]; tape[TS_DY3N3 + k] = dy3[k] * sv.n3[k]; tape[TS_DY3 + k] = dy3[k]; }
    layernorm64_bwd(dn3, sv.n3, sv.rstd3, dz3);
    float dy1[H], dn1[H], da1[H];
    for (int k = 0; k < H; ++k) {
        float s = 0.f;
        for (int j = 0; j < H; ++j) s = fmaf(P[o.w3 + j * H + k], dz3[j], s);
        dy1[k] = s;
        dn1[k] = s * P[o.g1 + k];
        tape[TS_DY1N1 + k] = s * sv.n1[k];
        tape[TS_DY1 + k] = s;
        tape[TP_DZ3 + k] = dz3[k];
    }
    layernorm64_bwd(dn1, sv.n1, sv.rstd1, da1);
    for (int k = 0; k < H; ++k) tape[TP_DZ1 + k] = da1[k] * act_bwd_from_out(sv.a1[k], act_id);
    for (int j = 0; j < MAXN; ++j) tape[TP_DLOG + j] = j < o.n ? dlogit[j] : 0.f;
}

}  // namespace orl_rnn
