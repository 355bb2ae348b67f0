// Tile primitives for the 64-wide policy / value MLPs of the PPO hot path (sm_90a, fp32 FFMA).
//
// Network (reference: MLPBase/MLPLayer openrl/modules/networks/utils/mlp.py:8-46,100-176 with
// layer_N == 1, hidden 64; heads openrl/modules/networks/utils/act.py, value_network.py:106-109):
//     x(d) -> fc1: Linear(d,64) -> act -> LayerNorm(64)
//          -> fc3: Linear(64,64) -> LayerNorm(64)
//          -> head: Linear(64,n)   (n logits | 1 value)
//
// Flat parameter layout of one net (float32, the order of the reference's state_dict):
//     W1[64][d] b1[64] g1[64] be1[64] W3[64][64] b3[64] g3[64] be3[64] Wh[n][64] bh[n]
//
// LayerNorm affine parameters are FOLDED into the following Linear when weights are staged in
// shared memory (W3f = W3*g1, b3f = b3 + W3.be1; Whf = Wh*g3, bhf = bh + Wh.be3), so tiles only
// carry the normalised activations n1, n3.  The backward pass therefore produces "folded"
// gradients (G1 = dZ1^T X, G3 = dZ3^T n1, GH = dL^T n3 and the bias sums); the finalize kernel
// (orl_ppo.cu) unfolds them into the true parameter gradients.
//
// A tile is M rows x 64 columns, activations row-major in shared memory with leading dimension
// LDA = 68 floats.  Thread t of the NT-thread CTA owns columns 4*tx..4*tx+3 (tx = t % 16) of rows
// ty + (NT/16)*i (ty = t / 16, i < RPT = M / (NT/16)); the 16 threads of a half-warp share a row,
// so LayerNorm statistics are 4-step xor-shuffles.
#pragma once
#include "orl_common.cuh"

namespace orl {

constexpr int H = 64;     // hidden width (cfg.hidden_size), fixed in this build
constexpr int LDA = 68;   // leading dimension of H-wide activation tiles in smem
constexpr int MAX_OUT = 8;  // max head width (n actions)
constexpr float LN_EPS = 1e-5f;

struct NetOffsets {
    int d, n;
    int w1, b1, g1, be1, w3, b3, g3, be3, wh, bh, ls, total;   // ls: logstd[n] (Gaussian head only)
};
__host__ __device__ inline NetOffsets net_offsets(int d, int n, int gaussian = 0) {
    NetOffsets o; o.d = d; o.n = n;
    int p = 0;
    o.w1 = p; p += H * d;  o.b1 = p; p += H;  o.g1 = p; p += H;  o.be1 = p; p += H;
    o.w3 = p; p += H * H;  o.b3 = p; p += H;  o.g3 = p; p += H;  o.be3 = p; p += H;
    o.wh = p; p += n * H;  o.bh = p; p += n;
    o.ls = p; if (gaussian) p += n;
    o.total = p;
    return o;
}
// folded-gradient vector layout of one net: G1[64][d] db1[64] G3[64][64] db3[64] GH[n][64] dbh[n]
struct FoldOffsets { int g1, db1, g3, db3, gh, dbh, dls, total; };   // dls: dL/dlogstd[n], always reserved
__host__ __device__ inline FoldOffsets fold_offsets(int d, int n) {
    FoldOffsets o; int p = 0;
    o.g1 = p; p += H * d;  o.db1 = p; p += H;  o.g3 = p; p += H * H;  o.db3 = p; p += H;
    o.gh = p; p += n * H;  o.dbh = p; p += n;  o.dls = p; p += n;  o.total = p;
    return o;
}

__host__ __device__ inline int pad4(int x) { return (x + 3) & ~3; }

// Shared-memory weight block of one net (folded).  Sizes in floats.
struct SmemWeights {
    float* w1t;   // [dp][64]  k-major: w1t[k*64 + j] = W1[j][k]        (dp = pad4(d), zero padded)
    float* b1;    // [64]
    float* w3t;   // [64][64]  k-major folded: w3t[k*64 + j] = W3[j][k]*g1[k]
    float* w3n;   // [64][64]  natural folded: w3n[j*64 + k] = W3[j][k]*g1[k]   (backward only)
    float* b3f;   // [64]
    float* whf;   // [8][64]   natural folded: whf[j*64 + k] = Wh[j][k]*g3[k]   (rows >= n zero)
    float* bhf;   // [8]
};
__host__ __device__ inline int smem_weights_floats(int d, bool backward) {
    return pad4(d) * H + H + H * H + (backward ? H * H : 0) + H + MAX_OUT * H + MAX_OUT;
}
__device__ inline SmemWeights carve_weights(float*& p, int d, bool backward) {
    SmemWeights w;
    w.w1t = p; p += pad4(d) * H;
    w.b1 = p; p += H;
    w.w3t = p; p += H * H;
    w.w3n = backward ? p : nullptr; if (backward) p += H * H;
    w.b3f = p; p += H;
    w.whf = p; p += MAX_OUT * H;
    w.bhf = p; p += MAX_OUT;
    return w;
}

// Stage + fold one net's parameters from the flat global buffer.  All threads of the CTA call it;
// ends with __syncthreads().
template <int NT>
__device__ inline void load_weights_folded(const SmemWeights& w, const float* __restrict__ params, int d, int n,
                                           bool backward) {
    const NetOffsets o = net_offsets(d, n);
    const int tid = threadIdx.x, dp = pad4(d);
    for (int i = tid; i < dp * H; i += NT) {
        const int k = i / H, j = i % H;
        w.w1t[i] = (k < d) ? params[o.w1 + j * d + k] : 0.f;
    }
    for (int i = tid; i < H; i += NT) w.b1[i] = params[o.b1 + i];
    for (int i = tid; i < H * H; i += NT) {
        const int j = i / H, k = i % H;  // coalesced read of W3[j][k]
        const float v = params[o.w3 + i] * params[o.g1 + k];
        w.w3t[k * H + j] = v;
        if (backward) w.w3n[i] = v;
    }
    for (int i = tid; i < MAX_OUT * H; i += NT) {
        const int j = i / H, k = i % H;
        w.whf[i] = (j < n) ? params[o.wh + j * H + k] * params[o.g3 + k] : 0.f;
    }
    // folded biases: one warp-sized group of threads per output
    for (int j = tid; j < H; j += NT) {
        float s = params[o.b3 + j];
        for (int k = 0; k < H; ++k) s = fmaf(params[o.w3 + j * H + k], params[o.be1 + k], s);
        w.b3f[j] = s;
    }
    for (int j = tid; j < MAX_OUT; j += NT) {
        float s = 0.f;
        if (j < n) {
            s = params[o.bh + j];
            for (int k = 0; k < H; ++k) s = fmaf(params[o.wh + j * H + k], params[o.be3 + k], s);
        }
        w.bhf[j] = s;
    }
    __syncthreads();
}

__device__ __forceinline__ float half_warp_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
}

// acc[i][c] (+)= sum_k A[row_i][k] * Bt[k][4*tx + c],  row_i = ty + TY*i, k < K (K % 4 == 0)
template <int RPT, int TY>
__device__ __forceinline__ void gemm_tile(const float* __restrict__ A, int lda, const float* __restrict__ Bt, int K,
                                          float (&acc)[RPT][4], int tx, int ty) {
    const float* a_base = A + ty * lda;
    const float* b_base = Bt + 4 * tx;
#pragma unroll 2
    for (int k0 = 0; k0 < K; k0 += 4) {
        const float4 b0 = *reinterpret_cast<const float4*>(b_base + (k0 + 0) * H);
        const float4 b1 = *reinterpret_cast<const float4*>(b_base + (k0 + 1) * H);
        const float4 b2 = *reinterpret_cast<const float4*>(b_base + (k0 + 2) * H);
        const float4 b3 = *reinterpret_cast<const float4*>(b_base + (k0 + 3) * H);
#pragma unroll
        for (int i = 0; i < RPT; ++i) {
            const float4 a = *reinterpret_cast<const float4*>(a_base + i * TY * lda + k0);
            acc[i][0] = fmaf(a.x, b0.x, acc[i][0]); acc[i][1] = fmaf(a.x, b0.y, acc[i][1]);
            acc[i][2] = fmaf(a.x, b0.z, acc[i][2]); acc[i][3] = fmaf(a.x, b0.w, acc[i][3]);
            acc[i][0] = fmaf(a.y, b1.x, acc[i][0]); acc[i][1] = fmaf(a.y, b1.y, acc[i][1]);
            acc[i][2] = fmaf(a.y, b1.z, acc[i][2]); acc[i][3] = fmaf(a.y, b1.w, acc[i][3]);
            acc[i][0] = fmaf(a.z, b2.x, acc[i][0]); acc[i][1] = fmaf(a.z, b2.y, acc[i][1]);
            acc[i][2] = fmaf(a.z, b2.z, acc[i][2]); acc[i][3] = fmaf(a.z, b2.w, acc[i][3]);
            acc[i][0] = fmaf(a.w, b3.x, acc[i][0]); acc[i][1] = fmaf(a.w, b3.y, acc[i][1]);
            acc[i][2] = fmaf(a.w, b3.z, acc[i][2]); acc[i][3] = fmaf(a.w, b3.w, acc[i][3]);
        }
    }
}

__device__ __forceinline__ float act_fwd(float z, int activation_id) {
    switch (activation_id) {
        case 0: return tanhf(z);
        case 1: return fmaxf(z, 0.f);
        case 2: return z > 0.f ? z : 0.01f * z;
        default: return z > 0.f ? z : expm1f(z);
    }
}
// derivative given the activation OUTPUT a (and, for the piecewise-linear ones, the sign bit)
__device__ __forceinline__ float act_bwd(float a, bool pos, int activation_id) {
    switch (activation_id) {
        case 0: return 1.f - a * a;
        case 1: return pos ? 1.f : 0.f;
        case 2: return pos ? 1.f : 0.01f;
        default: return pos ? 1.f : a + 1.f;
    }
}

// Row LayerNorm without affine on a thread's RPT x 4 block (torch.nn.LayerNorm statistics:
// biased variance, eps inside the sqrt).  acc <- (acc - mean) * rstd.
template <int RPT>
__device__ __forceinline__ void layernorm_rows(float (&acc)[RPT][4], float (&mu)[RPT], float (&rstd)[RPT]) {
#pragma unroll
    for (int i = 0; i < RPT; ++i) {
        float s = (acc[i][0] + acc[i][1]) + (acc[i][2] + acc[i][3]);
        s = half_warp_sum(s);
        const float m = s * (1.f / H);
        const float d0 = acc[i][0] - m, d1 = acc[i][1] - m, d2 = acc[i][2] - m, d3 = acc[i][3] - m;
        float v = (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
        v = half_warp_sum(v);
        const float r = 1.0f / sqrtf(v * (1.f / H) + LN_EPS);
        acc[i][0] = d0 * r; acc[i][1] = d1 * r; acc[i][2] = d2 * r; acc[i][3] = d3 * r;
        mu[i] = m; rstd[i] = r;
    }
}

// LayerNorm backward (no affine): dz = rstd * (dn - mean(dn) - n * mean(dn * n)), in place on dn.
template <int RPT>
__device__ __forceinline__ void layernorm_bwd_rows(float (&dn)[RPT][4], const float (&nrm)[RPT][4],
                                                   const float (&rstd)[RPT]) {
#pragma unroll
    for (int i = 0; i < RPT; ++i) {
        float s1 = (dn[i][0] + dn[i][1]) + (dn[i][2] + dn[i][3]);
        float s2 = (dn[i][0] * nrm[i][0] + dn[i][1] * nrm[i][1]) + (dn[i][2] * nrm[i][2] + dn[i][3] * nrm[i][3]);
        s1 = half_warp_sum(s1) * (1.f / H);
        s2 = half_warp_sum(s2) * (1.f / H);
#pragma unroll
        for (int c = 0; c < 4; ++c) dn[i][c] = rstd[i] * (dn[i][c] - s1 - nrm[i][c] * s2);
    }
}

template <int RPT, int TY>
__device__ __forceinline__ void store_tile(float* __restrict__ S, const float (&acc)[RPT][4], int tx, int ty) {
#pragma unroll
    for (int i = 0; i < RPT; ++i)
        *reinterpret_cast<float4*>(S + (ty + TY * i) * LDA + 4 * tx) =
            make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
}
template <int RPT, int TY>
__device__ __forceinline__ void load_tile(const float* __restrict__ S, float (&acc)[RPT][4], int tx, int ty) {
#pragma unroll
    for (int i = 0; i < RPT; ++i) {
        const float4 v = *reinterpret_cast<const float4*>(S + (ty + TY * i) * LDA + 4 * tx);
        acc[i][0] = v.x; acc[i][1] = v.y; acc[i][2] = v.z; acc[i][3] = v.w;
    }
}

// Trunk forward of one tile: Xs [M][ldx] (raw obs, zero padded to pad4(d)) -> N1s, N3s (normalised
// activations).  Optionally returns the per-row statistics and the activation sign bits needed by
// the backward pass.  Contains the __syncthreads() between the two layers; callers must sync
// before reading N3s from other threads.
template <int M, int NT, bool KEEP>
__device__ __forceinline__ void trunk_forward(const SmemWeights& w, const float* __restrict__ Xs, int ldx, int d,
                                              int activation_id, float* __restrict__ N1s, float* __restrict__ N3s,
                                              float (&mu1)[M / (NT / 16)], float (&rstd1)[M / (NT / 16)],
                                              float (&rstd3)[M / (NT / 16)], unsigned& posmask) {
    constexpr int TY = NT / 16, RPT = M / TY;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float acc[RPT][4];
    {
        const float4 b = *reinterpret_cast<const float4*>(w.b1 + 4 * tx);
#pragma unroll
        for (int i = 0; i < RPT; ++i) { acc[i][0] = b.x; acc[i][1] = b.y; acc[i][2] = b.z; acc[i][3] = b.w; }
    }
    gemm_tile<RPT, TY>(Xs, ldx, w.w1t, pad4(d), acc, tx, ty);
    unsigned pm = 0;
#pragma unroll
    for (int i = 0; i < RPT; ++i)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            if (KEEP && acc[i][c] > 0.f) pm |= 1u << (i * 4 + c);
            acc[i][c] = act_fwd(acc[i][c], activation_id);
        }
    posmask = pm;
    layernorm_rows<RPT>(acc, mu1, rstd1);
    store_tile<RPT, TY>(N1s, acc, tx, ty);
    __syncthreads();
    {
        const float4 b = *reinterpret_cast<const float4*>(w.b3f + 4 * tx);
#pragma unroll
        for (int i = 0; i < RPT; ++i) { acc[i][0] = b.x; acc[i][1] = b.y; acc[i][2] = b.z; acc[i][3] = b.w; }
    }
    gemm_tile<RPT, TY>(N1s, LDA, w.w3t, H, acc, tx, ty);
    float mu3[RPT];
    layernorm_rows<RPT>(acc, mu3, rstd3);
    store_tile<RPT, TY>(N3s, acc, tx, ty);
}

// Head dot products for the row owned by this thread group: PPR = NT / M threads per row
// (adjacent lanes), out[j] = bhf[j] + sum_k N3[row][k] * whf[j][k], valid in every lane of the group.
template <int M, int NT>
__device__ __forceinline__ void head_dots(const SmemWeights& w, const float* __restrict__ N3s, int n,
                                          float (&out)[MAX_OUT]) {
    constexpr int PPR = NT / M;
    static_assert(PPR == 1 || PPR == 2 || PPR == 4 || PPR == 8 || PPR == 16, "threads per row");
    const int row = threadIdx.x / PPR, part = threadIdx.x % PPR;
#pragma unroll
    for (int j = 0; j < MAX_OUT; ++j) out[j] = 0.f;
    for (int q = part; q < H / 4; q += PPR) {
        const float4 a = *reinterpret_cast<const float4*>(N3s + row * LDA + 4 * q);
#pragma unroll
        for (int j = 0; j < MAX_OUT; ++j) {
            if (j < n) {
                const float4 ww = *reinterpret_cast<const float4*>(w.whf + j * H + 4 * q);
                out[j] = fmaf(a.x, ww.x, fmaf(a.y, ww.y, fmaf(a.z, ww.z, fmaf(a.w, ww.w, out[j]))));
            }
        }
    }
#pragma unroll
    for (int j = 0; j < MAX_OUT; ++j) {
        if (j < n) {
#pragma unroll
            for (int o = PPR / 2; o > 0; o >>= 1) out[j] += __shfl_xor_sync(0xffffffffu, out[j], o);
            out[j] += w.bhf[j];
        }
    }
}

// torch.distributions.Categorical(logits=x): normalised logits nl = x - logsumexp(x), probs =
// softmax(nl).  Masked entries were set to -6e4 by the caller (distributions.py:71).
__device__ __forceinline__ void log_softmax_n(const float (&x)[MAX_OUT], int n, float (&nl)[MAX_OUT],
                                              float (&p)[MAX_OUT]) {
    float mx = x[0];
#pragma unroll
    for (int j = 1; j < MAX_OUT; ++j) if (j < n) mx = fmaxf(mx, x[j]);
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < MAX_OUT; ++j) if (j < n) s += expf(x[j] - mx);
    const float lse = mx + logf(s);
    float mx2 = -INFINITY;
#pragma unroll
    for (int j = 0; j < MAX_OUT; ++j) if (j < n) { nl[j] = x[j] - lse; mx2 = fmaxf(mx2, nl[j]); }
    float s2 = 0.f;
#pragma unroll
    for (int j = 0; j < MAX_OUT; ++j) if (j < n) { p[j] = expf(nl[j] - mx2); s2 += p[j]; }
#pragma unroll
    for (int j = 0; j < MAX_OUT; ++j) if (j < n) p[j] = p[j] / s2;
}


// Policy-gradient term of one (row, action-dimension): PPO clipped surrogate (ppo.py:300-319, with the
// optional dual clip :304-305) or the A2C loss -adv*logp (a2c.py:88).  Returns the loss contribution
// (to be weighted by the row weight) and d(loss)/d(logp); `ratio` comes back as the reported ratio.
struct PgTerm { float loss, dlogp, ratio; };
__device__ __forceinline__ PgTerm pg_term(float lp, float old_lp, float adv, float clip, int flags, float dual_coeff) {
    PgTerm o;
    if (flags & ORL_PPO_A2C) { o.loss = -adv * lp; o.dlogp = -adv; o.ratio = 0.f; return o; }
    const float raw = expf(lp - old_lp);
    float ratio = raw, dr = 1.f;                       // dr = d(ratio)/d(raw)
    if (flags & ORL_PPO_DUAL_CLIP) {                   // torch.min(ratio, coeff): ties split the gradient
        if (raw > dual_coeff) { ratio = dual_coeff; dr = 0.f; } else if (raw == dual_coeff) dr = 0.5f;
    }
    const float lo = 1.0f - clip, hi = 1.0f + clip;
    const float surr1 = ratio * adv, surr2 = fminf(fmaxf(ratio, lo), hi) * adv;
    const bool inside = ratio >= lo && ratio <= hi;
    const float sel = surr1 < surr2 ? 1.f : (surr1 > surr2 ? 0.f : (inside ? 1.f : 0.5f));
    o.loss = -fminf(surr1, surr2);
    o.dlogp = -sel * adv * dr * raw;
    o.ratio = ratio;
    return o;
}

}  // namespace orl
