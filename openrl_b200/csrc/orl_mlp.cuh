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
// (orl_ppo.cu) unfolds them into the true parameter gradients.  The fold and its inverse are written once,
// below fold_offsets (folded_w3 ... folded_bh, unfolded_grad).
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
constexpr int MAX_OUT = 8;  // head width bound NB of the per-thread head code (head_dots, sample_action, categorical_row)
constexpr int MAX_OUT_WIDE = 64;  // head width bound NB of the wide Categorical head: a logits tile in shared memory
constexpr int OBS_PANEL = 64;     // observation columns per fc1 K-panel of a wide observation (fc1_panels)
constexpr int LDX_PANEL = OBS_PANEL + 4;   // leading dimension of a staged observation panel
constexpr int MAX_OBS_WIDE = 256; // observation width bound of the panelled fc1 (widths <= 64 stage all of W1 at once)
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

// The LayerNorm fold, one element of net `o` at a time: W3f[j][k] = W3[j][k] g1[k], b3f[j] = b3[j] + W3[j] . be1,
// Whf[j][k] = Wh[j][k] g3[k] and bhf[j] = bh[j] + Wh[j] . be3 (both 0 for rows j >= n).  Every staging of folded
// weights calls these, so every kernel sees the same bits.
__device__ __forceinline__ float folded_w3(const float* P, const NetOffsets& o, int j, int k) { return P[o.w3 + j * H + k] * P[o.g1 + k]; }
__device__ __forceinline__ float folded_b3(const float* P, const NetOffsets& o, int j) {
    float s = P[o.b3 + j];
    for (int k = 0; k < H; ++k) s = fmaf(P[o.w3 + j * H + k], P[o.be1 + k], s);
    return s;
}
__device__ __forceinline__ float folded_wh(const float* P, const NetOffsets& o, int j, int k) {
    return j < o.n ? P[o.wh + j * H + k] * P[o.g3 + k] : 0.f;
}
__device__ __forceinline__ float folded_bh(const float* P, const NetOffsets& o, int j) {
    float s = 0.f;
    if (j < o.n) {
        s = P[o.bh + j];
        for (int k = 0; k < H; ++k) s = fmaf(P[o.wh + j * H + k], P[o.be3 + k], s);
    }
    return s;
}
// The inverse: the true gradient of parameter i (net_offsets order) from the net's folded gradient vector f.
__device__ __forceinline__ float unfolded_grad(const float* P, const NetOffsets& po, const FoldOffsets& fo, const float* f, int i) {
    if (i < po.b1) return f[fo.g1 + (i - po.w1)];
    if (i < po.g1) return f[fo.db1 + (i - po.b1)];
    if (i < po.be1) {  // dg1[k] = sum_j W3[j][k] * G3[j][k]
        const int k = i - po.g1; float s = 0.f;
        for (int j = 0; j < H; ++j) s = fmaf(P[po.w3 + j * H + k], f[fo.g3 + j * H + k], s);
        return s;
    }
    if (i < po.w3) {  // dbe1[k] = sum_j W3[j][k] * db3[j]
        const int k = i - po.be1; float s = 0.f;
        for (int j = 0; j < H; ++j) s = fmaf(P[po.w3 + j * H + k], f[fo.db3 + j], s);
        return s;
    }
    if (i < po.b3) {  // dW3[j][k] = G3[j][k]*g1[k] + db3[j]*be1[k]
        const int j = (i - po.w3) / H, k = (i - po.w3) % H;
        return fmaf(f[fo.g3 + j * H + k], P[po.g1 + k], f[fo.db3 + j] * P[po.be1 + k]);
    }
    if (i < po.g3) return f[fo.db3 + (i - po.b3)];
    if (i < po.be3) {
        const int k = i - po.g3; float s = 0.f;
        for (int j = 0; j < po.n; ++j) s = fmaf(P[po.wh + j * H + k], f[fo.gh + j * H + k], s);
        return s;
    }
    if (i < po.wh) {
        const int k = i - po.be3; float s = 0.f;
        for (int j = 0; j < po.n; ++j) s = fmaf(P[po.wh + j * H + k], f[fo.dbh + j], s);
        return s;
    }
    if (i < po.bh) {
        const int j = (i - po.wh) / H, k = (i - po.wh) % H;
        return fmaf(f[fo.gh + j * H + k], P[po.g3 + k], f[fo.dbh + j] * P[po.be3 + k]);
    }
    if (i < po.ls) return f[fo.dbh + (i - po.bh)];
    return f[fo.dls + (i - po.ls)];
}

__host__ __device__ inline int pad4(int x) { return (x + 3) & ~3; }

// Shared-memory weight block of one net (folded).  Sizes in floats.  NB is the head width bound: NB = 8 holds the head
// as 8 natural rows for the per-thread head dots; NB = 64 (Categorical heads of 9..64 actions) holds it k-major for the
// logits tile GEMM (head_tile) and, for the backward pass, natural for dn3 = dL . Whf.
struct SmemWeights {
    float* w1t;   // [dp][64]  k-major: w1t[k*64 + j] = W1[j][k]        (dp = pad4(d), zero padded)
    float* b1;    // [64]
    float* w3t;   // [64][64]  k-major folded: w3t[k*64 + j] = W3[j][k]*g1[k]
    float* w3n;   // [64][64]  natural folded: w3n[j*64 + k] = W3[j][k]*g1[k]   (backward only)
    float* b3f;   // [64]
    float* whf;   // [NB][64]  natural folded: whf[j*64 + k] = Wh[j][k]*g3[k]   (rows >= n zero; NB = 64: backward only)
    float* wht;   // [64][64]  k-major folded: wht[k*64 + j] = Wh[j][k]*g3[k]   (NB = 64 only; columns >= n zero)
    float* bhf;   // [NB]
};
template <int NB = MAX_OUT>
__host__ __device__ inline int smem_weights_floats(int d, bool backward) {
    const int head = NB == MAX_OUT ? MAX_OUT * H : (backward ? H * H : 0) + H * H;
    return pad4(d) * H + H + H * H + (backward ? H * H : 0) + H + head + NB;
}
template <int NB = MAX_OUT>
__device__ inline SmemWeights carve_weights(float*& p, int d, bool backward) {
    static_assert(NB == MAX_OUT || NB == MAX_OUT_WIDE, "head width bound");
    SmemWeights w;
    w.w1t = p; p += pad4(d) * H;
    w.b1 = p; p += H;
    w.w3t = p; p += H * H;
    w.w3n = backward ? p : nullptr; if (backward) p += H * H;
    w.b3f = p; p += H;
    if (NB == MAX_OUT) {
        w.whf = p; p += MAX_OUT * H;
        w.wht = nullptr;
    } else {
        w.whf = backward ? p : nullptr; if (backward) p += H * H;
        w.wht = p; p += H * H;
    }
    w.bhf = p; p += NB;
    return w;
}

// Stage + fold one net's parameters from the flat global buffer.  All threads of the CTA call it;
// ends with __syncthreads().  PANELS (d > 64): W1 is left out; fc1_panels stages it one panel at a time into a w1t
// carved at d = 64.
template <int NT, int NB = MAX_OUT, bool PANELS = false>
__device__ inline void load_weights_folded(const SmemWeights& w, const float* __restrict__ params, int d, int n,
                                           bool backward) {
    const NetOffsets o = net_offsets(d, n);
    const int tid = threadIdx.x, dp = pad4(d);
    if (!PANELS) {
        for (int i = tid; i < dp * H; i += NT) {
            const int k = i / H, j = i % H;
            w.w1t[i] = (k < d) ? params[o.w1 + j * d + k] : 0.f;
        }
    }
    for (int i = tid; i < H; i += NT) w.b1[i] = params[o.b1 + i];
    for (int i = tid; i < H * H; i += NT) {
        const int j = i / H, k = i % H;  // coalesced read of W3[j][k]
        const float v = folded_w3(params, o, j, k);
        w.w3t[k * H + j] = v;
        if (backward) w.w3n[i] = v;
    }
    if (NB == MAX_OUT) {
        for (int i = tid; i < MAX_OUT * H; i += NT) w.whf[i] = folded_wh(params, o, i / H, i % H);
    } else {
        for (int i = tid; i < H * H; i += NT) {
            const int j = i / H, k = i % H;
            const float v = folded_wh(params, o, j, k);
            w.wht[k * H + j] = v;
            if (backward) w.whf[i] = v;
        }
    }
    // folded biases: one warp-sized group of threads per output
    for (int j = tid; j < H; j += NT) w.b3f[j] = folded_b3(params, o, j);
    for (int j = tid; j < NB; j += NT) w.bhf[j] = folded_bh(params, o, j);
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

// The trunk after fc1's GEMM: acc holds Z1 = b1 + X W1^T on entry; activation + LayerNorm -> N1s, fc3 + LayerNorm ->
// N3s (normalised activations).  Optionally returns the per-row statistics and the activation sign bits needed by the
// backward pass.  Contains the __syncthreads() between the two layers; callers must sync before reading N3s from other
// threads.
template <int M, int NT, bool KEEP>
__device__ __forceinline__ void trunk_from_z1(const SmemWeights& w, float (&acc)[M / (NT / 16)][4], int activation_id,
                                              float* __restrict__ N1s, float* __restrict__ N3s,
                                              float (&mu1)[M / (NT / 16)], float (&rstd1)[M / (NT / 16)],
                                              float (&rstd3)[M / (NT / 16)], unsigned& posmask) {
    constexpr int TY = NT / 16, RPT = M / TY;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
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

// Trunk forward of one tile: Xs [M][ldx] (raw obs, zero padded to pad4(d)) -> N1s, N3s (trunk_from_z1).
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
    trunk_from_z1<M, NT, KEEP>(w, acc, activation_id, N1s, N3s, mu1, rstd1, rstd3, posmask);
}

// ---- fc1 of wide observations (64 < d <= 256) ------------------------------------------------------------------------
// A tile of d = 256 with all of W1 staged k-major would need 64 KB of W1 and a 128 x 260 observation tile: the update
// kernel would no longer fit in shared memory.  So fc1 runs as a loop over the P = ceil(d / 64) K-panels of the
// observation: Z1 = b1 + sum_p X[:, 64p..64p+64) W1[:, 64p..64p+64)^T, with the panel's W1 columns staged into a 64 x 64
// k-major w1t and the tile's observation columns into an M x LDX_PANEL Xs (the buffers of the d = 64 layout).  Panels
// are summed in order 0..P-1, so the bits do not depend on the grid.  row(r) gives the observation row r of the tile in
// global memory, or nullptr for a row outside it (staged as zeros).

// Xs[r][k] = obs row r, column 64p + k (0 beyond d).  No syncs.
template <int M, int NT, typename RowPtr>
__device__ __forceinline__ void stage_obs_panel(float* __restrict__ Xs, int d, int p, RowPtr&& row) {
    for (int i = threadIdx.x; i < M * LDX_PANEL; i += NT) {
        const int r = i / LDX_PANEL, k = i % LDX_PANEL, c = OBS_PANEL * p + k;
        const float* src = row(r);
        Xs[i] = (src != nullptr && k < OBS_PANEL && c < d) ? src[c] : 0.f;
    }
}

// acc = Z1 of the tile (b1 + X W1^T) over every panel.  W1 = params + net_offsets(d, n).w1.  Syncs before staging each
// panel and after it, so the caller need not sync before the call; on return Xs holds the last panel, P - 1.
template <int M, int NT, typename RowPtr>
__device__ __forceinline__ void fc1_panels(const SmemWeights& w, const float* __restrict__ W1, int d, float* __restrict__ Xs,
                                           RowPtr&& row, float (&acc)[M / (NT / 16)][4]) {
    constexpr int TY = NT / 16, RPT = M / TY;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    {
        const float4 b = *reinterpret_cast<const float4*>(w.b1 + 4 * tx);
#pragma unroll
        for (int i = 0; i < RPT; ++i) { acc[i][0] = b.x; acc[i][1] = b.y; acc[i][2] = b.z; acc[i][3] = b.w; }
    }
    const int P = (d + OBS_PANEL - 1) / OBS_PANEL;
    for (int p = 0; p < P; ++p) {
        __syncthreads();   // the previous panel's GEMM (or the caller's last reads of Xs / w1t) is done
        // 8 adjacent threads read 8 consecutive columns of one W1 row (32 bytes, where one column per thread would take
        // a sector each); the shared stores of a warp then fall into 4 banks
        for (int i = threadIdx.x; i < OBS_PANEL * H; i += NT) {
            const int k = 8 * (i / (8 * H)) + i % 8, j = (i / 8) % H, c = OBS_PANEL * p + k;
            w.w1t[k * H + j] = c < d ? W1[j * d + c] : 0.f;
        }
        stage_obs_panel<M, NT>(Xs, d, p, row);
        __syncthreads();
        gemm_tile<RPT, TY>(Xs, LDX_PANEL, w.w1t, min(OBS_PANEL, pad4(d - OBS_PANEL * p)), acc, tx, ty);
    }
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

// Logits tile of a wide head (NB = 64): Ls[m][j] = bhf[j] + sum_k N3s[m][k] Whf[j][k] for all 64 columns j (0 for j >= n),
// an M x 64 tile GEMM in the trunk's layout, stored with leading dimension LDA.  Callers sync before reading Ls.
template <int M, int NT>
__device__ __forceinline__ void head_tile(const SmemWeights& w, const float* __restrict__ N3s, float* __restrict__ Ls) {
    constexpr int TY = NT / 16, RPT = M / TY;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float acc[RPT][4];
    const float4 b = *reinterpret_cast<const float4*>(w.bhf + 4 * tx);
#pragma unroll
    for (int i = 0; i < RPT; ++i) { acc[i][0] = b.x; acc[i][1] = b.y; acc[i][2] = b.z; acc[i][3] = b.w; }
    gemm_tile<RPT, TY>(N3s, LDA, w.wht, H, acc, tx, ty);
    store_tile<RPT, TY>(Ls, acc, tx, ty);
}

}  // namespace orl
