// Warp-cooperative recurrent network step: ONE WARP per row, every 64-vector held as two registers per lane
// (elements `lane` and `lane + 32`), weights of one net staged once per CTA in shared memory as padded
// row-major matrices (leading dimension 65 floats, so that both W v — lane owns an output row — and
// W^T v — lane owns an input column — read conflict-free banks).  A warp advances R rows together: each weight
// read from shared memory feeds R FMAs (the mat-vecs are shared-memory-bandwidth bound, 4 B of weight per
// lane-FMA at R = 1), and the input vector of a mat-vec is parked in a per-warp shared scratch and read back as
// broadcast float4 (one wavefront per four inputs) instead of one shuffle per input.  LayerNorm by xor-shuffle
// reductions.  Nothing lives in local memory.
//
// Same math, same tape fields as the sequential restatement in orl_rnn_core.h (which the CPU test pins to
// the torch oracle); tests/debug_gru.py compares the tape of this implementation element-wise with the
// CPU core on the device's own rollout.  Summation orders differ (warp tree vs sequential): ~1e-7 relative.
//
// Tape row (floats): [0,1224) the P / Q / S fields of orl_rnn_core.h (inputs of the dW = sum P^T Q
// reductions), then the forward activations the backward step re-reads: A1 N1 N3 R Z NN GHN NO (64 each)
// and 8 scalars (rstd1, rstd3, rstd_rnn, mask, -).  A wide policy head (9..64 actions, NB = 64) appends dL/dlogits as
// a 64-vector at [TAPE_W, TAPE_WIDE); the 8-wide TP_DLOG field is left unused there.  A DiagGaussian policy head (1..8
// dimensions, NB = 8) keeps dL/dmean in TP_DLOG and appends the row's dL/dlogstd at [TAPE_W, TAPE_GAUSS).
//
// Head width bound NB (a template parameter): NB = 8 (MAXN) stages an 8-row head block and reduces each logit with a
// warp_sum into out[R][8] on every lane.  NB = 64 (MAXN_WIDE) treats the logits as one more lane-owned 64-vector
// (lane l owns actions l and l + 32): matvec64 over a 64-row head block whose rows >= n and bias entries >= n are zero.
// Per-lane arrays of 64 logits would spill under the 128-register cap of the 512-thread kernels.
//
// Observation width bound DX (a template parameter of step_forward): DX = 64 (H) takes x as a V2 and stages W1 at LD.
// DX = 256 (MAXD_WIDE, observations of 65..256 features): a row's x is loaded from global memory straight into its
// scratch row (SCR = 256 floats), W1 is staged at the odd leading dimension w1_ld(d) = pad4(d) + 1 (load_net<NB, 256>) and
// fc1 is matvec64 with K = pad4(d).  With a tape, x also goes to an X field of MAXD_WIDE floats appended to the row
// (tape_width_x), the Q operand of the 64-column panels of dW1; TQ_X is left unused there.  Only fc1 depends on d.
#pragma once
#include "orl_mlp.cuh"
#include "orl_rnn_core.h"

namespace orl_rnnw {
using orl::warp_sum;
namespace rc = orl_rnn;

constexpr int H = 64, G3 = 192, LD = 65, MAXN = 8, MAXN_WIDE = 64;
constexpr int TW_A1 = rc::TAPE, TW_N1 = TW_A1 + 64, TW_N3 = TW_N1 + 64, TW_R = TW_N3 + 64, TW_Z = TW_R + 64, TW_NN = TW_Z + 64,
              TW_GHN = TW_NN + 64, TW_NO = TW_GHN + 64, TW_SC = TW_NO + 64, TAPE_W = TW_SC + 8;   // 1744
constexpr int TW_DLW = TAPE_W, TAPE_WIDE = TW_DLW + 64;   // 1808: the wide policy head's dL/dlogits (P operand of Wh, bh)
constexpr int TW_DLS = TAPE_W, TAPE_GAUSS = TW_DLS + 8;   // 1752: a DiagGaussian policy head's dL/dlogstd (column sums)
__host__ __device__ constexpr int head_bound(int n) { return n > MAXN ? MAXN_WIDE : MAXN; }
// the row width before the X field: it depends on the head kind as well as on n
__host__ __device__ constexpr int tape_width(int n, bool gauss = false) { return gauss ? TAPE_GAUSS : n > MAXN ? TAPE_WIDE : TAPE_W; }
constexpr int MAXD_WIDE = 256;
__host__ __device__ constexpr int w1_ld(int d) { return ((d + 3) & ~3) + 1; }
// a wide-observation row (d > 64): the X field [tape_width(n, gauss), tape_width(n, gauss) + MAXD_WIDE) follows the row
__host__ __device__ constexpr int tape_width_x(int n, int d, bool gauss = false) { return tape_width(n, gauss) + (d > H ? MAXD_WIDE : 0); }

struct V2 { float a, b; };

struct SmemNet {
    const float *w1, *w3, *wih, *whh, *wh;                                  // [rows][LD]
    const float *b1, *g1, *be1, *b3, *g3, *be3, *bih, *bhh, *gr, *ber, *bh;  // vectors
};
// shared-memory floats of one net staged by load_net<NB, DX>: W1 at LD (DX = 64) or at w1_ld(d) (DX = 256), then the rest
template <int NB = MAXN, int DX = H>
__host__ __device__ constexpr int smem_net_floats(int d) {
    return (H + H + G3 + G3 + NB) * LD + 8 * H + 2 * G3 + NB + (DX == H ? 0 : H * (w1_ld(d) - LD));
}

// Stage one net (flat layout of rc::rnn_offsets) into shared memory; W1 columns k >= d and head rows m >= n are zero.
// DX = 64: W1 at LD, staged in one loop with W3.  DX = 256: W1 [64][w1_ld(d)].
template <int NB = MAXN, int DX = H>
__device__ inline SmemNet load_net(float* s, const float* __restrict__ P, const rc::Offsets& o, int tid, int nthreads) {
    static_assert(NB == MAXN || NB == MAXN_WIDE, "head width bound");
    static_assert(DX == H || DX == MAXD_WIDE, "observation width bound");
    const int ld1 = DX == H ? LD : w1_ld(o.d);
    float* w1 = s; s += H * ld1;
    float* w3 = s; s += H * LD;
    float* wih = s; s += G3 * LD;
    float* whh = s; s += G3 * LD;
    float* wh = s; s += NB * LD;
    float* vec = s;   // b1 g1 be1 b3 g3 be3 gr ber (64 each) | bih bhh (192 each) | bh (NB)
    if constexpr (DX == H) {
        for (int i = tid; i < H * LD; i += nthreads) {
            const int j = i / LD, k = i % LD;
            w1[i] = k < o.d ? P[o.w1 + j * o.d + k] : 0.f;
            w3[i] = k < H ? P[o.w3 + j * H + k] : 0.f;
        }
    } else {
        for (int i = tid; i < H * ld1; i += nthreads) {
            const int j = i / ld1, k = i % ld1;
            w1[i] = k < o.d ? P[o.w1 + j * o.d + k] : 0.f;
        }
        for (int i = tid; i < H * LD; i += nthreads) {
            const int j = i / LD, k = i % LD;
            w3[i] = k < H ? P[o.w3 + j * H + k] : 0.f;
        }
    }
    for (int i = tid; i < G3 * LD; i += nthreads) {
        const int j = i / LD, k = i % LD;
        wih[i] = k < H ? P[o.wih + j * H + k] : 0.f;
        whh[i] = k < H ? P[o.whh + j * H + k] : 0.f;
    }
    for (int i = tid; i < NB * LD; i += nthreads) {
        const int j = i / LD, k = i % LD;
        wh[i] = (j < o.n && k < H) ? P[o.wh + j * H + k] : 0.f;
    }
    for (int i = tid; i < H; i += nthreads) {
        vec[i] = P[o.b1 + i]; vec[H + i] = P[o.g1 + i]; vec[2 * H + i] = P[o.be1 + i];
        vec[3 * H + i] = P[o.b3 + i]; vec[4 * H + i] = P[o.g3 + i]; vec[5 * H + i] = P[o.be3 + i];
        vec[6 * H + i] = P[o.gr + i]; vec[7 * H + i] = P[o.ber + i];
    }
    for (int i = tid; i < G3; i += nthreads) { vec[8 * H + i] = P[o.bih + i]; vec[8 * H + G3 + i] = P[o.bhh + i]; }
    for (int i = tid; i < NB; i += nthreads) vec[8 * H + 2 * G3 + i] = i < o.n ? P[o.bh + i] : 0.f;
    SmemNet n;
    n.w1 = w1; n.w3 = w3; n.wih = wih; n.whh = whh; n.wh = wh;
    n.b1 = vec; n.g1 = vec + H; n.be1 = vec + 2 * H; n.b3 = vec + 3 * H; n.g3 = vec + 4 * H; n.be3 = vec + 5 * H;
    n.gr = vec + 6 * H; n.ber = vec + 7 * H; n.bih = vec + 8 * H; n.bhh = vec + 8 * H + G3; n.bh = vec + 8 * H + 2 * G3;
    return n;
}

__device__ __forceinline__ V2 ldv(const float* p, int lane) { return V2{p[lane], p[lane + 32]}; }
__device__ __forceinline__ void stv(float* p, int lane, V2 v) { p[lane] = v.a; p[lane + 32] = v.b; }

constexpr int SCR = 256;   // per-row scratch floats in shared memory: slot A [0,64), slot B [64,256)
__host__ __device__ constexpr int smem_scratch_floats(int warps, int R) { return warps * R * SCR; }

// normalised = (v - mean) * rstd over the 64 elements
__device__ __forceinline__ V2 ln_fwd(V2 v, float& rstd) {
    const float m = warp_sum(v.a + v.b) * (1.f / H);
    const float da = v.a - m, db = v.b - m;
    const float q = warp_sum(da * da + db * db) * (1.f / H);
    rstd = 1.f / sqrtf(q + rc::LN_EPS);
    return V2{da * rstd, db * rstd};
}
__device__ __forceinline__ V2 ln_bwd(V2 dn, V2 n, float rstd) {
    const float s1 = warp_sum(dn.a + dn.b) * (1.f / H);
    const float s2 = warp_sum(dn.a * n.a + dn.b * n.b) * (1.f / H);
    return V2{rstd * (dn.a - s1 - n.a * s2), rstd * (dn.b - s1 - n.b * s2)};
}

// Park the R lane-distributed 64-vectors in scratch slot `off` (row r at scr + r*SCR + off).
template <int R>
__device__ __forceinline__ void park(float* scr, int off, const V2 (&v)[R], int lane) {
    __syncwarp();   // every lane is done reading what the slot held before
#pragma unroll
    for (int r = 0; r < R; ++r) stv(scr + r * SCR + off, lane, v[r]);
    __syncwarp();
}

// out[r]_j = bias_j + sum_{k<K4} W[j][k] * in[r][k]; lane owns rows j = lane, lane+32 of the 64-row block at W (leading
// dimension ld, odd); in = scratch slot (K4 = K rounded up to 4: the inputs / weight columns beyond K are zero).
template <int R>
__device__ __forceinline__ void matvec64(const float* W, const float* bias, const float* scr, int off, int K, int lane, V2 (&out)[R],
                                         int ld = LD) {
    float s0[R], s1[R];
#pragma unroll
    for (int r = 0; r < R; ++r) { s0[r] = bias[lane]; s1[r] = bias[lane + 32]; }
    const float* r0 = W + lane * ld;
    const float* r1 = W + (lane + 32) * ld;
    const int K4 = (K + 3) & ~3;
    for (int k = 0; k < K4; k += 4) {
        const float w00 = r0[k], w01 = r0[k + 1], w02 = r0[k + 2], w03 = r0[k + 3];
        const float w10 = r1[k], w11 = r1[k + 1], w12 = r1[k + 2], w13 = r1[k + 3];
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const float4 v = *reinterpret_cast<const float4*>(scr + r * SCR + off + k);
            s0[r] = fmaf(w00, v.x, s0[r]); s0[r] = fmaf(w01, v.y, s0[r]); s0[r] = fmaf(w02, v.z, s0[r]); s0[r] = fmaf(w03, v.w, s0[r]);
            s1[r] = fmaf(w10, v.x, s1[r]); s1[r] = fmaf(w11, v.y, s1[r]); s1[r] = fmaf(w12, v.z, s1[r]); s1[r] = fmaf(w13, v.w, s1[r]);
        }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) out[r] = V2{s0[r], s1[r]};
}
// the three gate blocks (r, z, n) of a [192][64] matrix: three 64-row passes over the same parked input
template <int R>
__device__ __forceinline__ void matvec192(const float* W, const float* bias, const float* scr, int off, int lane, V2 (&out)[3][R]) {
#pragma unroll
    for (int g = 0; g < 3; ++g) matvec64<R>(W + g * H * LD, bias + g * H, scr, off, H, lane, out[g]);
}
// out[r]_k = sum_{j<J} W[j][k] * in[r][j]; lane owns columns k = lane, lane+32; in = scratch slot of J floats
template <int R>
__device__ __forceinline__ void matvecT(const float* W, const float* scr, int off, int J, int lane, V2 (&out)[R]) {
    float s0[R], s1[R];
#pragma unroll
    for (int r = 0; r < R; ++r) { s0[r] = 0.f; s1[r] = 0.f; }
    for (int j = 0; j < J; j += 4) {
        const float* w = W + j * LD + lane;
        const float w00 = w[0], w01 = w[LD], w02 = w[2 * LD], w03 = w[3 * LD];
        const float w10 = w[32], w11 = w[LD + 32], w12 = w[2 * LD + 32], w13 = w[3 * LD + 32];
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const float4 v = *reinterpret_cast<const float4*>(scr + r * SCR + off + j);
            s0[r] = fmaf(w00, v.x, s0[r]); s0[r] = fmaf(w01, v.y, s0[r]); s0[r] = fmaf(w02, v.z, s0[r]); s0[r] = fmaf(w03, v.w, s0[r]);
            s1[r] = fmaf(w10, v.x, s1[r]); s1[r] = fmaf(w11, v.y, s1[r]); s1[r] = fmaf(w12, v.z, s1[r]); s1[r] = fmaf(w13, v.w, s1[r]);
        }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) out[r] = V2{s0[r], s1[r]};
}

__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + expf(-x)); }

// ---- the wide head's row reductions over lane-owned logits (lane l: action l in .a, action l + 32 in .b) ----
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// x_j of one action j (the same j on every lane), on every lane
__device__ __forceinline__ float warp_pick(V2 x, int j) { return __shfl_sync(0xffffffffu, j < 32 ? x.a : x.b, j & 31); }
// index of the first maximum of the lane-owned values over the actions marked ok (action 0 always is), on every lane
__device__ __forceinline__ int warp_argmax(V2 v, bool ok_a, bool ok_b, int lane) {
    float bv = ok_a ? v.a : -INFINITY;
    int bi = lane;
    if (ok_b && v.b > bv) { bv = v.b; bi = lane + 32; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    return bi;
}
// log-softmax of the logits of actions 0..n-1, masked in place (-6e4 where mask_row[j] == 0), the maths of
// log_softmax_n with the max and the sums as warp reductions: lse = mx + log sum exp(x - mx), mx2 = mx - lse (the max of
// the rounded x - lse, rounding being monotone), p = exp(x - lse - mx2) / s2.  Actions j >= n take no part.
struct WarpSoftmax {
    float lse, mx2, s2;
    bool in_a, in_b;       // this lane's actions are < n
    bool live_a, live_b;   // ... and legal
    __device__ __forceinline__ float nl(float x) const { return x - lse; }
    __device__ __forceinline__ float pr(float x) const { return expf(x - lse - mx2) / s2; }
};
__device__ __forceinline__ WarpSoftmax warp_log_softmax(V2& x, int n, const float* mask_row, int lane) {
    WarpSoftmax r;
    r.in_a = lane < n; r.in_b = lane + 32 < n;
    r.live_a = r.in_a; r.live_b = r.in_b;
    if (mask_row) {
        if (r.in_a && mask_row[lane] == 0.f) { x.a = -6e4f; r.live_a = false; }
        if (r.in_b && mask_row[lane + 32] == 0.f) { x.b = -6e4f; r.live_b = false; }
    }
    const float mx = warp_max(fmaxf(r.in_a ? x.a : -INFINITY, r.in_b ? x.b : -INFINITY));
    r.lse = mx + logf(warp_sum((r.in_a ? expf(x.a - mx) : 0.f) + (r.in_b ? expf(x.b - mx) : 0.f)));
    r.mx2 = mx - r.lse;
    r.s2 = warp_sum((r.in_a ? expf(x.a - r.lse - r.mx2) : 0.f) + (r.in_b ? expf(x.b - r.lse - r.mx2) : 0.f));
    return r;
}

// head outputs of one row: NB = 8, out[m] for m < n on every lane; NB = 64, the lane-owned logits
template <int NB> struct HeadOut { using type = float[MAXN]; };
template <> struct HeadOut<MAXN_WIDE> { using type = V2; };
// observation of one row: DX = 64, lane-owned (zero beyond d); DX = 256, the row's d floats in global memory
template <int DX> struct XIn { using type = V2; };
template <> struct XIn<MAXD_WIDE> { using type = const float*; };

// Load R observation rows of d <= 256 features into their scratch rows, zero from d up to the end of the last 64-column
// panel; with a tape, also into its X field at xoff (the Q operand of the dW1 panels: every column a panel reads is finite).
template <int R>
__device__ __forceinline__ void stage_x(float* scr, const float* const (&x)[R], int d, float* const (&tape)[R], int xoff, int lane) {
    const int kp = (d + 63) & ~63;
    __syncwarp();   // every lane is done reading what the scratch held before
#pragma unroll
    for (int r = 0; r < R; ++r) {
        for (int k = lane; k < kp; k += 32) {
            const float v = k < d ? x[r][k] : 0.f;
            scr[r * SCR + k] = v;
            if (tape[r]) tape[r][xoff + k] = v;
        }
    }
    __syncwarp();
}

// One forward step of R rows.  x: observation (XIn; zero beyond d), h_in: hidden state, out[r]: the head outputs (HeadOut).
// tape[r] != nullptr: the Q operands and the activations for the backward step go to the row's tape.
// scr: this warp's scratch (R * SCR floats of shared memory).  W: staged by load_net<NB, DX>.  GAUSS: a DiagGaussian
// policy head (NB = 8), whose rows put the X field after TW_DLS.
template <int R, int NB = MAXN, int DX = H, bool GAUSS = false>
__device__ __forceinline__ void step_forward(const SmemNet& W, float* scr, int d, int n, int act_id, const typename XIn<DX>::type (&x)[R],
                                             const V2 (&h_in)[R], const float (&mask)[R], V2 (&h_out)[R],
                                             typename HeadOut<NB>::type (&out)[R], float* const (&tape)[R], int lane) {
    static_assert(DX == H || DX == MAXD_WIDE, "observation width bound");
    static_assert(!GAUSS || NB == MAXN, "a DiagGaussian head has up to 8 dimensions");
    const V2 g1 = ldv(W.g1, lane), be1 = ldv(W.be1, lane), g3 = ldv(W.g3, lane), be3 = ldv(W.be3, lane);
    V2 t0[R], y1[R], y3[R], hm[R];
    if constexpr (DX == H) {
        park<R>(scr, 0, x, lane);
        matvec64<R>(W.w1, W.b1, scr, 0, d, lane, t0);
    } else {
        stage_x<R>(scr, x, d, tape, GAUSS ? TAPE_GAUSS : NB == MAXN ? TAPE_W : TAPE_WIDE, lane);
        matvec64<R>(W.w1, W.b1, scr, 0, d, lane, t0, w1_ld(d));
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const V2 a1{rc::act_fwd(t0[r].a, act_id), rc::act_fwd(t0[r].b, act_id)};
        float rstd1;
        const V2 n1 = ln_fwd(a1, rstd1);
        y1[r] = V2{fmaf(n1.a, g1.a, be1.a), fmaf(n1.b, g1.b, be1.b)};
        if (tape[r]) {
            if constexpr (DX == H) stv(tape[r] + rc::TQ_X, lane, x[r]);
            stv(tape[r] + TW_A1, lane, a1); stv(tape[r] + TW_N1, lane, n1);
            stv(tape[r] + rc::TQ_Y1, lane, y1[r]);
            if (lane == 0) { tape[r][TW_SC] = rstd1; tape[r][TW_SC + 3] = mask[r]; }
        }
    }
    park<R>(scr, 0, y1, lane);
    matvec64<R>(W.w3, W.b3, scr, 0, H, lane, t0);
#pragma unroll
    for (int r = 0; r < R; ++r) {
        float rstd3;
        const V2 n3 = ln_fwd(t0[r], rstd3);
        y3[r] = V2{fmaf(n3.a, g3.a, be3.a), fmaf(n3.b, g3.b, be3.b)};
        hm[r] = V2{h_in[r].a * mask[r], h_in[r].b * mask[r]};
        if (tape[r]) {
            stv(tape[r] + TW_N3, lane, n3); stv(tape[r] + rc::TQ_Y3, lane, y3[r]); stv(tape[r] + rc::TQ_HM, lane, hm[r]);
            if (lane == 0) tape[r][TW_SC + 1] = rstd3;
        }
    }
    V2 gi[3][R], gh[3][R];
    park<R>(scr, 0, y3, lane);
    matvec192<R>(W.wih, W.bih, scr, 0, lane, gi);
    park<R>(scr, 0, hm, lane);
    matvec192<R>(W.whh, W.bhh, scr, 0, lane, gh);
    const V2 gr = ldv(W.gr, lane), ber = ldv(W.ber, lane);
    [[maybe_unused]] V2 ov[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const V2 rg{sigm(gi[0][r].a + gh[0][r].a), sigm(gi[0][r].b + gh[0][r].b)};
        const V2 z{sigm(gi[1][r].a + gh[1][r].a), sigm(gi[1][r].b + gh[1][r].b)};
        const V2 nn{tanhf(fmaf(rg.a, gh[2][r].a, gi[2][r].a)), tanhf(fmaf(rg.b, gh[2][r].b, gi[2][r].b))};
        h_out[r] = V2{fmaf(z.a, hm[r].a, (1.f - z.a) * nn.a), fmaf(z.b, hm[r].b, (1.f - z.b) * nn.b)};
        float rstdr;
        const V2 no = ln_fwd(h_out[r], rstdr);
        const V2 o{fmaf(no.a, gr.a, ber.a), fmaf(no.b, gr.b, ber.b)};
        if constexpr (NB == MAXN) {
#pragma unroll
            for (int m = 0; m < MAXN; ++m) {
                out[r][m] = 0.f;
                if (m < n) out[r][m] = W.bh[m] + warp_sum(fmaf(W.wh[m * LD + lane], o.a, W.wh[m * LD + 32 + lane] * o.b));
            }
        } else {
            ov[r] = o;
        }
        if (tape[r]) {
            stv(tape[r] + rc::TQ_O, lane, o); stv(tape[r] + TW_R, lane, rg); stv(tape[r] + TW_Z, lane, z);
            stv(tape[r] + TW_NN, lane, nn); stv(tape[r] + TW_GHN, lane, gh[2][r]); stv(tape[r] + TW_NO, lane, no);
            if (lane == 0) tape[r][TW_SC + 2] = rstdr;
        }
    }
    if constexpr (NB == MAXN_WIDE) {   // logits = bh + Wh o over the 64-row head block (zero rows and bias beyond n)
        park<R>(scr, 0, ov, lane);
        matvec64<R>(W.wh, W.bh, scr, 0, H, lane, out);
    }
}

// Backward of one step of R rows from their tape rows (written by step_forward; dL/dout in TP_DLOG, or for NB = 64 the
// lane-owned 64-vector at TW_DLW, zero beyond n).  dh holds dL/dh_out arriving from the following step on entry and
// dL/dh_in (already multiplied by the mask) on exit; the P / S tape fields are written.
template <int R, int NB = MAXN>
__device__ __forceinline__ void step_backward(const SmemNet& W, float* scr, int n, int act_id, float* const (&tape)[R], V2 (&dh)[R], int lane) {
    const V2 gr = ldv(W.gr, lane), g3 = ldv(W.g3, lane), g1 = ldv(W.g1, lane);
    V2 dgi[3][R], dgh[3][R], dhm[R];
    float mask[R];
    [[maybe_unused]] V2 dovw[R];
    if constexpr (NB == MAXN_WIDE) {   // dL/do = Wh^T dL/dlogits over the pad4(n) head rows
        V2 dl[R];
#pragma unroll
        for (int r = 0; r < R; ++r) dl[r] = ldv(tape[r] + TW_DLW, lane);
        park<R>(scr, 0, dl, lane);
        matvecT<R>(W.wh, scr, 0, (n + 3) & ~3, lane, dovw);
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
        V2 dov{0.f, 0.f};
        float rstdr;
        if constexpr (NB == MAXN) {
            float dl[MAXN];
#pragma unroll
            for (int m = 0; m < MAXN; ++m) dl[m] = tape[r][rc::TP_DLOG + m];
            rstdr = tape[r][TW_SC + 2];
            mask[r] = tape[r][TW_SC + 3];
#pragma unroll
            for (int m = 0; m < MAXN; ++m)
                if (m < n) { dov.a = fmaf(W.wh[m * LD + lane], dl[m], dov.a); dov.b = fmaf(W.wh[m * LD + 32 + lane], dl[m], dov.b); }
        } else {
            rstdr = tape[r][TW_SC + 2];
            mask[r] = tape[r][TW_SC + 3];
            dov = dovw[r];
        }
        const V2 no = ldv(tape[r] + TW_NO, lane);
        stv(tape[r] + rc::TS_DONO, lane, V2{dov.a * no.a, dov.b * no.b});
        stv(tape[r] + rc::TS_DO, lane, dov);
        V2 d = ln_bwd(V2{dov.a * gr.a, dov.b * gr.b}, no, rstdr);
        d.a += dh[r].a; d.b += dh[r].b;
        const V2 rg = ldv(tape[r] + TW_R, lane), z = ldv(tape[r] + TW_Z, lane), nn = ldv(tape[r] + TW_NN, lane);
        const V2 ghn = ldv(tape[r] + TW_GHN, lane), hm = ldv(tape[r] + rc::TQ_HM, lane);
        const float dhv[2] = {d.a, d.b}, rv[2] = {rg.a, rg.b}, zv[2] = {z.a, z.b}, nv[2] = {nn.a, nn.b};
        const float gv[2] = {ghn.a, ghn.b}, hv[2] = {hm.a, hm.b};
        float o_r[2], o_z[2], o_n[2], o_hn[2], o_hm[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const float dnn = dhv[e] * (1.f - zv[e]), dz = dhv[e] * (hv[e] - nv[e]);
            o_hm[e] = dhv[e] * zv[e];
            const float dnpre = dnn * (1.f - nv[e] * nv[e]);
            const float dr = dnpre * gv[e];
            o_z[e] = dz * zv[e] * (1.f - zv[e]);
            o_r[e] = dr * rv[e] * (1.f - rv[e]);
            o_n[e] = dnpre;
            o_hn[e] = dnpre * rv[e];
        }
        dgi[0][r] = V2{o_r[0], o_r[1]}; dgi[1][r] = V2{o_z[0], o_z[1]}; dgi[2][r] = V2{o_n[0], o_n[1]};
        dgh[0][r] = dgi[0][r]; dgh[1][r] = dgi[1][r]; dgh[2][r] = V2{o_hn[0], o_hn[1]};
        dhm[r] = V2{o_hm[0], o_hm[1]};
#pragma unroll
        for (int g = 0; g < 3; ++g) { stv(tape[r] + rc::TP_DGI + g * H, lane, dgi[g][r]); stv(tape[r] + rc::TP_DGH + g * H, lane, dgh[g][r]); }
    }
    V2 dy3[R], t[R], dz3[R], dy1[R];
#pragma unroll
    for (int g = 0; g < 3; ++g) park<R>(scr, 64 + g * H, dgi[g], lane);
    matvecT<R>(W.wih, scr, 64, G3, lane, dy3);
#pragma unroll
    for (int g = 0; g < 3; ++g) park<R>(scr, 64 + g * H, dgh[g], lane);
    matvecT<R>(W.whh, scr, 64, G3, lane, t);
#pragma unroll
    for (int r = 0; r < R; ++r) {
        dh[r] = V2{(dhm[r].a + t[r].a) * mask[r], (dhm[r].b + t[r].b) * mask[r]};
        const float rstd3 = tape[r][TW_SC + 1];
        const V2 n3 = ldv(tape[r] + TW_N3, lane);
        stv(tape[r] + rc::TS_DY3N3, lane, V2{dy3[r].a * n3.a, dy3[r].b * n3.b});
        stv(tape[r] + rc::TS_DY3, lane, dy3[r]);
        dz3[r] = ln_bwd(V2{dy3[r].a * g3.a, dy3[r].b * g3.b}, n3, rstd3);
        stv(tape[r] + rc::TP_DZ3, lane, dz3[r]);
    }
    park<R>(scr, 0, dz3, lane);
    matvecT<R>(W.w3, scr, 0, H, lane, dy1);
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const float rstd1 = tape[r][TW_SC];
        const V2 n1 = ldv(tape[r] + TW_N1, lane), a1 = ldv(tape[r] + TW_A1, lane);
        stv(tape[r] + rc::TS_DY1N1, lane, V2{dy1[r].a * n1.a, dy1[r].b * n1.b});
        stv(tape[r] + rc::TS_DY1, lane, dy1[r]);
        const V2 da1 = ln_bwd(V2{dy1[r].a * g1.a, dy1[r].b * g1.b}, n1, rstd1);
        stv(tape[r] + rc::TP_DZ1, lane, V2{da1.a * rc::act_bwd_from_out(a1.a, act_id), da1.b * rc::act_bwd_from_out(a1.b, act_id)});
    }
}

}  // namespace orl_rnnw
