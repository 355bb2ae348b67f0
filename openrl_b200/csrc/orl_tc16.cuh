// Split-fp16 operand primitives for the "2 x fp16" GEMMs of the PPO update and the forward passes (sm_90a wgmma),
// plus the TMA / cp.async staging primitives.
//
// Split: x = hi + lo, hi = fp16(x), lo = fp16(x - hi)  (22 significand bits);  A.B ~= Al.Bh + Ah.Bl + Ah.Bh
// accumulated in fp32: on 64..256-long dot products the error is at or below that of an fp32 FFMA chain, i.e. the
// tensor-core path keeps the 1e-4 loss-parity bar.
//
// Operand buffer ("row-major panel buffer"): a matrix of R rows x F fp16 features is stored as F/8 panels;
// panel p holds features [8p, 8p+8) of every row as R consecutive 16-byte units:
//        element (row r, feature f) at  (f/8) * R*16 + r*16 + (f%8)*2.
// A thread that owns a row writes 16-byte vectors (conflict-free: consecutive rows are consecutive units).
// The SAME buffer is read by the tensor core in both majors, by descriptor only (no transposed copies); every
// 8 x 16-byte block is one core matrix of the no-swizzle layout:
//   * K-major  (rows = M/N index, features = K): LBO = R*16 (next 8 features), SBO = 128 (next 8 rows);
//     the k-slice of one MMA (K = 16) starts at panel k0/8, the 64-row block m0 at byte m0*16.
//   * MN-major (rows = K index, features = M/N): SBO = R*16 (next 8 features along M/N), LBO = 128 (next 8
//     rows along K); the k-slice of one MMA starts at row r0, the 64-feature block m0 at panel m0/8.
#pragma once
#include <cuda_fp16.h>

#include "orl_mlp.cuh"
#include "orl_tc.cuh"

namespace orl {
namespace tc {

constexpr uint32_t W_PANEL = H * 16;   // one panel of the W3f hi / lo buffers: 8 features of the 64 fc3 output rows

// wgmma descriptor = constant part (LBO, SBO; layout type 0 = no swizzle) | start address
__device__ __forceinline__ uint64_t desc_const(uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) | ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32);
}
__device__ __forceinline__ uint64_t desc_at(uint64_t dconst, uint32_t smem_addr) { return dconst | (uint64_t)((smem_addr >> 4) & 0x3FFF); }

// two floats -> packed fp16 pairs (hi, lo) of the split; round-to-nearest, saturating (no inf)
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(b), "f"(a));   // d = {hi half: first src, lo half: second src}
    const __half2 h = *reinterpret_cast<const __half2*>(&hi);
    const float2 hf = __half22float2(h);
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(b - hf.y), "f"(a - hf.x));
}
// 8 consecutive features of one row -> one 16-byte unit of the hi buffer and one of the lo buffer
__device__ __forceinline__ void split_store8(uint8_t* hi_unit, uint8_t* lo_unit, const float* v, float scale) {
    uint4 h, l;
    split2(v[0] * scale, v[1] * scale, h.x, l.x);
    split2(v[2] * scale, v[3] * scale, h.y, l.y);
    split2(v[4] * scale, v[5] * scale, h.z, l.z);
    split2(v[6] * scale, v[7] * scale, h.w, l.w);
    *reinterpret_cast<uint4*>(hi_unit) = h;
    *reinterpret_cast<uint4*>(lo_unit) = l;
}

// Stage one net's folded weights for the tensor-core kernels; all nt threads of the CTA call it, no barrier.  Writes the
// fp32 block w1t[8][64] (k-major, zero padded) b1[64] b3f[64] whf[8][64] bhf[8] at `small`, and W3f as 8 split-fp16
// panels of 64 rows at Wh / Wl.
__device__ __forceinline__ void stage_weights_tc(float* small, uint8_t* Wh, uint8_t* Wl, const float* __restrict__ params, int d, int n,
                                                 int nt) {
    const int tid = threadIdx.x;
    const NetOffsets po = net_offsets(d, n);
    float* w1t = small; float* b1 = w1t + 8 * H; float* b3f = b1 + H; float* whf = b3f + H; float* bhf = whf + MAX_OUT * H;
    for (int i = tid; i < 8 * H; i += nt) { const int k = i / H, j = i % H; w1t[i] = (k < d) ? params[po.w1 + j * d + k] : 0.f; }
    for (int i = tid; i < H; i += nt) b1[i] = params[po.b1 + i];
    for (int i = tid; i < H * 8; i += nt) {   // item = (panel p, row j): lanes own consecutive rows -> conflict-free 16-byte stores
        const int pnl = i / H, j = i % H;
        float w8[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) w8[c] = folded_w3(params, po, j, 8 * pnl + c);
        const uint32_t off = (uint32_t)pnl * W_PANEL + j * 16;
        split_store8(Wh + off, Wl + off, w8, 1.0f);
    }
    for (int i = tid; i < MAX_OUT * H; i += nt) whf[i] = folded_wh(params, po, i / H, i % H);
    for (int j = tid; j < H; j += nt) b3f[j] = folded_b3(params, po, j);
    for (int j = tid; j < MAX_OUT; j += nt) bhf[j] = folded_bh(params, po, j);
}

// ---- the per-row forward of the tensor-core kernels (update, critic values, rollouts) ----------------------------------
// A row is owned by 64 / CW threads of one warp, each holding the CW consecutive hidden columns [cb, cb + CW):
//   CW = 32, halves  : warp w owns tile rows [16w, +16), lane l row 16w + l % 16, half l / 16 (the rows of warp w's
//                      slice of the wgmma accumulator fragment, so Z3 reaches its row owners within the warp);
//   CW = 16, quarters: lane 4r + qd holds row r of the warp, quarter qd (the CartPole rollout).
// The row functions compute over the thread's columns; the row's threads combine their partials between the calls
// (row_sum_stats, row_sum_head), in one fixed order per layout, so every thread of a row holds the same statistics.
constexpr int S_LD = 68;   // row pitch of the fp32 staging tile of Z3 (floats): the row-per-thread float4 reads are conflict-free

#define FOR_OUT(j) _Pragma("unroll") for (int j = 0; j < NOUT; ++j) if (NOUT != 8 || j < n)

// ACT == 1: ReLU (the reference's default activation_id) compiled in; ACT == -1: runtime activation_id (tanh / leaky / elu
// expand to ~60 instructions per element, which the fully unrolled row code cannot afford in the instruction cache)
template <int ACT>
__device__ __forceinline__ float act_tc(float z, int activation_id) { return ACT == 1 ? fmaxf(z, 0.f) : act_fwd(z, activation_id); }

// barrier of this thread's warpgroup (named barriers 1 and 2)
__device__ __forceinline__ void warpgroup_sync(int g) { asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory"); }

// the row's partial sums -> the whole row's, on every thread of the row.  Halves: own + other (lane l ^ 16); quarters:
// (((0 + p0) + p1) + p2) + p3 over the lanes of the row
template <int CW>
__device__ __forceinline__ void row_sum_stats(float& s, float& sq) {
    if constexpr (CW == 32) {
        s += __shfl_xor_sync(0xffffffffu, s, 16); sq += __shfl_xor_sync(0xffffffffu, sq, 16);
    } else {
        const int qbase = (threadIdx.x & 31) & ~3;
        float ts = 0.f, tq = 0.f;
#pragma unroll
        for (int p = 0; p < 4; ++p) { ts += __shfl_sync(0xffffffffu, s, qbase + p); tq += __shfl_sync(0xffffffffu, sq, qbase + p); }
        s = ts; sq = tq;
    }
}
// the row's partial head dots -> the whole row's.  Halves: own + other; quarters: (p0 + p1) + (p2 + p3)
template <int CW, int NOUT>
__device__ __forceinline__ void row_sum_head(float (&out)[MAX_OUT], int n) {
    if constexpr (CW == 32) {
        FOR_OUT(j) out[j] += __shfl_xor_sync(0xffffffffu, out[j], 16);
    } else {
        const int qbase = (threadIdx.x & 31) & ~3;
        FOR_OUT(j) {
            const float p0 = __shfl_sync(0xffffffffu, out[j], qbase), p1 = __shfl_sync(0xffffffffu, out[j], qbase + 1);
            const float p2 = __shfl_sync(0xffffffffu, out[j], qbase + 2), p3 = __shfl_sync(0xffffffffu, out[j], qbase + 3);
            out[j] = (p0 + p1) + (p2 + p3);
        }
    }
}

// LayerNorm statistics of a 64-wide row from its sum and sum of squares
struct LnStats {
    float mu, var, rstd;   // var includes LN_EPS
};
__device__ __forceinline__ LnStats ln_stats(float s, float sq) {
    LnStats l;
    l.mu = s * (1.f / H);
    l.var = fmaxf(sq * (1.f / H) - l.mu * l.mu, 0.f) + LN_EPS;
    l.rstd = 1.0f / sqrtf(l.var);
    return l;
}

// fc1 (K = d <= 8) + activation over this thread's columns, and their LayerNorm-1 partial sums.  Returns the sign bits of
// the pre-activations (bit i: column cb + i), which the activation backward of the update needs.
template <int CW, int ACT>
__device__ __forceinline__ unsigned row_fc1(const float (&x)[8], int d, const float* w1t, const float* b1s, int cb, int activation_id,
                                            float (&n1)[CW], float& s, float& sq) {
#pragma unroll
    for (int q4 = 0; q4 < CW; q4 += 4) {
        const float4 b = *reinterpret_cast<const float4*>(b1s + cb + q4);
        n1[q4] = b.x; n1[q4 + 1] = b.y; n1[q4 + 2] = b.z; n1[q4 + 3] = b.w;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        if (k < d) {
#pragma unroll
            for (int q4 = 0; q4 < CW; q4 += 4) {
                const float4 wv = *reinterpret_cast<const float4*>(w1t + k * H + cb + q4);
                n1[q4] = fmaf(x[k], wv.x, n1[q4]); n1[q4 + 1] = fmaf(x[k], wv.y, n1[q4 + 1]);
                n1[q4 + 2] = fmaf(x[k], wv.z, n1[q4 + 2]); n1[q4 + 3] = fmaf(x[k], wv.w, n1[q4 + 3]);
            }
        }
    }
    unsigned posmask = 0u;
    s = 0.f; sq = 0.f;
#pragma unroll
    for (int i = 0; i < CW; ++i) {
        if (n1[i] > 0.f) posmask |= 1u << i;
        n1[i] = act_tc<ACT>(n1[i], activation_id);
        s += n1[i]; sq = fmaf(n1[i], n1[i], sq);
    }
    return posmask;
}

// LayerNorm-1 normalise of this thread's columns, stored as split fp16 into the n1 panels (`panel` bytes per panel)
template <int CW>
__device__ __forceinline__ void row_ln1_store(float (&n1)[CW], const LnStats& l, uint8_t* R1h, uint8_t* R1l, uint32_t panel, int row, int cb) {
#pragma unroll
    for (int i = 0; i < CW; ++i) n1[i] = (n1[i] - l.mu) * l.rstd;
#pragma unroll
    for (int q8 = 0; q8 < CW; q8 += 8) {
        const uint32_t off = (uint32_t)((cb + q8) >> 3) * panel + row * 16;
        split_store8(R1h + off, R1l + off, n1 + q8, 1.0f);
    }
}

// this thread's columns of Z3 from the staging tile, + b3f, and their LayerNorm-3 partial sums
template <int CW>
__device__ __forceinline__ void row_z3(const float* S, int row, int cb, const float* b3f, float (&n3)[CW], float& s, float& sq) {
#pragma unroll
    for (int q4 = 0; q4 < CW; q4 += 4) {
        const float4 v = *reinterpret_cast<const float4*>(S + row * S_LD + cb + q4);
        n3[q4] = v.x; n3[q4 + 1] = v.y; n3[q4 + 2] = v.z; n3[q4 + 3] = v.w;
    }
    s = 0.f; sq = 0.f;
#pragma unroll
    for (int i = 0; i < CW; ++i) { n3[i] += b3f[cb + i]; s += n3[i]; sq = fmaf(n3[i], n3[i], sq); }
}

// LayerNorm-3 normalise of this thread's columns and the partial head dots over them (out[j] = 0 for the unused heads)
template <int CW, int NOUT>
__device__ __forceinline__ void row_head(float (&n3)[CW], const LnStats& l, const float* whf, int cb, int n, float (&out)[MAX_OUT]) {
#pragma unroll
    for (int j = 0; j < MAX_OUT; ++j) out[j] = 0.f;
#pragma unroll
    for (int q4 = 0; q4 < CW; q4 += 4) {
#pragma unroll
        for (int i = 0; i < 4; ++i) n3[q4 + i] = (n3[q4 + i] - l.mu) * l.rstd;
        FOR_OUT(j) {
            const float4 wv = *reinterpret_cast<const float4*>(whf + j * H + cb + q4);
            out[j] = fmaf(n3[q4], wv.x, fmaf(n3[q4 + 1], wv.y, fmaf(n3[q4 + 2], wv.z, fmaf(n3[q4 + 3], wv.w, out[j]))));
        }
    }
}

// ---- TMA (cp.async.bulk.tensor) + mbarrier transaction accounting ----
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* dst, const void* tmap, int c0, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.1d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2}], [%3];" ::"r"(smem_u32(dst)),
                 "l"(tmap), "r"(c0), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const void* tmap, int c0, int c1, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(smem_u32(dst)),
                 "l"(tmap), "r"(c0), "r"(c1), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) { asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory"); }

// ---- per-thread asynchronous global -> shared copies (gathered minibatch rows) ----
__device__ __forceinline__ void cp_async4(void* dst, const void* src, bool valid) {
    const int sz = valid ? 4 : 0;   // src-size 0: zero fill, nothing is read
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async16(void* dst, const void* src, bool valid) {
    const int sz = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

}  // namespace tc
}  // namespace orl
