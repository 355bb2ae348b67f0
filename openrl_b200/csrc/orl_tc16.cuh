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

#include "orl_tc.cuh"

namespace orl {
namespace tc {

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
