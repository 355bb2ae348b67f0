// PPO minibatch forward+backward on the Hopper tensor cores (wgmma, split-fp16 operands, FP32
// accumulate) — produces the same folded partial gradients and loss sums as ppo_fwdbwd_kernel
// (orl_ppo.cu) at fp32-class accuracy (orl_tc16.cuh).  Selected with ORL_PPO_TENSORCORE; categorical
// heads, obs widths <= 8 (CartPole, GridWorld).  Reference: openrl/algorithms/ppo.py:46-361.
//
// CTA = 256 threads = 128 tile rows x 2 column halves = 2 warpgroups, one CTA per SM (~171 KB shared
// memory): warp w owns rows [16w, +16), lane l row 16w + l % 16 and columns [32 (l / 16), +32), so every
// row-wise operation (fc1 with K = d <= 8, LayerNorm forward/backward, head, loss) is thread-local apart
// from four exchanges with lane l ^ 16 (shuffles).  The per-tile GEMM results (Z3, dN1) arrive in the
// warpgroups' accumulator registers in the wgmma fragment layout, whose rows [16w, +16) sit in warp w, and
// reach the row-owning lanes through an fp32 staging tile in shared memory within the warp.  GEMM1 and
// GEMM2 read only the issuing warpgroup's rows (warpgroup barrier); GEMM3a / GEMM3b reduce over all 128
// rows (CTA barrier).  GEMM3a / GEMM3b have no consumer inside the tile loop: they stay in flight under
// the LayerNorm-1 backward and the next tile's staging wait, fc1 and activation, and are waited for just
// before the next tile overwrites R1.
//
// All matrix operands live in row-major panel buffers (orl_tc16.cuh) as fp16 hi/lo pairs, written by
// the row-owning threads with 16-byte stores and read K-major or MN-major by descriptor only:
//   R1 = [ n1 (8 panels) | CST = (1, mu3, std3, 0..) | X ]   rows = tile rows
//   R2 = [ dZ3 (8 panels) | U = dL * rstd3 ]                  rows = tile rows
//   R3 = [ dZ1 (8 panels) ]                                   rows = tile rows       (GEMM3a may still read R1)
//   W  = W3f [64 out rows][64 in features]
// Four GEMMs per 128-row tile, each as three MMA passes (Al.Bh, Ah.Bl, Ah.Bh), issued by one thread:
//   GEMM1  Z3 [128x64]  = n1 . W3f^T                 A = R1 K-major,  B = W K-major     (fwd fc3)
//   GEMM2  dN1[128x64]  = dZ3 . W3f                  A = R2 K-major,  B = W MN-major    (bwd-data fc3)
//   GEMM3a Ga [128x80] += R2^T . R1                  both MN-major, K = 128 tile rows (warpgroup g: rows [64g, +64)):
//            lanes 0..63  : G3 = dZ3^T n1 (cols 0..63), db3 (col 64 = the ones column)
//            lanes 64..71 : Q = U^T n1, su = U^T 1, smu = U^T mu3, sdl = U^T std3  (-> GH, dbh, below)
//   GEMM3b Gb [64x16]  += dZ1^T . [CST | X]          both MN-major: db1 (col 0), G1 = dZ1^T X (cols 8..15); warpgroup 1
// Ga / Gb stay in accumulator registers for the whole kernel.  GH = dL^T n3 needs no n3 tile: with n3 = (Z3 + b3f - mu3) rstd3
// and Z3 = n1 W3f^T,   GH[j][k] = sum_i Q[j][i] W3f[k][i] + b3f[k] su[j] - smu[j]   (evaluated once at the end).
// fp16 carries 22 significand bits as hi + lo only while hi >= 2^-3 (below, lo is subnormal), so every backward
// operand is scaled by a power of two chosen per minibatch to put its TYPICAL magnitude near 2^4: dZ3 / dZ1 by
// S_z ~ 8 rows / max|Whf| (head weights are tiny: gain 0.01), U by S_u ~ 8 rows, observations by 16; the accumulators
// are multiplied by the exact inverse when flushed, conversions saturate instead of overflowing.  `rows` is the count
// the row weights divide by: sum(active) of the minibatch when the net's active-mask option is on (a live row then
// weighs active / sum(active)), else the row count.  Headroom: a scaled operand reaches 65504 at ~2^12 times its
// typical size, i.e. when |dL/dlogit| x rstd3 of a row is ~4000 times that of a unit-advantage row.
//
// Minibatch tiles are staged in shared memory one tile ahead: TMA (cp.async.bulk.tensor: the 128 x d
// observation tile and the scalar columns, zero-filled past the end) when the minibatch is a contiguous
// row range, per-thread cp.async gathers when it is an index list (shuffled minibatches).
#include <cuda.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>

#include "orl_loss.cuh"
#include "orl_tc16.cuh"

namespace orl {
int ppo_stride_host(int obs_dim, int critic_obs_dim, int n_actions);
}

namespace {
using namespace orl;
using namespace orl::tc;

constexpr int T_M = 128, T_NT = 256;
constexpr int CW = 32;                         // columns per thread
constexpr uint32_t PANEL = T_M * 16;           // 8 fp16 features of 128 rows
constexpr int R1_PANELS = 10, R2_PANELS = 9, R3_PANELS = 8;
constexpr int P_CST = 8, P_X = 9, P_U = 8;
constexpr int N_LOSS_TC = 8;
// staging tile of the per-tile GEMM results: 128 rows x 64 fp32 at row pitch S_LD (orl_tc16.cuh);
// the final Ga [128][GA_LD] / Gb [64][GB_LD] staging reuses R1 / R2
constexpr int GA_LD = 84, GB_LD = 20;
// the fp32 W3f^T of the final GH contraction, in R3 at row pitch W3T_LD (conflict-free stores and reads)
constexpr int W3T_LD = 65;
// shared-memory carve-up (bytes)
constexpr uint32_t OFF_R1H = 0, OFF_R1L = OFF_R1H + R1_PANELS * PANEL, OFF_R2H = OFF_R1L + R1_PANELS * PANEL,
                   OFF_R2L = OFF_R2H + R2_PANELS * PANEL, OFF_WH = OFF_R2L + R2_PANELS * PANEL, OFF_WL = OFF_WH + 8 * W_PANEL,
                   OFF_R3H = OFF_WL + 8 * W_PANEL, OFF_R3L = OFF_R3H + R3_PANELS * PANEL,
                   OFF_S = OFF_R3L + R3_PANELS * PANEL, OFF_STAGE = OFF_S + T_M * S_LD * 4;
static_assert((T_M * GA_LD + 64 * GB_LD) * 4 <= OFF_WH, "the Ga / Gb staging fits in R1 + R2");
static_assert(OFF_STAGE % 128 == 0, "TMA destination alignment");
static_assert(H * W3T_LD * 4 <= OFF_S - OFF_R3H, "the W3f^T of the flush fits in R3");
static_assert(H * 8 + 6 * H + H * H + MAX_OUT * (H + 1) <= (OFF_S - OFF_R3H) / 4, "the parameter copy of the prologue fits in R3");
static_assert(OFF_R2L + 16 * PANEL <= OFF_R3H, "the 16-panel A descriptors of GEMM3a stop short of R3 (written while they run)");
constexpr int N_SCAL = 4;                      // scalar columns staged per row

struct TcMaps {   // TMA descriptors of the flattened rollout buffers (built by the launcher)
    CUtensorMap obs_p, obs_c, actions, old_logp, adv, value_preds, returns, active;
};

__host__ __device__ inline uint32_t tc_stage_bytes(int d) { return (uint32_t)((T_M * d * 4 + 127) & ~127) + N_SCAL * T_M * 4; }
__host__ __device__ inline uint32_t tc_small_off(int d) { return OFF_STAGE + tc_stage_bytes(d); }
// fp32 weights: w1t[8][64] b1[64] b3f[64] whf[8][64] bhf[8] swh[8]; flush scratch: Q[8][64] su smu sdl[3][8], loss
// partials [3][8 warps]; staging mbarrier
constexpr uint32_t SMALL_FLOATS = 8 * H + H + H + MAX_OUT * H + 2 * MAX_OUT;
constexpr uint32_t XCH_FLOATS = MAX_OUT * H + 3 * MAX_OUT + 3 * 8;
__host__ __device__ inline uint32_t tc_smem_bytes(int d) { return tc_small_off(d) + 4 * (SMALL_FLOATS + XCH_FLOATS) + 8; }

// Phase stamps for tools/update_epoch_profile.py, compiled in only with -DORL_PROFILE_PHASES (never in the normal
// build): thread 0 of every CTA records %globaltimer and %clock64 at kernel entry, first tile staged, tile loop end and
// kernel exit, and the SM it ran on.  orl_profile_phases_read copies the last launch's stamps to the host.
constexpr int PH_MAX_CTAS = 1024, PH_WORDS = 9;
#ifdef ORL_PROFILE_PHASES
__device__ unsigned long long g_phases[PH_MAX_CTAS][PH_WORDS];
__device__ __forceinline__ void phase_stamp(int k) {
    if (threadIdx.x != 0 || blockIdx.x >= PH_MAX_CTAS) return;
    unsigned long long t, c;
    unsigned sm;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    asm volatile("mov.u64 %0, %%clock64;" : "=l"(c));
    asm volatile("mov.u32 %0, %%smid;" : "=r"(sm));
    g_phases[blockIdx.x][k] = t;
    g_phases[blockIdx.x][4 + k] = c;
    g_phases[blockIdx.x][8] = sm;
}
#else
__device__ __forceinline__ void phase_stamp(int) {}
#endif

// the activation's derivative; ACT as for act_tc (orl_tc16.cuh)
template <int ACT>
__device__ __forceinline__ float act_bwd_t(float a, bool pos, int activation_id) { return ACT == 1 ? (pos ? 1.f : 0.f) : act_bwd(a, pos, activation_id); }

template <bool POLICY, int NOUT, int ACT, bool TMA>
__device__ __forceinline__ void tc_net_pass(const OrlPpoArgs& a, const TcMaps& maps, uint8_t* smem, int cta, int G, int stride) {
    const int d = POLICY ? a.obs_dim : a.critic_obs_dim;
    const int n = POLICY ? (NOUT == 8 ? a.n_actions : NOUT) : 1;
    const float* params = POLICY ? a.policy_params : a.critic_params;
    const float* obs = POLICY ? a.policy_obs : a.critic_obs;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // warp w owns tile rows [16w, +16): the rows of its wgmma accumulator fragment, so the per-tile GEMM results
    // reach the row owners within the warp.  Warpgroup g (= w / 4) owns rows [64g, +64).
    const int row = 16 * warp + (lane & 15), half = lane >> 4, wg = warp >> 2;   // this thread: tile row, column half, warpgroup
    const int cb = CW * half;                                                    // first column of the half
    const NetOffsets po = net_offsets(d, n);

    uint8_t* R1h = smem + OFF_R1H; uint8_t* R1l = smem + OFF_R1L;
    uint8_t* R2h = smem + OFF_R2H; uint8_t* R2l = smem + OFF_R2L;
    uint8_t* Wh = smem + OFF_WH;   uint8_t* Wl = smem + OFF_WL;
    uint8_t* R3h = smem + OFF_R3H; uint8_t* R3l = smem + OFF_R3L;
    float* S = reinterpret_cast<float*>(smem + OFF_S);                                  // [128][S_LD]
    float* st_obs = reinterpret_cast<float*>(smem + OFF_STAGE);                        // [128][d]
    float* st_sc = reinterpret_cast<float*>(smem + OFF_STAGE + ((T_M * d * 4 + 127) & ~127));   // [4][128]
    float* w1t = reinterpret_cast<float*>(smem + tc_small_off(d));   // [8][64] k-major, zero padded
    float* b1s = w1t + 8 * H;
    float* b3f = b1s + H;
    float* whf = b3f + H;                        // [8][64] folded head
    float* bhf = whf + MAX_OUT * H;
    float* swh = bhf + MAX_OUT;                  // [8] row sums of whf
    float* qs = swh + MAX_OUT;                   // flush: [8][64] Q rows, then su[8], smu[8], sdl[8]
    float* red = qs + MAX_OUT * H + 3 * MAX_OUT; // flush: [3][8] per-warp loss sums
    uint64_t* bar_st = reinterpret_cast<uint64_t*>(red + 3 * 8);  // TMA staging

    // ---- staging of the minibatch rows, one tile ahead ----
    const long long n_tiles = (a.batch_rows + T_M - 1) / T_M;
    const float* sc0 = POLICY ? a.actions : a.value_preds;
    const float* sc1 = POLICY ? a.old_log_probs : a.returns;
    const float* sc2 = POLICY ? a.advantages : nullptr;
    const uint32_t stage_tx = (uint32_t)(T_M * d * 4) + (POLICY ? 4u : 3u) * T_M * 4;
    auto issue_tma = [&](long long tile) {   // one thread
        const int r0 = (int)(a.row_begin + tile * T_M);
        mbar_expect_tx(bar_st, stage_tx);
        tma_load_2d(st_obs, POLICY ? &maps.obs_p : &maps.obs_c, 0, r0, bar_st);
        tma_load_1d(st_sc + 0 * T_M, POLICY ? &maps.actions : &maps.value_preds, r0, bar_st);
        tma_load_1d(st_sc + 1 * T_M, POLICY ? &maps.old_logp : &maps.returns, r0, bar_st);
        if (POLICY) tma_load_1d(st_sc + 2 * T_M, &maps.adv, r0, bar_st);
        tma_load_1d(st_sc + 3 * T_M, &maps.active, r0, bar_st);
    };
    auto issue_gather = [&](long long gi) {   // every thread: half 0 the observation row, half 1 the scalars
        const bool v = gi >= 0;
        const long long g = v ? gi : 0;
        if (half == 0) {
            if ((d & 3) == 0) {
                for (int k = 0; k < d; k += 4) cp_async16(st_obs + row * d + k, obs + g * d + k, v);
            } else {
                for (int k = 0; k < d; ++k) cp_async4(st_obs + row * d + k, obs + g * d + k, v);
            }
        } else {
            cp_async4(st_sc + 0 * T_M + row, sc0 + g, v);
            cp_async4(st_sc + 1 * T_M + row, sc1 + g, v);
            if (POLICY) cp_async4(st_sc + 2 * T_M + row, sc2 + g, v);
            cp_async4(st_sc + 3 * T_M + row, a.active_masks + g, v);
        }
        cp_async_commit();
    };
    auto row_index = [&](long long tile) -> long long {   // global row of this thread's tile row, -1 past the end
        if (tile >= n_tiles) return -1;
        const long long r = tile * T_M + row;
        if (r >= a.batch_rows) return -1;
        return a.indices ? a.indices[r] : a.row_begin + r;
    };
    // the first tile's rows are requested before the weights are staged, so that their load runs under the fold below
    long long gi_next = -1;
    if (TMA) {
        if (tid == 0) {
            mbar_init(bar_st, 1);
            fence_proxy_async();   // the initialised barrier, before the TMA unit signals it
            if (cta < n_tiles) { tma_prefetch_desc(POLICY ? &maps.obs_p : &maps.obs_c); issue_tma(cta); }
        }
    } else {
        issue_gather(row_index(cta));
        gi_next = row_index(cta + G);
    }
    long long gi = row_index(cta);

    // ---- stage weights (folded); the fc3 matrix as split fp16 ----
    // The fold runs on a copy of the net's parameters in R3 (free until the first tile): one round of independent
    // global loads, and the 64-deep chains of b3f, bhf and swh then read shared memory.  The same values through the
    // same expressions: every staged weight keeps its bits.
    float* pcopy = reinterpret_cast<float*>(R3h);
    for (int i = tid; i < po.total; i += T_NT) pcopy[i] = params[i];
    // the minibatch constants' global loads go out with the copy's
    const bool pol_masks = a.flags & ORL_PPO_POLICY_ACTIVE_MASKS, val_masks = a.flags & ORL_PPO_VALUE_ACTIVE_MASKS;
    const MbConsts mb = mb_consts(a);
    const double rows_d = loss_rows(a);
    __syncthreads();
    stage_weights_tc(w1t, Wh, Wl, pcopy, d, n, T_NT);
    // swh on warp 4, while warp 0 runs the b3f and bhf chains of stage_weights_tc
    if (tid >= 4 * 32 && tid < 4 * 32 + MAX_OUT) {   // from the parameters, not from the rounded whf
        const int j = tid - 4 * 32;
        float rs = 0.f;
        if (j < n) for (int k = 0; k < H; ++k) rs += folded_wh(pcopy, po, j, k);
        swh[j] = rs;
    }
    // panels that are read before their first per-tile write: zero them (U of lanes beyond n, X beyond d are rewritten per tile)
    if (half == 0) {
        const uint4 z = make_uint4(0u, 0u, 0u, 0u);
        *reinterpret_cast<uint4*>(R1h + P_CST * PANEL + row * 16) = z; *reinterpret_cast<uint4*>(R1l + P_CST * PANEL + row * 16) = z;
        *reinterpret_cast<uint4*>(R1h + P_X * PANEL + row * 16) = z;   *reinterpret_cast<uint4*>(R1l + P_X * PANEL + row * 16) = z;
        *reinterpret_cast<uint4*>(R2h + P_U * PANEL + row * 16) = z;   *reinterpret_cast<uint4*>(R2l + P_U * PANEL + row * 16) = z;
    }
    fence_proxy_async();
    __syncthreads();
    // weight-gradient accumulators for the whole kernel: Ga rows [64 half, +64), Gb (warpgroup 1)
    float ga[40], gb[8];
#pragma unroll
    for (int i = 0; i < 40; ++i) ga[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) gb[i] = 0.f;

    // operand scales of the backward GEMMs (powers of two; see the header comment)
    // wmax = max |whf| over the CTA (a maximum: the same value in any order)
    float wmax = 0.f;
    for (int i = tid; i < MAX_OUT * H; i += T_NT) wmax = fmaxf(wmax, fabsf(whf[i]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wmax = fmaxf(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
    if (lane == 0) red[warp] = wmax;
    __syncthreads();
#pragma unroll
    for (int w = 0; w < T_NT / 32; ++w) wmax = fmaxf(wmax, red[w]);
    // with active masks a live row weighs active / sum(active), not 1 / rows: scale by the rows that carry the weight
    const double live_d = (POLICY ? pol_masks : val_masks) ? fmin(rows_d, a.mb_stats[2]) : rows_d;
    const int e_rows = (int)ceil(log2(fmax(live_d, 1.0)));
    const int e_u = min(e_rows + 3, 60);
    const int e_z = min(max(e_rows + 3 - (int)floorf(log2f(fmaxf(wmax, 1e-12f))), 0), 60);
    const float Sz = exp2f((float)e_z), Su = exp2f((float)e_u);
    constexpr float SX = 16.f, K1 = 0.25f;          // observations x 16; dZ1 is stored as S_z / 4
    const float invSz = exp2f(-(float)e_z), invSu = exp2f(-(float)e_u), invS1 = invSz * (1.f / K1);

    // ---- MMA descriptors (constant parts) ----
    const uint64_t dK_A = desc_const(PANEL, 128), dK_W = desc_const(W_PANEL, 128);      // K-major
    const uint64_t dMN_A = desc_const(128, PANEL), dMN_W = desc_const(128, W_PANEL);    // MN-major
    const uint32_t aR1h = smem_u32(R1h), aR1l = smem_u32(R1l), aR2h = smem_u32(R2h), aR2l = smem_u32(R2l), aWh = smem_u32(Wh), aWl = smem_u32(Wl);
    const uint32_t aR3h = smem_u32(R3h), aR3l = smem_u32(R3l);

    float loss0 = 0.f, loss1 = 0.f, loss2 = 0.f;
    uint32_t it = 0;
    for (long long tile = cta; tile < n_tiles; tile += G, ++it) {
        const uint32_t par = it & 1u;
        // ---- this tile's rows from the staging buffer ----
        if (TMA) mbar_wait(bar_st, par);
        else { cp_async_wait_all(); __syncwarp(); }   // a row's gathers are issued by its two lanes
        if (it == 0) phase_stamp(1);
        const bool valid = gi >= 0;
        float x[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) x[k] = 0.f;
        if (d == 4) {   // one 16-byte load per row (conflict-free); other widths: scalar loads
            const float4 v = *reinterpret_cast<const float4*>(st_obs + row * 4);
            x[0] = v.x; x[1] = v.y; x[2] = v.z; x[3] = v.w;
        } else {
#pragma unroll
            for (int k = 0; k < 8; ++k) if (k < d) x[k] = st_obs[row * d + k];
        }
        // rows past the minibatch's end: the gather zero-fills them, TMA loads whatever the buffer holds there (the
        // partial last tile of a range that ends inside the buffer).  Their dL is 0, but a NaN or inf in x would still
        // reach GEMM3a / GEMM3b through n1 and the X panel (0 x NaN), so they run on x = 0 on both paths.
        if (!valid) {
#pragma unroll
            for (int k = 0; k < 8; ++k) x[k] = 0.f;
        }
        const float row_a = st_sc[0 * T_M + row], row_b = st_sc[1 * T_M + row];
        const float row_c = POLICY ? st_sc[2 * T_M + row] : 0.f, active = st_sc[3 * T_M + row];

        // ---- fc1 + activation + LayerNorm-1 (this thread: columns [cb, cb+32) of its row) ----
        float n1[CW], s, sq;
        const unsigned posmask = row_fc1<CW, ACT>(x, d, w1t, b1s, cb, a.activation_id, n1, s, sq);
        // the previous tile's GEMM3a / GEMM3b have been in flight up to here.  They must complete before R1 is
        // overwritten below; waiting here rather than there keeps ptxas from placing its own wait inside the divergent
        // slow path of the square root, which would serialise every wgmma of the kernel.
        wgmma_wait<0>();
        row_sum_stats<CW>(s, sq);
        const LnStats l1 = ln_stats(s, sq);

        // GEMM3a / GEMM3b of both warpgroups read every row of R1, R2 and R3: all have completed past this barrier.
        // It also means every thread has read its staged row, which the TMA issued after GEMM1 overwrites.
        __syncthreads();
        row_ln1_store<CW>(n1, l1, R1h, R1l, PANEL, row, cb);
        if (half == 0) split_store8(R1h + P_X * PANEL + row * 16, R1l + P_X * PANEL + row * 16, x, SX);
        fence_proxy_async();
        warpgroup_sync(wg);   // GEMM1 reads only this warpgroup's rows of R1
        float z[32];   // GEMM1: Z3 = n1 . W3f^T, rows [64g, +64)
#pragma unroll
        for (int i = 0; i < 32; ++i) z[i] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int pass = 0; pass < 3; ++pass) {
            const uint32_t aa = (pass == 0 ? aR1l : aR1h) + wg * 64 * 16, bb = pass == 1 ? aWl : aWh;
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
                wgmma_f16_n64<0, 0>(z, desc_at(dK_A, aa + 2 * kk * PANEL), desc_at(dK_W, bb + 2 * kk * W_PANEL), (pass | kk) > 0);
        }
        wgmma_commit();   // the only group in flight
        if (TMA && tid == 0 && tile + G < n_tiles) issue_tma(tile + G);   // the staging buffer was consumed before the CTA barrier above
        long long gi_cur = gi;
        if (!TMA) {
            issue_gather(gi_next);
            gi = gi_next;
            gi_next = row_index(tile + 2 * G);
        } else {
            gi = row_index(tile + G);
        }

        wgmma_wait<0>();
        frag_store<64>(z, S + wg * 64 * S_LD, S_LD);
        __syncwarp();   // rows [16 warp, +16) of S: written and read by this warp

        // ---- Z3 (staging tile) + b3f -> LayerNorm-3 -> n3 (registers only) -> head ----
        float n3[CW], s3, q3;
        row_z3<CW>(S, row, cb, b3f, n3, s3, q3);
        row_sum_stats<CW>(s3, q3);
        const LnStats l3 = ln_stats(s3, q3);
        float out[MAX_OUT];
        row_head<CW, NOUT>(n3, l3, whf, cb, n, out);
        row_sum_head<CW, NOUT>(out, n);
        // dot[j] = sum_k Whf[j][k] n3[k] (needed by the LayerNorm-3 backward); logits add the folded bias
        float dot[MAX_OUT];
#pragma unroll
        for (int j = 0; j < MAX_OUT; ++j) { dot[j] = out[j]; out[j] += (j < NOUT && j < n) ? bhf[j] : 0.f; }

        // ---- head loss + dL/dhead (both halves compute it; half 0 accumulates the sums) ----
        float dl[MAX_OUT];
#pragma unroll
        for (int j = 0; j < MAX_OUT; ++j) dl[j] = 0.f;
        if (valid) {
            if (POLICY) {
                const float wrow = mb.weight(pol_masks, active);
                const CatRow c = categorical_row<NOUT>(a, out, n, a.action_masks ? a.action_masks + gi_cur * n : nullptr, (int)row_a, row_b,
                                                       apply_adv_norm(mb.adv, row_c), wrow, dl);
                if (half == 0) { loss0 += c.loss * wrow; loss1 += c.ent * wrow; loss2 += c.ratio; }
            } else {
                const float target = (a.flags & ORL_PPO_VALUENORM) ? (row_b - mb.vn_mean) / mb.vn_std : row_b;
                const ValueTerm vt = value_term(out[0], row_a, target, a.clip_param, a.huber_delta, a.flags);
                const float wrow = mb.weight(val_masks, active);
                if (half == 0) loss0 += vt.loss * wrow;
                dl[0] = a.value_loss_coef * wrow * vt.dv;
            }
        }
        // ---- dn3 = dL . Whf ; LayerNorm-3 backward -> dZ3 (single pass: the two row means are
        //      mean(dn3) = sum_j dL[j] rowsum(Whf[j]) / 64 and mean(dn3 n3) = sum_j dL[j] dot[j] / 64), scaled by S ----
        float m1 = 0.f, m2 = 0.f;
#pragma unroll
        for (int j = 0; j < MAX_OUT; ++j) dl[j] *= Sz;
        FOR_OUT(j) { m1 = fmaf(dl[j], swh[j], m1); m2 = fmaf(dl[j], dot[j], m2); }
        m1 *= (1.f / H); m2 *= (1.f / H);
#pragma unroll
        for (int q8 = 0; q8 < CW; q8 += 8) {
            float g8[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) g8[i] = 0.f;
#pragma unroll
            for (int q4 = 0; q4 < 8; q4 += 4) {
                FOR_OUT(j) {
                    const float4 wv = *reinterpret_cast<const float4*>(whf + j * H + cb + q8 + q4);
                    g8[q4] = fmaf(dl[j], wv.x, g8[q4]); g8[q4 + 1] = fmaf(dl[j], wv.y, g8[q4 + 1]);
                    g8[q4 + 2] = fmaf(dl[j], wv.z, g8[q4 + 2]); g8[q4 + 3] = fmaf(dl[j], wv.w, g8[q4 + 3]);
                }
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) g8[i] = l3.rstd * (g8[i] - m1 - n3[q8 + i] * m2);
            const uint32_t off = (uint32_t)((cb + q8) >> 3) * PANEL + row * 16;
            split_store8(R2h + off, R2l + off, g8, 1.0f);   // dZ3 row slice
        }
        if (half == 0) {
            float u8[8], c8[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) { u8[j] = dl[j] * (l3.rstd * (Su * invSz)); c8[j] = 0.f; }
            c8[0] = 1.0f; c8[1] = l3.mu; c8[2] = l3.var * l3.rstd;   // std3 = var3 / sqrt(var3)
            split_store8(R2h + P_U * PANEL + row * 16, R2l + P_U * PANEL + row * 16, u8, 1.0f);
            split_store8(R1h + P_CST * PANEL + row * 16, R1l + P_CST * PANEL + row * 16, c8, 1.0f);
        }
        fence_proxy_async();
        warpgroup_sync(wg);   // GEMM2 reads only this warpgroup's rows of R2
        // GEMM2: dN1 = dZ3 . W3f (rows [64g, +64)) ; GEMM3a: Ga += R2^T . R1 (rows [64g, +64))
#pragma unroll
        for (int i = 0; i < 32; ++i) z[i] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int pass = 0; pass < 3; ++pass) {
            const uint32_t aa = (pass == 0 ? aR2l : aR2h) + wg * 64 * 16, bb = pass == 1 ? aWl : aWh;
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
                wgmma_f16_n64<0, 1>(z, desc_at(dK_A, aa + 2 * kk * PANEL), desc_at(dMN_W, bb + kk * 256), (pass | kk) > 0);
        }
        wgmma_commit();
        __syncthreads();   // GEMM3a reduces over all 128 rows of R1 and R2
#pragma unroll
        for (int pass = 0; pass < 3; ++pass) {
            const uint32_t aa = (pass == 0 ? aR2l : aR2h) + wg * 8 * PANEL, bb = pass == 1 ? aR1l : aR1h;
#pragma unroll
            for (int kk = 0; kk < 8; ++kk)
                wgmma_f16_n80<1, 1>(ga, desc_at(dMN_A, aa + kk * 256), desc_at(dMN_A, bb + kk * 256), 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();   // GEMM2 has completed; GEMM3a runs on under the row work below and the next tile's fc1
        frag_store<64>(z, S + wg * 64 * S_LD, S_LD);
        __syncwarp();
        // ---- dN1 (staging tile) -> LayerNorm-1 backward -> activation backward -> dZ1 (R3) ----
        {
            float g[CW];
#pragma unroll
            for (int q4 = 0; q4 < CW; q4 += 4) {
                const float4 v = *reinterpret_cast<const float4*>(S + row * S_LD + cb + q4);
                g[q4] = v.x; g[q4 + 1] = v.y; g[q4 + 2] = v.z; g[q4 + 3] = v.w;
            }
            float t1 = 0.f, t2 = 0.f;
#pragma unroll
            for (int i = 0; i < CW; ++i) { t1 += g[i]; t2 = fmaf(g[i], n1[i], t2); }
            row_sum_stats<CW>(t1, t2);
            t1 *= (1.f / H); t2 *= (1.f / H);
            const float std1 = 1.0f / l1.rstd;
#pragma unroll
            for (int i = 0; i < CW; ++i) {
                const float da = l1.rstd * (g[i] - t1 - n1[i] * t2);
                const float aval = fmaf(n1[i], std1, l1.mu);                       // activation output
                g[i] = da * (K1 * act_bwd_t<ACT>(aval, (posmask >> i) & 1u, a.activation_id));
            }
#pragma unroll
            for (int q8 = 0; q8 < CW; q8 += 8) {
                const uint32_t off = (uint32_t)((cb + q8) >> 3) * PANEL + row * 16;
                split_store8(R3h + off, R3l + off, g + q8, 1.0f);
            }
        }
        fence_proxy_async();
        // GEMM3b (warpgroup 1) reduces dZ1 over all 128 rows: warpgroup 0 only signals that its rows are stored
        if (wg == 1) {   // GEMM3b: Gb += dZ1^T . [CST | X], waited for before the next tile overwrites R1
            asm volatile("bar.sync 3, 256;" ::: "memory");
            wgmma_fence();
#pragma unroll
            for (int pass = 0; pass < 3; ++pass) {
                const uint32_t aa = pass == 0 ? aR3l : aR3h, bb = (pass == 1 ? aR1l : aR1h) + P_CST * PANEL;
#pragma unroll
                for (int kk = 0; kk < 8; ++kk)
                    wgmma_f16_n16<1, 1>(gb, desc_at(dMN_A, aa + kk * 256), desc_at(dMN_A, bb + kk * 256), 1u);
            }
            wgmma_commit();
        } else {
            asm volatile("bar.arrive 3, 256;" ::: "memory");
        }
    }
    wgmma_wait<0>();   // the last tile's GEMM3a / GEMM3b
    phase_stamp(2);

    // ---- flush: Ga / Gb (accumulator registers -> staging in R1 / R2) -> partial folded gradients ----
    float* part = a.partials + (size_t)((POLICY ? 0 : G) + cta) * stride;
    const FoldOffsets fo = fold_offsets(d, n);
    float* qsu = qs + MAX_OUT * H;
    if (it > 0) {
        float* gas = reinterpret_cast<float*>(smem);   // [128][GA_LD]
        float* gbs = gas + T_M * GA_LD;                // [64][GB_LD]
        float* w3t = reinterpret_cast<float*>(R3h);    // [64][W3T_LD]
        __syncthreads();   // every MMA has completed: R1 / R2 are free
        frag_store<80>(ga, gas + wg * 64 * GA_LD, GA_LD);
        if (wg == 1) frag_store<16>(gb, gbs, GB_LD);
        // W3f as fp32 for GH below, transposed into R3 (free once the last GEMM3b has completed): w3t[i][k] = W3f[k][i]
        for (int e = tid; e < H * H; e += T_NT) w3t[(e & 63) * W3T_LD + (e >> 6)] = folded_w3(params, po, e >> 6, e & 63);
        __syncthreads();
        // Ga rows [0, 64) are G3, rows [64, 64 + n) Q: consecutive threads take consecutive columns (coalesced stores)
        for (int e = tid; e < H * H; e += T_NT) part[fo.g3 + e] = gas[(e >> 6) * GA_LD + (e & 63)] * invSz;
        for (int e = tid; e < n * H; e += T_NT) qs[e] = gas[(H + (e >> 6)) * GA_LD + (e & 63)];
        if (half == 0) {
            const float* c8 = gas + row * GA_LD + 64;
            if (row < H) part[fo.db3 + row] = c8[0] * invSz;
            else if (row < H + n) { qsu[row - H] = c8[0]; qsu[8 + row - H] = c8[1]; qsu[16 + row - H] = c8[2]; }
            if (row < H) {
                const float* g16 = gbs + row * GB_LD;
                part[fo.db1 + row] = g16[0] * invS1;
#pragma unroll
                for (int c = 0; c < 8; ++c) if (c < d) part[fo.g1 + row * d + c] = g16[8 + c] * (invS1 * (1.f / SX));
            }
        }
        __syncthreads();
        // GH[j][k] = sum_i Q[j][i] W3f[k][i] + b3f[k] su[j] - smu[j] ; dbh[j] = sdl[j]
        for (int o = tid; o < n * H; o += T_NT) {
            const int j = o >> 6, k = o & 63;
            float acc = 0.f;
            for (int i = 0; i < H; ++i) acc = fmaf(qs[j * H + i], w3t[i * W3T_LD + k], acc);
            acc = fmaf(b3f[k], qsu[j], acc) - qsu[8 + j];
            part[fo.gh + o] = acc * invSu;
            if (k == 0) { part[fo.dbh + j] = qsu[16 + j] * invSu; part[fo.dls + j] = 0.f; }
        }
    } else {
        for (int i = tid; i < fo.total; i += T_NT) part[i] = 0.f;   // an idle CTA
    }
    {
        float v[3] = {loss0, loss1, loss2};
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 3; ++k) { const float sv = warp_sum(v[k]); if (lane == 0) red[k * 8 + warp] = sv; }
        __syncthreads();
        if (tid < N_LOSS_TC) {
            float sv = 0.f;
            if (tid < 3) for (int wv = 0; wv < T_NT / 32; ++wv) sv += red[tid * 8 + wv];
            part[stride - N_LOSS_TC + tid] = sv;
        }
    }
}

// blockIdx -> (net, cta): CTAs [0, G) are the policy net and [G, 2G) the critic net.  With one CTA per SM and
// G = #SMs they run as two waves, the policy CTAs first.
template <int NOUT, int ACT, bool TMA>
__global__ void __launch_bounds__(T_NT, 1) ppo_fwdbwd_tc_kernel(const OrlPpoArgs a, const __grid_constant__ TcMaps maps, int stride) {
    extern __shared__ __align__(1024) uint8_t smem_tc[];
    const int G = a.grid_per_net;
    const bool policy = (int)blockIdx.x < G;
    const int cta = policy ? (int)blockIdx.x : (int)blockIdx.x - G;
    phase_stamp(0);
    if (policy) tc_net_pass<true, NOUT, ACT, TMA>(a, maps, smem_tc, cta, G, stride);
    else tc_net_pass<false, 1, ACT, TMA>(a, maps, smem_tc, cta, G, stride);
    phase_stamp(3);
}

using TcKernel = void (*)(const OrlPpoArgs, const TcMaps, int);
template <int NOUT, int ACT>
TcKernel pick_staging(bool tma) { return tma ? ppo_fwdbwd_tc_kernel<NOUT, ACT, true> : ppo_fwdbwd_tc_kernel<NOUT, ACT, false>; }
template <int NOUT>
TcKernel pick_act(int activation_id, bool tma) { return activation_id == 1 ? pick_staging<NOUT, 1>(tma) : pick_staging<NOUT, -1>(tma); }
TcKernel pick_kernel(int n_actions, int activation_id, bool tma) {
    if (n_actions == 2) return pick_act<2>(activation_id, tma);
    if (n_actions == 5) return pick_act<5>(activation_id, tma);
    return pick_act<8>(activation_id, tma);
}

// ---- host: TMA descriptors of the flattened rollout buffers ----
using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}
bool make_map_rows(CUtensorMap* m, const float* base, long long rows, int width) {   // (rows, width) fp32, box = 128 rows x width
    EncodeTiledFn fn = encode_tiled_fn();
    if (!fn || !base) return false;
    if (width == 1) {
        cuuint64_t dims[1] = {(cuuint64_t)rows};
        cuuint64_t strides[1] = {0};
        cuuint32_t box[1] = {T_M}, es[1] = {1};
        return fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 1, const_cast<float*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
    }
    cuuint64_t dims[2] = {(cuuint64_t)width, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)width * 4};
    cuuint32_t box[2] = {(cuuint32_t)width, T_M}, es[2] = {1, 1};
    return fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
struct MapKey {
    const void* p[8]; long long rows; int d, dc;
    bool operator<(const MapKey& o) const {
        for (int i = 0; i < 8; ++i) if (p[i] != o.p[i]) return p[i] < o.p[i];
        if (rows != o.rows) return rows < o.rows;
        if (d != o.d) return d < o.d;
        return dc < o.dc;
    }
};
// descriptors are pure functions of (pointers, shapes): cache them so the steady state does no driver calls
const TcMaps* maps_for(const OrlPpoArgs& a) {
    static std::map<MapKey, TcMaps> cache;
    static std::mutex mu;
    MapKey k{{a.policy_obs, a.critic_obs, a.actions, a.old_log_probs, a.advantages, a.value_preds, a.returns, a.active_masks},
             a.total_rows, a.obs_dim, a.critic_obs_dim};
    std::lock_guard<std::mutex> lock(mu);
    auto it = cache.find(k);
    if (it != cache.end()) return &it->second;
    TcMaps m;
    const bool ok = make_map_rows(&m.obs_p, a.policy_obs, a.total_rows, a.obs_dim) && make_map_rows(&m.obs_c, a.critic_obs, a.total_rows, a.critic_obs_dim) &&
                    make_map_rows(&m.actions, a.actions, a.total_rows, 1) && make_map_rows(&m.old_logp, a.old_log_probs, a.total_rows, 1) &&
                    make_map_rows(&m.adv, a.advantages, a.total_rows, 1) && make_map_rows(&m.value_preds, a.value_preds, a.total_rows, 1) &&
                    make_map_rows(&m.returns, a.returns, a.total_rows, 1) && make_map_rows(&m.active, a.active_masks, a.total_rows, 1);
    if (!ok) return nullptr;
    if (cache.size() > 64) cache.clear();
    return &cache.emplace(k, m).first->second;
}

}  // namespace

namespace orl {
int launch_ppo_fwdbwd_tc(const OrlPpoArgs& a, cudaStream_t st) {
    if (a.obs_dim > 8 || a.critic_obs_dim > 8) {
        set_last_error("orl_ppo_fwdbwd: ORL_PPO_TENSORCORE supports observation widths <= 8 (got %d / %d)", a.obs_dim, a.critic_obs_dim);
        return ORL_ERR_UNSUPPORTED;
    }
    const int dmax = std::max(a.obs_dim, a.critic_obs_dim);
    const size_t smem = tc_smem_bytes(dmax);
    const int stride = ppo_stride_host(a.obs_dim, a.critic_obs_dim, a.n_actions);
    // TMA staging: contiguous row range, rows of 16-byte multiples (d % 4 == 0), 16-byte aligned bases
    const bool tma_ok = a.indices == nullptr && (a.obs_dim % 4 == 0) && (a.critic_obs_dim % 4 == 0) &&
                        ((reinterpret_cast<uintptr_t>(a.policy_obs) | reinterpret_cast<uintptr_t>(a.critic_obs) | reinterpret_cast<uintptr_t>(a.actions) |
                          reinterpret_cast<uintptr_t>(a.old_log_probs) | reinterpret_cast<uintptr_t>(a.advantages) | reinterpret_cast<uintptr_t>(a.value_preds) |
                          reinterpret_cast<uintptr_t>(a.returns) | reinterpret_cast<uintptr_t>(a.active_masks)) & 15) == 0 &&
                        a.row_begin + (((a.batch_rows + T_M - 1) / T_M) * T_M) < (1ll << 31);
    const TcMaps* maps = tma_ok ? maps_for(a) : nullptr;
    TcKernel kern = pick_kernel(a.n_actions, a.activation_id, maps != nullptr);
    if (int e = allow_dynamic_smem(kern, tc_smem_bytes(8), true)) return e;
    TcMaps none;
    if (!maps) memset(&none, 0, sizeof(none));
    kern<<<2 * a.grid_per_net, T_NT, smem, st>>>(a, maps ? *maps : none, stride);
    return check_cuda(cudaGetLastError(), "ppo_fwdbwd_tc_kernel");
}
}  // namespace orl

#ifdef ORL_PROFILE_PHASES
// the stamps of the last ppo_fwdbwd_tc_kernel launch: [PH_MAX_CTAS][PH_WORDS] u64 (not part of the declared C-ABI)
extern "C" int orl_profile_phases_read(unsigned long long* host) {
    return orl::check_cuda(cudaMemcpyFromSymbol(host, g_phases, sizeof(g_phases)), "orl_profile_phases_read");
}
#endif
