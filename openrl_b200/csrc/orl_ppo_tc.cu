// PPO minibatch forward+backward on the Hopper tensor cores (wgmma, split-fp16 operands, FP32
// accumulate) — produces the same folded partial gradients and loss sums as ppo_fwdbwd_kernel
// (orl_ppo.cu) at fp32-class accuracy (orl_tc16.cuh).  Selected with ORL_PPO_TENSORCORE; categorical
// heads, obs widths <= 8 (CartPole, GridWorld).  Reference: openrl/algorithms/ppo.py:46-361.
//
// CTA = 256 threads = 128 tile rows x 2 column halves = 2 warpgroups, one CTA per SM (~147 KB shared
// memory): warps w and w+4 own the same 32 rows and 32 columns each, so every row-wise operation (fc1
// with K = d <= 8, LayerNorm forward/backward, head, loss) is thread-local apart from three two-float
// exchanges and one head exchange through shared memory (named barriers per row group).  The per-tile
// GEMM results (Z3, dN1) arrive in the warpgroups' accumulator registers in the wgmma fragment layout
// and reach the row-owning threads through an fp32 staging tile in shared memory.
//
// All matrix operands live in row-major panel buffers (orl_tc16.cuh) as fp16 hi/lo pairs, written by
// the row-owning threads with 16-byte stores and read K-major or MN-major by descriptor only:
//   R1 = [ n1 (8 panels) | CST = (1, mu3, std3, 0..) | X ]   rows = tile rows       (dZ1 reuses the n1 panels)
//   R2 = [ dZ3 (8 panels) | U = dL * rstd3 ]                  rows = tile rows
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
// are multiplied by the exact inverse when flushed, conversions saturate instead of overflowing.
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

#include "orl_mlp.cuh"
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
constexpr uint32_t PANEL_W = H * 16;
constexpr int R1_PANELS = 10, R2_PANELS = 9;
constexpr int P_CST = 8, P_X = 9, P_U = 8;
constexpr int N_LOSS_TC = 8;
// staging tile of the per-tile GEMM results: 128 rows x 64 fp32, row pitch 68 floats (conflict-free row reads);
// the final Ga [128][GA_LD] / Gb [64][GB_LD] staging reuses R1 / R2
constexpr int S_LD = 68, GA_LD = 84, GB_LD = 20;
// shared-memory carve-up (bytes)
constexpr uint32_t OFF_R1H = 0, OFF_R1L = OFF_R1H + R1_PANELS * PANEL, OFF_R2H = OFF_R1L + R1_PANELS * PANEL,
                   OFF_R2L = OFF_R2H + R2_PANELS * PANEL, OFF_WH = OFF_R2L + R2_PANELS * PANEL, OFF_WL = OFF_WH + 8 * PANEL_W,
                   OFF_S = OFF_WL + 8 * PANEL_W, OFF_STAGE = OFF_S + T_M * S_LD * 4;
static_assert((T_M * GA_LD + 64 * GB_LD) * 4 <= OFF_WH, "the Ga / Gb staging fits in R1 + R2");
static_assert(OFF_STAGE % 128 == 0, "TMA destination alignment");
static_assert(OFF_R2L + 16 * PANEL <= OFF_STAGE + 4096, "the 16-panel A descriptors stay inside the allocation");
constexpr int N_SCAL = 4;                      // scalar columns staged per row

struct TcMaps {   // TMA descriptors of the flattened rollout buffers (built by the launcher)
    CUtensorMap obs_p, obs_c, actions, old_logp, adv, value_preds, returns, active;
};

struct AdvNormTc { float m0, s0, m1, s1; bool two; };

#define FOR_OUT(j) _Pragma("unroll") for (int j = 0; j < NOUT; ++j) if (NOUT != 8 || j < n)
// row-group barrier: the two warps that share rows [32g, 32g+32) (g = warp % 4)
#define ROWGROUP_SYNC()                                                        \
    do {                                                                       \
        switch (warp & 3) {                                                    \
            case 0: asm volatile("bar.sync 1, 64;" ::: "memory"); break;       \
            case 1: asm volatile("bar.sync 2, 64;" ::: "memory"); break;       \
            case 2: asm volatile("bar.sync 3, 64;" ::: "memory"); break;       \
            default: asm volatile("bar.sync 4, 64;" ::: "memory"); break;      \
        }                                                                      \
    } while (0)

__host__ __device__ inline uint32_t tc_stage_bytes(int d) { return (uint32_t)((T_M * d * 4 + 127) & ~127) + N_SCAL * T_M * 4; }
__host__ __device__ inline uint32_t tc_small_off(int d) { return OFF_STAGE + tc_stage_bytes(d); }
// fp32 weights: w1t[8][64] b1[64] b3f[64] whf[8][64] bhf[8] swh[8]; exchange: xs[2][128][2] xh[8][2][128]; staging mbarrier
constexpr uint32_t SMALL_FLOATS = 8 * H + H + H + MAX_OUT * H + 2 * MAX_OUT;
constexpr uint32_t XCH_FLOATS = 2 * T_M * 2 + 2 * T_M * 8;
__host__ __device__ inline uint32_t tc_smem_bytes(int d) { return tc_small_off(d) + 4 * (SMALL_FLOATS + XCH_FLOATS) + 8; }

// ACT == 1: ReLU (the reference's default activation_id) compiled in; ACT == -1: runtime activation_id (tanh / leaky / elu
// expand to ~60 instructions per element, which the fully unrolled row code cannot afford in the instruction cache)
template <int ACT>
__device__ __forceinline__ float act_fwd_t(float z, int activation_id) { return ACT == 1 ? fmaxf(z, 0.f) : act_fwd(z, activation_id); }
template <int ACT>
__device__ __forceinline__ float act_bwd_t(float a, bool pos, int activation_id) { return ACT == 1 ? (pos ? 1.f : 0.f) : act_bwd(a, pos, activation_id); }

template <bool POLICY, int NOUT, int ACT, bool TMA>
__device__ __forceinline__ void tc_net_pass(const OrlPpoArgs& a, const TcMaps& maps, uint8_t* smem, int cta, int G, int stride) {
    const int d = POLICY ? a.obs_dim : a.critic_obs_dim;
    const int n = POLICY ? (NOUT == 8 ? a.n_actions : NOUT) : 1;
    const float* params = POLICY ? a.policy_params : a.critic_params;
    const float* obs = POLICY ? a.policy_obs : a.critic_obs;
    const int tid = threadIdx.x, warp = tid >> 5;
    const int row = tid & 127, half = tid >> 7;   // this thread: tile row, column half (= its warpgroup)
    const int cb = CW * half;                     // first column of the half
    const NetOffsets po = net_offsets(d, n);

    uint8_t* R1h = smem + OFF_R1H; uint8_t* R1l = smem + OFF_R1L;
    uint8_t* R2h = smem + OFF_R2H; uint8_t* R2l = smem + OFF_R2L;
    uint8_t* Wh = smem + OFF_WH;   uint8_t* Wl = smem + OFF_WL;
    float* S = reinterpret_cast<float*>(smem + OFF_S);                                  // [128][S_LD]
    float* st_obs = reinterpret_cast<float*>(smem + OFF_STAGE);                        // [128][d]
    float* st_sc = reinterpret_cast<float*>(smem + OFF_STAGE + ((T_M * d * 4 + 127) & ~127));   // [4][128]
    float* w1t = reinterpret_cast<float*>(smem + tc_small_off(d));   // [8][64] k-major, zero padded
    float* b1s = w1t + 8 * H;
    float* b3f = b1s + H;
    float* whf = b3f + H;                        // [8][64] folded head
    float* bhf = whf + MAX_OUT * H;
    float* swh = bhf + MAX_OUT;                  // [8] row sums of whf
    float* xs = swh + MAX_OUT;                   // [2][128][2] statistics exchange
    float* xh = xs + 2 * T_M * 2;                // [2][128][8] head exchange (flush scratch afterwards)
    uint64_t* bar_st = reinterpret_cast<uint64_t*>(xh + 2 * T_M * 8);  // TMA staging

    // ---- stage weights (folded); the fc3 matrix as split fp16 ----
    for (int i = tid; i < 8 * H; i += T_NT) { const int k = i / H, j = i % H; w1t[i] = (k < d) ? params[po.w1 + j * d + k] : 0.f; }
    for (int i = tid; i < H; i += T_NT) b1s[i] = params[po.b1 + i];
    for (int i = tid; i < H * 8; i += T_NT) {   // item = (panel p, row j): lanes own consecutive rows -> conflict-free 16-byte stores
        const int pnl = i / H, j = i % H;
        float w8[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) w8[c] = params[po.w3 + j * H + 8 * pnl + c] * params[po.g1 + 8 * pnl + c];
        const uint32_t off = (uint32_t)pnl * PANEL_W + j * 16;
        split_store8(Wh + off, Wl + off, w8, 1.0f);
    }
    for (int i = tid; i < MAX_OUT * H; i += T_NT) { const int j = i / H, k = i % H; whf[i] = (j < n) ? params[po.wh + j * H + k] * params[po.g3 + k] : 0.f; }
    for (int j = tid; j < H; j += T_NT) {
        float s = params[po.b3 + j];
        for (int k = 0; k < H; ++k) s = fmaf(params[po.w3 + j * H + k], params[po.be1 + k], s);
        b3f[j] = s;
    }
    for (int j = tid; j < MAX_OUT; j += T_NT) {
        float s = 0.f;
        if (j < n) { s = params[po.bh + j]; for (int k = 0; k < H; ++k) s = fmaf(params[po.wh + j * H + k], params[po.be3 + k], s); }
        bhf[j] = s;
        float rs = 0.f;
        if (j < n) for (int k = 0; k < H; ++k) rs += params[po.wh + j * H + k] * params[po.g3 + k];
        swh[j] = rs;
    }
    // panels that are read before their first per-tile write: zero them (U of lanes beyond n, X beyond d are rewritten per tile)
    if (half == 0) {
        const uint4 z = make_uint4(0u, 0u, 0u, 0u);
        *reinterpret_cast<uint4*>(R1h + P_CST * PANEL + row * 16) = z; *reinterpret_cast<uint4*>(R1l + P_CST * PANEL + row * 16) = z;
        *reinterpret_cast<uint4*>(R1h + P_X * PANEL + row * 16) = z;   *reinterpret_cast<uint4*>(R1l + P_X * PANEL + row * 16) = z;
        *reinterpret_cast<uint4*>(R2h + P_U * PANEL + row * 16) = z;   *reinterpret_cast<uint4*>(R2l + P_U * PANEL + row * 16) = z;
    }
    if (tid == 0) mbar_init(bar_st, 1);
    fence_proxy_async();
    __syncthreads();
    // weight-gradient accumulators for the whole kernel: Ga rows [64 half, +64), Gb (warpgroup 1)
    float ga[40], gb[8];
#pragma unroll
    for (int i = 0; i < 40; ++i) ga[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) gb[i] = 0.f;

    // ---- minibatch constants ----
    const bool pol_masks = a.flags & ORL_PPO_POLICY_ACTIVE_MASKS, val_masks = a.flags & ORL_PPO_VALUE_ACTIVE_MASKS;
    const double rows_d = (double)(a.norm_rows > 0 ? a.norm_rows : a.batch_rows);
    const float inv_rows = (float)(1.0 / rows_d), inv_act = (float)(1.0 / a.mb_stats[2]);
    // operand scale of the backward GEMMs: 2^e ~ rows / 16 (row weights are ~ 1/rows)
    // operand scales of the backward GEMMs (powers of two; see the header comment)
    float wmax = 0.f;
    for (int i = 0; i < MAX_OUT * H; ++i) wmax = fmaxf(wmax, fabsf(whf[i]));   // smem broadcast reads, once per kernel
    const int e_rows = (int)ceil(log2(fmax(rows_d, 1.0)));
    const int e_u = min(e_rows + 3, 60);
    const int e_z = min(max(e_rows + 3 - (int)floorf(log2f(fmaxf(wmax, 1e-12f))), 0), 60);
    const float Sz = exp2f((float)e_z), Su = exp2f((float)e_u);
    constexpr float SX = 16.f, K1 = 0.25f;          // observations x 16; dZ1 is stored as S_z / 4
    const float invSz = exp2f(-(float)e_z), invSu = exp2f(-(float)e_u), invS1 = invSz * (1.f / K1);
    AdvNormTc an = {0.f, 1.f, 0.f, 1.f, false};
    float vn_mean = 0.f, vn_std = 1.f;
    if (POLICY) {  // ppo.py:402-409
        const double* gs = a.gae_stats;
        const double n_all = gs[ORL_GS_COUNT], n_act = gs[ORL_GS_ACT_COUNT];
        const double mean_all = gs[ORL_GS_ADV_SUM] / n_all;
        const double var_all = fmax(gs[ORL_GS_ADV_SQSUM] / n_all - mean_all * mean_all, 0.0);
        double mean_act = gs[ORL_GS_ADV_ACT_SUM] / n_act;
        double std_act = sqrt(fmax(gs[ORL_GS_ADV_ACT_SQSUM] / n_act - mean_act * mean_act, 0.0));
        if (a.flags & ORL_PPO_ADV_NORMALIZE) {
            const double s0 = (double)((float)sqrt(var_all)) + 1e-5;
            an.two = true; an.m0 = (float)mean_all; an.s0 = (float)s0;
            mean_act = (mean_act - mean_all) / s0; std_act = std_act / s0;
        }
        an.m1 = (float)mean_act; an.s1 = (float)((double)((float)std_act) + 1e-5);
    } else if (a.flags & ORL_PPO_VALUENORM) {
        const float bm = (float)(a.mb_stats[0] / rows_d), bsq = (float)(a.mb_stats[1] / rows_d);
        const float beta = (float)a.vn_beta, omw = (float)(1.0 - a.vn_beta);
        float st[3];
        st[0] = __fadd_rn(__fmul_rn(a.vn_state[0], beta), __fmul_rn(bm, omw));
        st[1] = __fadd_rn(__fmul_rn(a.vn_state[1], beta), __fmul_rn(bsq, omw));
        st[2] = __fadd_rn(__fmul_rn(a.vn_state[2], beta), __fmul_rn(1.0f, omw));
        const VnScalars s = vn_mean_std(st);
        vn_mean = s.mean; vn_std = s.std;
    }

    // ---- MMA descriptors (constant parts) ----
    const uint64_t dK_A = desc_const(PANEL, 128), dK_W = desc_const(PANEL_W, 128);      // K-major
    const uint64_t dMN_A = desc_const(128, PANEL), dMN_W = desc_const(128, PANEL_W);    // MN-major
    const uint32_t aR1h = smem_u32(R1h), aR1l = smem_u32(R1l), aR2h = smem_u32(R2h), aR2l = smem_u32(R2l), aWh = smem_u32(Wh), aWl = smem_u32(Wl);

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
    long long gi_next = -1;
    if (TMA) {
        if (tid == 0 && cta < n_tiles) { tma_prefetch_desc(POLICY ? &maps.obs_p : &maps.obs_c); issue_tma(cta); }
    } else {
        issue_gather(row_index(cta));
        gi_next = row_index(cta + G);
    }
    long long gi = row_index(cta);

    float loss0 = 0.f, loss1 = 0.f, loss2 = 0.f;
    uint32_t it = 0;
    for (long long tile = cta; tile < n_tiles; tile += G, ++it) {
        const uint32_t par = it & 1u;
        // ---- this tile's rows from the staging buffer ----
        if (TMA) mbar_wait(bar_st, par);
        else { cp_async_wait_all(); __syncthreads(); }
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
        const float row_a = st_sc[0 * T_M + row], row_b = st_sc[1 * T_M + row];
        const float row_c = POLICY ? st_sc[2 * T_M + row] : 0.f, active = st_sc[3 * T_M + row];

        // ---- fc1 + activation + LayerNorm-1 (this thread: columns [cb, cb+32) of its row) ----
        float n1[CW];
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
        unsigned posmask = 0u;   // sign bits of this thread's pre-activations
        float s = 0.f, sq = 0.f;
#pragma unroll
        for (int i = 0; i < CW; ++i) {
            if (n1[i] > 0.f) posmask |= 1u << i;
            n1[i] = act_fwd_t<ACT>(n1[i], a.activation_id);
            s += n1[i]; sq = fmaf(n1[i], n1[i], sq);
        }
        {   // exchange 1 (slot xs): LayerNorm-1 statistics
            *reinterpret_cast<float2*>(xs + (half * T_M + row) * 2) = make_float2(s, sq);
            ROWGROUP_SYNC();
            const float2 o = *reinterpret_cast<const float2*>(xs + ((half ^ 1) * T_M + row) * 2);
            s += o.x; sq += o.y;
        }
        const float mu1 = s * (1.f / H);
        const float rstd1 = 1.0f / sqrtf(fmaxf(sq * (1.f / H) - mu1 * mu1, 0.f) + LN_EPS);
#pragma unroll
        for (int i = 0; i < CW; ++i) n1[i] = (n1[i] - mu1) * rstd1;

        // previous tile's GEMM3b (warpgroup 1) must have finished reading R1
        if (it > 0) __syncthreads();
#pragma unroll
        for (int q8 = 0; q8 < CW; q8 += 8) {
            const uint32_t off = (uint32_t)((cb + q8) >> 3) * PANEL + row * 16;
            split_store8(R1h + off, R1l + off, n1 + q8, 1.0f);
        }
        if (half == 0) split_store8(R1h + P_X * PANEL + row * 16, R1l + P_X * PANEL + row * 16, x, SX);
        fence_proxy_async();
        __syncthreads();
        float z[32];   // GEMM1: Z3 = n1 . W3f^T, rows [64 half, +64)
#pragma unroll
        for (int i = 0; i < 32; ++i) z[i] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int pass = 0; pass < 3; ++pass) {
            const uint32_t aa = (pass == 0 ? aR1l : aR1h) + half * 64 * 16, bb = pass == 1 ? aWl : aWh;
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
                wgmma_f16_n64<0, 0>(z, desc_at(dK_A, aa + 2 * kk * PANEL), desc_at(dK_W, bb + 2 * kk * PANEL_W), (pass | kk) > 0);
        }
        wgmma_commit();
        if (TMA && tid == 0 && tile + G < n_tiles) issue_tma(tile + G);   // the staging buffer was consumed before the barrier above
        long long gi_cur = gi;
        if (!TMA) {
            issue_gather(gi_next);
            gi = gi_next;
            gi_next = row_index(tile + 2 * G);
        } else {
            gi = row_index(tile + G);
        }

        wgmma_wait0();
        frag_store<64>(z, S + half * 64 * S_LD, S_LD);
        __syncthreads();

        // ---- Z3 (staging tile) + b3f -> LayerNorm-3 -> n3 (registers only) ----
        float n3[CW];
#pragma unroll
        for (int q4 = 0; q4 < CW; q4 += 4) {
            const float4 v = *reinterpret_cast<const float4*>(S + row * S_LD + cb + q4);
            n3[q4] = v.x; n3[q4 + 1] = v.y; n3[q4 + 2] = v.z; n3[q4 + 3] = v.w;
        }
        float s3 = 0.f, q3 = 0.f;
#pragma unroll
        for (int i = 0; i < CW; ++i) { n3[i] += b3f[cb + i]; s3 += n3[i]; q3 = fmaf(n3[i], n3[i], q3); }
        {   // exchange 2 (slot xs; the barrier before GEMM1 separates it from exchange 1)
            *reinterpret_cast<float2*>(xs + (half * T_M + row) * 2) = make_float2(s3, q3);
            ROWGROUP_SYNC();
            const float2 o = *reinterpret_cast<const float2*>(xs + ((half ^ 1) * T_M + row) * 2);
            s3 += o.x; q3 += o.y;
        }
        const float mu3 = s3 * (1.f / H);
        const float var3 = fmaxf(q3 * (1.f / H) - mu3 * mu3, 0.f) + LN_EPS;
        const float rstd3 = 1.0f / sqrtf(var3);
        float out[MAX_OUT];
#pragma unroll
        for (int j = 0; j < MAX_OUT; ++j) out[j] = 0.f;
#pragma unroll
        for (int q4 = 0; q4 < CW; q4 += 4) {
#pragma unroll
            for (int i = 0; i < 4; ++i) n3[q4 + i] = (n3[q4 + i] - mu3) * rstd3;
            FOR_OUT(j) {
                const float4 wv = *reinterpret_cast<const float4*>(whf + j * H + cb + q4);
                out[j] = fmaf(n3[q4], wv.x, fmaf(n3[q4 + 1], wv.y, fmaf(n3[q4 + 2], wv.z, fmaf(n3[q4 + 3], wv.w, out[j]))));
            }
        }
        {   // exchange 3 (slot xh): partial head dots
            FOR_OUT(j) xh[(j * 2 + half) * T_M + row] = out[j];   // [j][half][row]: lanes are consecutive words (conflict-free)
            ROWGROUP_SYNC();
            FOR_OUT(j) out[j] += xh[(j * 2 + (half ^ 1)) * T_M + row];
        }
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
                unsigned masked = 0;
                if (a.action_masks) {
#pragma unroll
                    for (int j = 0; j < MAX_OUT; ++j)
                        if (j < n && a.action_masks[gi_cur * n + j] == 0.f) { out[j] = -6e4f; masked |= 1u << j; }
                }
                float nl[MAX_OUT], pr[MAX_OUT];
                log_softmax_n(out, n, nl, pr);
                const int act = (int)row_a;
                float lp = nl[0];
#pragma unroll
                for (int j = 1; j < MAX_OUT; ++j) if (j == act) lp = nl[j];
                float adv = row_c;
                if (an.two) adv = (adv - an.m0) / an.s0;
                adv = (adv - an.m1) / an.s1;
                const PgTerm pg = pg_term(lp, row_b, adv, a.clip_param, a.flags, a.dual_clip_coeff);
                const float wrow = pol_masks ? active * inv_act : inv_rows;
                float ent = 0.f;
#pragma unroll
                for (int j = 0; j < MAX_OUT; ++j) if (j < n) ent -= pr[j] * nl[j];
                if (half == 0) { loss0 += pg.loss * wrow; loss1 += ent * wrow; loss2 += pg.ratio; }
                const float dlp = pg.dlogp * wrow, went = a.entropy_coef * wrow;
#pragma unroll
                for (int j = 0; j < MAX_OUT; ++j)
                    if (j < n && !((masked >> j) & 1u)) dl[j] = dlp * ((j == act ? 1.f : 0.f) - pr[j]) + went * pr[j] * (nl[j] + ent);
            } else {
                const float v = out[0], vp = row_a, ret = row_b;
                const float target = (a.flags & ORL_PPO_VALUENORM) ? (ret - vn_mean) / vn_std : ret;
                const float diff = v - vp;
                const float clipped = vp + fminf(fmaxf(diff, -a.clip_param), a.clip_param);
                const float e_c = target - clipped, e_o = target - v, dlt = a.huber_delta;
                const bool hub = a.flags & ORL_PPO_HUBER;
                const float l_c = hub ? (fabsf(e_c) <= dlt ? 0.5f * e_c * e_c : dlt * (fabsf(e_c) - 0.5f * dlt)) : 0.5f * e_c * e_c;
                const float l_o = hub ? (fabsf(e_o) <= dlt ? 0.5f * e_o * e_o : dlt * (fabsf(e_o) - 0.5f * dlt)) : 0.5f * e_o * e_o;
                const float gc = hub ? (fabsf(e_c) <= dlt ? e_c : (e_c > 0.f ? dlt : -dlt)) : e_c;
                const float go = hub ? (fabsf(e_o) <= dlt ? e_o : (e_o > 0.f ? dlt : -dlt)) : e_o;
                float l = l_o, dv = -go;
                if (a.flags & ORL_PPO_CLIP_VALUE) {
                    const bool inrange = diff >= -a.clip_param && diff <= a.clip_param;
                    const float dc = inrange ? -gc : 0.f;
                    if (l_o > l_c) { l = l_o; dv = -go; } else if (l_c > l_o) { l = l_c; dv = dc; } else { l = l_o; dv = 0.5f * (-go) + 0.5f * dc; }
                }
                const float wrow = val_masks ? active * inv_act : inv_rows;
                if (half == 0) loss0 += l * wrow;
                dl[0] = a.value_loss_coef * wrow * dv;
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
            for (int i = 0; i < 8; ++i) g8[i] = rstd3 * (g8[i] - m1 - n3[q8 + i] * m2);
            const uint32_t off = (uint32_t)((cb + q8) >> 3) * PANEL + row * 16;
            split_store8(R2h + off, R2l + off, g8, 1.0f);   // dZ3 row slice
        }
        if (half == 0) {
            float u8[8], c8[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) { u8[j] = dl[j] * (rstd3 * (Su * invSz)); c8[j] = 0.f; }
            c8[0] = 1.0f; c8[1] = mu3; c8[2] = var3 * rstd3;   // std3 = var3 / sqrt(var3)
            split_store8(R2h + P_U * PANEL + row * 16, R2l + P_U * PANEL + row * 16, u8, 1.0f);
            split_store8(R1h + P_CST * PANEL + row * 16, R1l + P_CST * PANEL + row * 16, c8, 1.0f);
        }
        fence_proxy_async();
        __syncthreads();
        // GEMM2: dN1 = dZ3 . W3f (rows [64 half, +64)) ; GEMM3a: Ga += R2^T . R1 (rows [64 half, +64))
#pragma unroll
        for (int i = 0; i < 32; ++i) z[i] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int pass = 0; pass < 3; ++pass) {
            const uint32_t aa = (pass == 0 ? aR2l : aR2h) + half * 64 * 16, bb = pass == 1 ? aWl : aWh;
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
                wgmma_f16_n64<0, 1>(z, desc_at(dK_A, aa + 2 * kk * PANEL), desc_at(dMN_W, bb + kk * 256), (pass | kk) > 0);
        }
#pragma unroll
        for (int pass = 0; pass < 3; ++pass) {
            const uint32_t aa = (pass == 0 ? aR2l : aR2h) + half * 8 * PANEL, bb = pass == 1 ? aR1l : aR1h;
#pragma unroll
            for (int kk = 0; kk < 8; ++kk)
                wgmma_f16_n80<1, 1>(ga, desc_at(dMN_A, aa + kk * 256), desc_at(dMN_A, bb + kk * 256), 1u);
        }
        wgmma_commit();
        wgmma_wait0();
        frag_store<64>(z, S + half * 64 * S_LD, S_LD);
        __syncthreads();   // dN1 is staged, and both warpgroups' GEMM3a have finished reading n1 from R1
        // ---- dN1 (staging tile) -> LayerNorm-1 backward -> activation backward -> dZ1 (into the n1 panels of R1) ----
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
            {   // exchange 4 (slot xs; the barrier before GEMM2 separates it from exchange 2)
                *reinterpret_cast<float2*>(xs + (half * T_M + row) * 2) = make_float2(t1, t2);
                ROWGROUP_SYNC();
                const float2 o = *reinterpret_cast<const float2*>(xs + ((half ^ 1) * T_M + row) * 2);
                t1 += o.x; t2 += o.y;
            }
            t1 *= (1.f / H); t2 *= (1.f / H);
            const float std1 = 1.0f / rstd1;
#pragma unroll
            for (int i = 0; i < CW; ++i) {
                const float da = rstd1 * (g[i] - t1 - n1[i] * t2);
                const float aval = fmaf(n1[i], std1, mu1);                          // activation output
                g[i] = da * (K1 * act_bwd_t<ACT>(aval, (posmask >> i) & 1u, a.activation_id));
            }
#pragma unroll
            for (int q8 = 0; q8 < CW; q8 += 8) {
                const uint32_t off = (uint32_t)((cb + q8) >> 3) * PANEL + row * 16;
                split_store8(R1h + off, R1l + off, g + q8, 1.0f);
            }
        }
        fence_proxy_async();
        __syncthreads();
        if (half == 1) {   // GEMM3b: Gb += dZ1^T . [CST | X]
            wgmma_fence();
#pragma unroll
            for (int pass = 0; pass < 3; ++pass) {
                const uint32_t aa = pass == 0 ? aR1l : aR1h, bb = (pass == 1 ? aR1l : aR1h) + P_CST * PANEL;
#pragma unroll
                for (int kk = 0; kk < 8; ++kk)
                    wgmma_f16_n16<1, 1>(gb, desc_at(dMN_A, aa + kk * 256), desc_at(dMN_A, bb + kk * 256), 1u);
            }
            wgmma_commit();
            wgmma_wait0();
        }
    }

    // ---- flush: Ga / Gb (accumulator registers -> staging in R1 / R2) -> partial folded gradients ----
    float* part = a.partials + (size_t)((POLICY ? 0 : G) + cta) * stride;
    const FoldOffsets fo = fold_offsets(d, n);
    float* qs = xh;              // [8][64] Q rows, then su[8], smu[8], sdl[8]
    float* qsu = qs + MAX_OUT * H;
    if (it > 0) {
        float* gas = reinterpret_cast<float*>(smem);   // [128][GA_LD]
        float* gbs = gas + T_M * GA_LD;                // [64][GB_LD]
        __syncthreads();   // every MMA has completed: R1 / R2 are free
        frag_store<80>(ga, gas + half * 64 * GA_LD, GA_LD);
        if (half == 1) frag_store<16>(gb, gbs, GB_LD);
        __syncthreads();
        {   // Ga columns [32*half, 32*half+32) of this row
            float v[32];
#pragma unroll
            for (int c = 0; c < 32; ++c) v[c] = gas[row * GA_LD + 32 * half + c];
            if (row < H) {
#pragma unroll
                for (int c = 0; c < 32; ++c) part[fo.g3 + row * H + 32 * half + c] = v[c] * invSz;
            } else if (row < H + n) {
#pragma unroll
                for (int c = 0; c < 32; ++c) qs[(row - H) * H + 32 * half + c] = v[c];
            }
        }
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
            for (int i = 0; i < H; ++i) acc = fmaf(qs[j * H + i], params[po.w3 + k * H + i] * params[po.g1 + i], acc);
            acc = fmaf(b3f[k], qsu[j], acc) - qsu[8 + j];
            part[fo.gh + o] = acc * invSu;
            if (k == 0) { part[fo.dbh + j] = qsu[16 + j] * invSu; part[fo.dls + j] = 0.f; }
        }
    } else {
        for (int i = tid; i < fo.total; i += T_NT) part[i] = 0.f;   // an idle CTA
    }
    {
        float v[3] = {loss0, loss1, loss2};
        float* red = xs;
        const int lane = tid & 31;
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
    if (policy) tc_net_pass<true, NOUT, ACT, TMA>(a, maps, smem_tc, cta, G, stride);
    else tc_net_pass<false, 1, ACT, TMA>(a, maps, smem_tc, cta, G, stride);
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
    {
        static std::mutex mu;
        static std::map<TcKernel, bool> prepared;
        std::lock_guard<std::mutex> lock(mu);
        if (!prepared.count(kern)) {
            int e = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc_smem_bytes(8)), "cudaFuncSetAttribute(ppo_fwdbwd_tc)");
            if (e) return e;
            cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
            prepared[kern] = true;
        }
    }
    TcMaps none;
    if (!maps) memset(&none, 0, sizeof(none));
    kern<<<2 * a.grid_per_net, T_NT, smem, st>>>(a, maps ? *maps : none, stride);
    return check_cuda(cudaGetLastError(), "ppo_fwdbwd_tc_kernel");
}
}  // namespace orl
