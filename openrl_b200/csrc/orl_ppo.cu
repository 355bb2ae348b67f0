// PPO minibatch update: fused gather + forward + loss + backward (orl_ppo_fwdbwd), deterministic
// partial reduction (orl_ppo_reduce) and unfold + clip + Adam (orl_ppo_apply).
// Reference semantics: openrl/algorithms/ppo.py:46-361 (see include/openrl_b200.h).
//
// orl_ppo_fwdbwd: persistent CTAs of 256 threads; CTAs [0, G) run the policy net, [G, 2G) the
// critic net (the two losses are independent once the minibatch moments are known).  A CTA walks
// tiles of 128 minibatch rows; per tile it runs, entirely in shared memory / registers,
//   trunk forward (2 tile GEMMs + LayerNorms)  -> head + loss + dLoss/dhead (2 lanes per row)
//   -> dn3 = dL.Whf, LN3 backward -> G3 += dZ3^T n1 ; dn1 = dZ3.W3f, LN1 + activation backward
//   -> G1 += dZ1^T X
// with the weight-gradient blocks (4x4 per thread) accumulated in registers across all tiles of
// the CTA and written once at the end.  fp32 FFMA throughout (1e-4 loss-parity bar; see DESIGN.md).
// Arithmetic per row (d=4, n=2, both nets): ~53 kFLOP; bytes per row: ~60 B  => fp32-pipe bound.
#include <algorithm>

#include "orl_adam.cuh"

namespace {
using namespace orl;

constexpr int P_M = 128;   // rows per tile
constexpr int P_NT = 256;  // threads per CTA
constexpr int P_TY = P_NT / 16, P_RPT = P_M / P_TY;
constexpr int DLW = 8;     // leading dimension of the dL/dhead tile
constexpr int N_LOSS = 8;  // loss-sum slots at the tail of a partial row

__host__ __device__ inline int ppo_stride(int obs_dim, int critic_obs_dim, int n_actions) {
    const int a = orl::fold_offsets(obs_dim, n_actions).total, b = orl::fold_offsets(critic_obs_dim, 1).total;
    return ((a > b ? a : b) + N_LOSS + 3) & ~3;
}

__host__ __device__ inline int ppo_grads_stride(int obs_dim, int critic_obs_dim, int n_actions) {
    const int a = orl::net_offsets(obs_dim, n_actions, 1).total, b = orl::net_offsets(critic_obs_dim, 1).total;
    return ((a > b ? a : b) + 3) & ~3;
}

struct WgMap { int jb, kb, mg, MG; bool active; };
__device__ __forceinline__ WgMap wg_map(int JB, int KB) {
    WgMap m;
    const int nb = JB * KB;
    m.MG = P_NT / nb;
    const int tid = threadIdx.x;
    m.active = tid < nb * m.MG;
    const int b = tid % nb;
    m.mg = tid / nb;
    m.jb = b / KB;
    m.kb = b % KB;
    return m;
}
// g[a][b] += sum_{m = mg, mg+MG, ...} P[m][4jb+a] * Q[m][4kb+b];  db[a] += P[m][4jb+a] when kb == 0
__device__ __forceinline__ void wgrad_acc(const float* __restrict__ P, int ldp, const float* __restrict__ Q, int ldq,
                                          const WgMap& mp, float (&g)[4][4], float (&db)[4]) {
    if (!mp.active) return;
    const float* pp = P + 4 * mp.jb;
    const float* qq = Q + 4 * mp.kb;
    const bool bias = mp.kb == 0;
#pragma unroll 4
    for (int m = mp.mg; m < P_M; m += mp.MG) {
        const float4 p = *reinterpret_cast<const float4*>(pp + m * ldp);
        const float4 q = *reinterpret_cast<const float4*>(qq + m * ldq);
        g[0][0] = fmaf(p.x, q.x, g[0][0]); g[0][1] = fmaf(p.x, q.y, g[0][1]); g[0][2] = fmaf(p.x, q.z, g[0][2]); g[0][3] = fmaf(p.x, q.w, g[0][3]);
        g[1][0] = fmaf(p.y, q.x, g[1][0]); g[1][1] = fmaf(p.y, q.y, g[1][1]); g[1][2] = fmaf(p.y, q.z, g[1][2]); g[1][3] = fmaf(p.y, q.w, g[1][3]);
        g[2][0] = fmaf(p.z, q.x, g[2][0]); g[2][1] = fmaf(p.z, q.y, g[2][1]); g[2][2] = fmaf(p.z, q.z, g[2][2]); g[2][3] = fmaf(p.z, q.w, g[2][3]);
        g[3][0] = fmaf(p.w, q.x, g[3][0]); g[3][1] = fmaf(p.w, q.y, g[3][1]); g[3][2] = fmaf(p.w, q.z, g[3][2]); g[3][3] = fmaf(p.w, q.w, g[3][3]);
        if (bias) { db[0] += p.x; db[1] += p.y; db[2] += p.z; db[3] += p.w; }
    }
}

// Reduce a thread-block-distributed gradient (4x4 blocks, MG row groups) through shared scratch and
// write rows < jdim, cols < kdim to global out[j*kdim + k]; bias sums to out_b[j].
__device__ __forceinline__ void wgrad_flush(float* __restrict__ scratch, const WgMap& mp, int JB, int KB,
                                            const float (&g)[4][4], const float (&db)[4], int jdim, int kdim,
                                            float* __restrict__ out, float* __restrict__ out_b) {
    const int W = 4 * KB, R = 4 * JB;
    __syncthreads();
    if (mp.active) {
        float* s = scratch + (size_t)mp.mg * (R * W + R);
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b) s[(4 * mp.jb + a) * W + 4 * mp.kb + b] = g[a][b];
        if (mp.kb == 0) {
#pragma unroll
            for (int a = 0; a < 4; ++a) s[R * W + 4 * mp.jb + a] = db[a];
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < R * W + R; i += P_NT) {
        float v = 0.f;
        for (int g2 = 0; g2 < mp.MG; ++g2) v += scratch[(size_t)g2 * (R * W + R) + i];
        if (i < R * W) {
            const int j = i / W, k = i % W;
            if (j < jdim && k < kdim) out[j * kdim + k] = v;
        } else {
            const int j = i - R * W;
            if (j < jdim) out_b[j] = v;
        }
    }
}


// NB: head width bound of the policy pass (orl_mlp.cuh).  NB = 64, Categorical heads of 9..64 actions: the logits are a
// 128 x 64 tile (head_tile) in the DZs buffer, which the row loss overwrites with dL/dlogits; dn3 = dL . Whf is a tile
// GEMM with K = pad4(n) and GH += dL^T n3 a wgrad_acc with JB = ceil(n / 4).  dZ3 goes to DZs only after both have read
// dL, so the dL tile needs no buffer of its own (that keeps obs width 64 within the 227 KB of shared memory).
// PANELS: an observation wider than 64 (orl_mlp.cuh, fc1_panels) in the buffers of the d = 64 layout.  The forward runs
// fc1 panel by panel; the backward re-stages each panel (the last one is still in Xs) and forms G1_p = dZ1^T X_p with
// one 4x4 block per thread (MG = 1), which the thread adds into its own elements of this CTA's partial row: one owner
// per element, tiles in the CTA's order, no atomics.
// GAUSS (NB = 64): a DiagGaussian head of 1..64 dimensions (ORL_HEAD_GAUSSIAN_WIDE) on the same tiles.  The means are the
// head tile; the loss is elementwise per (row, dimension), so it runs dimension-parallel: thread t owns dimension
// j = t % 64 of rows t / 64, t / 64 + 4, ..., writes dL/dmean over the mean (the dL tile of the Categorical pass) and
// keeps dL/dlogstd of its rows in one register; the 4 partials of a dimension are added in row-group order at the flush.
template <bool POLICY, int NB = MAX_OUT, bool PANELS = false, bool GAUSS = false>
__device__ __forceinline__ void ppo_net_pass(const OrlPpoArgs& a, float* smem, int cta, int G) {
    constexpr bool WIDE = NB == MAX_OUT_WIDE;
    static_assert(POLICY || !WIDE, "the critic's head is one value");
    static_assert(WIDE || !GAUSS, "GAUSS is the wide DiagGaussian head");
    static_assert(P_NT % MAX_OUT_WIDE == 0, "whole row groups of the dimension-parallel loss");
    const int d = POLICY ? a.obs_dim : a.critic_obs_dim;
    const int n = POLICY ? a.n_actions : 1;
    const float* params = POLICY ? a.policy_params : a.critic_params;
    const float* obs = POLICY ? a.policy_obs : a.critic_obs;
    const int dp = PANELS ? OBS_PANEL : pad4(d), ldx = dp + 4;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;

    float* p = smem;
    SmemWeights w = carve_weights<NB>(p, PANELS ? OBS_PANEL : d, true);
    float* Xs = p;  p += P_M * ldx;
    float* N1s = p; p += P_M * LDA;
    float* N3s = p; p += P_M * LDA;
    float* DZs = p; p += P_M * LDA;
    float* DLs = p; if (!WIDE) p += P_M * DLW;
    float* row_a = p; p += P_M;   // policy: action      | critic: value_pred
    float* row_b = p; p += P_M;   // policy: old logp    | critic: return
    float* row_c = p; p += P_M;   // policy: raw adv
    float* row_act = p; p += P_M; // active mask
    float* red = p; p += 32;
    long long* row_idx = reinterpret_cast<long long*>(p); p += 2 * P_M;

    load_weights_folded<P_NT, NB, PANELS>(w, params, d, n, true);

    const bool pol_masks = a.flags & ORL_PPO_POLICY_ACTIVE_MASKS, val_masks = a.flags & ORL_PPO_VALUE_ACTIVE_MASKS;
    const MbConsts mb = mb_consts(a);

    const WgMap map3 = wg_map(16, 16);
    const WgMap map1 = wg_map(16, dp / 4);
    const int JBH = WIDE ? (n + 3) / 4 : n > 4 ? 2 : 1;
    const WgMap maph = wg_map(JBH, 16);
    float g3[4][4] = {}, g1[4][4] = {}, gh[4][4] = {}, db3[4] = {}, db1[4] = {}, dbh[4] = {};
    const bool gaussian = POLICY && !WIDE && a.head_kind == ORL_HEAD_GAUSSIAN;
    float dls_acc[MAX_OUT] = {};   // dL/dlogstd partial sums of this thread's rows (Gaussian head)
    float dls_wide = 0.f;          // GAUSS: dL/dlogstd[tid % 64] over this thread's rows
    float loss0 = 0.f, loss1 = 0.f, loss2 = 0.f;  // policy: policy_loss, entropy, ratio | critic: value_loss

    // G1 element (row 4 jb + r, column 64 pnl + 4 kb + c) of a panelled pass lives in this CTA's partial row; its owner
    // zeroes it first
    const int n_panels = (d + OBS_PANEL - 1) / OBS_PANEL;
    float* g1_part = nullptr;
    if constexpr (PANELS)
        g1_part = a.partials + (size_t)((POLICY ? 0 : G) + cta) * ppo_stride(a.obs_dim, a.critic_obs_dim, a.n_actions) +
                  fold_offsets(d, n).g1;
    auto g1_at = [&](int pnl, int r, int c) -> float* {
        return g1_part + (4 * map1.jb + r) * d + OBS_PANEL * pnl + 4 * map1.kb + c;
    };
    if constexpr (PANELS) {
        for (int pnl = 0; pnl < n_panels; ++pnl)
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c)
                    if (OBS_PANEL * pnl + 4 * map1.kb + c < d) *g1_at(pnl, r, c) = 0.f;
    }
    auto obs_row = [&](int r) -> const float* { return row_idx[r] >= 0 ? obs + row_idx[r] * d : nullptr; };

    const long long n_tiles = (a.batch_rows + P_M - 1) / P_M;
    for (long long tile = cta; tile < n_tiles; tile += G) {
        const long long r0 = tile * P_M;
        const int rows_here = (int)min((long long)P_M, a.batch_rows - r0);
        // ---- gather (replay_data.py:616-646) ----
        if (tid < P_M) {
            long long gi = -1;
            if (tid < rows_here) gi = a.indices ? a.indices[r0 + tid] : a.row_begin + r0 + tid;
            row_idx[tid] = gi;
            if (gi >= 0) {
                if (POLICY) { row_a[tid] = a.actions[gi]; row_b[tid] = a.old_log_probs[gi]; row_c[tid] = a.advantages[gi]; }
                else { row_a[tid] = a.value_preds[gi]; row_b[tid] = a.returns[gi]; }
                row_act[tid] = a.active_masks[gi];
            }
        }
        __syncthreads();
        // ---- (gather +) forward ----
        float mu1[P_RPT], rstd1[P_RPT], rstd3[P_RPT];
        unsigned posmask;
        float acc[P_RPT][4];
        if constexpr (PANELS) {
            fc1_panels<P_M, P_NT>(w, params + net_offsets(d, n).w1, d, Xs, obs_row, acc);
            trunk_from_z1<P_M, P_NT, true>(w, acc, a.activation_id, N1s, N3s, mu1, rstd1, rstd3, posmask);
        } else {
            for (int i = tid; i < P_M * ldx; i += P_NT) {
                const int r = i / ldx, k = i % ldx;
                const long long gi = row_idx[r];
                Xs[i] = (gi >= 0 && k < d) ? obs[gi * d + k] : 0.f;
            }
            __syncthreads();
            trunk_forward<P_M, P_NT, true>(w, Xs, ldx, d, a.activation_id, N1s, N3s, mu1, rstd1, rstd3, posmask);
        }
        __syncthreads();
        if constexpr (WIDE) {
            head_tile<P_M, P_NT>(w, N3s, DZs);
            __syncthreads();
            if constexpr (GAUSS) {   // the means tile becomes the dL/dmean tile, K = pad4(n) columns
                constexpr int RG = P_NT / MAX_OUT_WIDE;   // row groups
                const int j = tid % MAX_OUT_WIDE;
                if (j < pad4(n)) {
                    const float ls = j < n ? params[net_offsets(d, n, 1).ls + j] : 0.f, std = expf(ls), var = std * std;
                    const float ent_j = gaussian_entropy(ls);
                    for (int r = tid / MAX_OUT_WIDE; r < P_M; r += RG) {
                        float* x = DZs + r * LDA + j;
                        if (r < rows_here && j < n) {
                            const long long gi = row_idx[r];
                            const float active = row_act[r];
                            const float wrow = mb.weight(pol_masks, active);
                            const float went_row = pol_masks ? active * mb.inv_act : mb.inv_rows / (float)n;
                            const float diff = a.actions[gi * n + j] - *x;
                            const PgTerm pg = pg_term(gaussian_log_prob(diff, std, ls), a.old_log_probs[gi * n + j],
                                                      apply_adv_norm(mb.adv, row_c[r]), a.clip_param, a.flags, a.dual_clip_coeff);
                            loss0 += pg.loss * wrow;
                            loss1 += ent_j * went_row;
                            loss2 += pg.ratio / (float)n;
                            const float dlp = pg.dlogp * wrow;
                            *x = dlp * diff / var;
                            dls_wide += dlp * (diff * diff / var - 1.0f) - a.entropy_coef * went_row;
                        } else {
                            *x = 0.f;
                        }
                    }
                }
            } else if (tid < P_M) {   // one thread per row: the logits row becomes the dL/dlogits row
                float* x = DZs + tid * LDA;
                if (tid < rows_here) {
                    const long long gi = row_idx[tid];
                    const float wrow = mb.weight(pol_masks, row_act[tid]);
                    const CatRow c = wide_categorical_row(a, x, n, a.action_masks ? a.action_masks + gi * n : nullptr, (int)row_a[tid],
                                                          row_b[tid], apply_adv_norm(mb.adv, row_c[tid]), wrow);
                    loss0 += c.loss * wrow;
                    loss1 += c.ent * wrow;
                    loss2 += c.ratio;
                } else {
                    for (int j = 0; j < pad4(n); ++j) x[j] = 0.f;
                }
            }
            __syncthreads();
            // ---- backward: head -> LN3 ----
#pragma unroll
            for (int i = 0; i < P_RPT; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }
            gemm_tile<P_RPT, P_TY>(DZs, LDA, w.whf, pad4(n), acc, tx, ty);   // dn3 = dL . Whf
            wgrad_acc(DZs, LDA, N3s, LDA, maph, gh, dbh);                   // GH += dL^T n3
            {
                float nrm[P_RPT][4];
                load_tile<P_RPT, P_TY>(N3s, nrm, tx, ty);
                layernorm_bwd_rows<P_RPT>(acc, nrm, rstd3);
            }
            __syncthreads();                                                 // all reads of dL done
            store_tile<P_RPT, P_TY>(DZs, acc, tx, ty);                       // dZ3
            __syncthreads();
        } else {
            float out[MAX_OUT];
            head_dots<P_M, P_NT>(w, N3s, n, out);
            {
                constexpr int PPR = P_NT / P_M;
                const int row = tid / PPR;
                if (tid % PPR == 0) {
                    float dl[DLW];
#pragma unroll
                    for (int j = 0; j < DLW; ++j) dl[j] = 0.f;
                    if (row < rows_here) {
                        const float active = row_act[row];
                        if (POLICY && gaussian) {
                            const long long gi = row_idx[row];
                            const float went_row = pol_masks ? active * mb.inv_act : mb.inv_rows / (float)n;
                            gaussian_row(a, out, n, params + net_offsets(d, n, 1).ls, a.actions + gi * n, a.old_log_probs + gi * n,
                                         apply_adv_norm(mb.adv, row_c[row]), mb.weight(pol_masks, active), went_row, dl, dls_acc,
                                         loss0, loss1, loss2);
                        } else if (POLICY) {
                            const long long gi = row_idx[row];
                            const float wrow = mb.weight(pol_masks, active);
                            const CatRow c = categorical_row(a, out, n, a.action_masks ? a.action_masks + gi * n : nullptr, (int)row_a[row],
                                                             row_b[row], apply_adv_norm(mb.adv, row_c[row]), wrow, dl);
                            loss0 += c.loss * wrow;
                            loss1 += c.ent * wrow;
                            loss2 += c.ratio;
                        } else {
                            const float ret = row_b[row];
                            const float target = (a.flags & ORL_PPO_VALUENORM) ? (ret - mb.vn_mean) / mb.vn_std : ret;
                            const ValueTerm vt = value_term(out[0], row_a[row], target, a.clip_param, a.huber_delta, a.flags);
                            const float wrow = mb.weight(val_masks, active);
                            loss0 += vt.loss * wrow;
                            dl[0] = a.value_loss_coef * wrow * vt.dv;
                        }
                    }
                    *reinterpret_cast<float4*>(DLs + row * DLW) = make_float4(dl[0], dl[1], dl[2], dl[3]);
                    *reinterpret_cast<float4*>(DLs + row * DLW + 4) = make_float4(dl[4], dl[5], dl[6], dl[7]);
                }
            }
            __syncthreads();

            // ---- backward: head -> LN3 ----
#pragma unroll
            for (int i = 0; i < P_RPT; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }
            for (int j = 0; j < n; ++j) {
                const float4 wv = *reinterpret_cast<const float4*>(w.whf + j * H + 4 * tx);
#pragma unroll
                for (int i = 0; i < P_RPT; ++i) {
                    const float dlv = DLs[(ty + P_TY * i) * DLW + j];
                    acc[i][0] = fmaf(dlv, wv.x, acc[i][0]); acc[i][1] = fmaf(dlv, wv.y, acc[i][1]);
                    acc[i][2] = fmaf(dlv, wv.z, acc[i][2]); acc[i][3] = fmaf(dlv, wv.w, acc[i][3]);
                }
            }
            {
                float nrm[P_RPT][4];
                load_tile<P_RPT, P_TY>(N3s, nrm, tx, ty);
                layernorm_bwd_rows<P_RPT>(acc, nrm, rstd3);
            }
            store_tile<P_RPT, P_TY>(DZs, acc, tx, ty);   // dZ3
            wgrad_acc(DLs, DLW, N3s, LDA, maph, gh, dbh);  // GH += dL^T n3
            __syncthreads();
        }

        // ---- fc3 backward ----
        wgrad_acc(DZs, LDA, N1s, LDA, map3, g3, db3);  // G3 += dZ3^T n1
#pragma unroll
        for (int i = 0; i < P_RPT; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }
        gemm_tile<P_RPT, P_TY>(DZs, LDA, w.w3n, H, acc, tx, ty);  // dn1 = dZ3 . W3f
        {
            float nrm[P_RPT][4];
            load_tile<P_RPT, P_TY>(N1s, nrm, tx, ty);
            layernorm_bwd_rows<P_RPT>(acc, nrm, rstd1);
#pragma unroll
            for (int i = 0; i < P_RPT; ++i) {
                const float stdv = 1.0f / rstd1[i];
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const float aval = fmaf(nrm[i][c], stdv, mu1[i]);
                    acc[i][c] *= act_bwd(aval, (posmask >> (i * 4 + c)) & 1u, a.activation_id);
                }
            }
        }
        __syncthreads();                               // all reads of dZ3 done
        store_tile<P_RPT, P_TY>(DZs, acc, tx, ty);     // dZ1
        __syncthreads();
        if constexpr (PANELS) {   // G1_p = dZ1^T X_p, last panel first (it is still in Xs); db1 with panel 0
            for (int pnl = n_panels - 1; pnl >= 0; --pnl) {
                if (pnl != n_panels - 1) {
                    stage_obs_panel<P_M, P_NT>(Xs, d, pnl, obs_row);
                    __syncthreads();
                }
                float gp[4][4] = {}, dbp[4] = {};
                wgrad_acc(DZs, LDA, Xs, LDX_PANEL, map1, gp, dbp);
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    if (pnl == 0) db1[r] += dbp[r];
#pragma unroll
                    for (int c = 0; c < 4; ++c)
                        if (OBS_PANEL * pnl + 4 * map1.kb + c < d) *g1_at(pnl, r, c) += gp[r][c];
                }
                __syncthreads();
            }
        } else {
            wgrad_acc(DZs, LDA, Xs, ldx, map1, g1, db1);   // G1 += dZ1^T X
            __syncthreads();
        }
    }

    // ---- flush this CTA's partial folded gradients + loss sums ----
    const int stride = ppo_stride(a.obs_dim, a.critic_obs_dim, a.n_actions);
    float* part = a.partials + (size_t)((POLICY ? 0 : G) + cta) * stride;
    const FoldOffsets fo = fold_offsets(d, n);
    float* scratch = N1s;  // >= 16*(64*4+64) floats needed at most; N1s..DZs is 3*128*68 floats
    if constexpr (PANELS) {   // G1 is in place; one thread per 4 rows of db1 (MG = 1)
        if (map1.kb == 0) {
#pragma unroll
            for (int r = 0; r < 4; ++r) part[fo.db1 + 4 * map1.jb + r] = db1[r];
        }
    } else {
        wgrad_flush(scratch, map1, 16, dp / 4, g1, db1, H, d, part + fo.g1, part + fo.db1);
    }
    wgrad_flush(scratch, map3, 16, 16, g3, db3, H, H, part + fo.g3, part + fo.db3);
    wgrad_flush(scratch, maph, JBH, 16, gh, dbh, n, H, part + fo.gh, part + fo.dbh);
    __syncthreads();
    if (GAUSS) {    // dL/dlogstd: the 4 row groups' partials of each dimension, in row-group order
        scratch[tid] = dls_wide;
        __syncthreads();
        if (tid < n) {
            float sv = 0.f;
            for (int g2 = 0; g2 < P_NT / MAX_OUT_WIDE; ++g2) sv += scratch[g2 * MAX_OUT_WIDE + tid];
            part[fo.dls + tid] = sv;
        }
        __syncthreads();
    } else if (WIDE) {     // no logstd: a Categorical head
        if (tid < n) part[fo.dls + tid] = 0.f;
    } else if (POLICY) {   // dL/dlogstd: block reduction of the per-thread partial sums (zero for categorical heads)
        const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
        for (int j = 0; j < MAX_OUT; ++j) {
            const float sv = warp_sum(dls_acc[j]);
            if (lane == 0) scratch[j * 8 + warp] = sv;
        }
        __syncthreads();
        if (tid < n) {
            float sv = 0.f;
            for (int wv = 0; wv < P_NT / 32; ++wv) sv += scratch[tid * 8 + wv];
            part[fo.dls + tid] = sv;
        }
        __syncthreads();
    } else if (tid < n) {
        part[fo.dls + tid] = 0.f;
    }
    {
        float v[3] = {loss0, loss1, loss2};
        const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float s = warp_sum(v[k]);
            if (lane == 0) red[k * 8 + warp] = s;
        }
        __syncthreads();
        if (tid < N_LOSS) {
            float s = 0.f;
            if (tid < 3) for (int wv = 0; wv < P_NT / 32; ++wv) s += red[tid * 8 + wv];
            part[stride - N_LOSS + tid] = s;
        }
    }
}

// PANELS_POLICY / PANELS_CRITIC: that net's observation is wider than 64 and its pass runs fc1 in panels
template <int NB, bool PANELS_POLICY, bool PANELS_CRITIC>
__global__ void __launch_bounds__(P_NT, 1) ppo_fwdbwd_kernel(const OrlPpoArgs a) {
    extern __shared__ __align__(16) float smem[];
    const int G = a.grid_per_net;
    if ((int)blockIdx.x < G) ppo_net_pass<true, NB, PANELS_POLICY>(a, smem, blockIdx.x, G);
    else ppo_net_pass<false, MAX_OUT, PANELS_CRITIC>(a, smem, blockIdx.x - G, G);
}

// the update of a DiagGaussian head of 1..64 dimensions (ORL_HEAD_GAUSSIAN_WIDE); the critic pass is the NB = 8 one
template <bool PANELS_POLICY, bool PANELS_CRITIC>
__global__ void __launch_bounds__(P_NT, 1) ppo_fwdbwd_gaussian_wide_kernel(const OrlPpoArgs a) {
    extern __shared__ __align__(16) float smem[];
    const int G = a.grid_per_net;
    if ((int)blockIdx.x < G) ppo_net_pass<true, MAX_OUT_WIDE, PANELS_POLICY, true>(a, smem, blockIdx.x, G);
    else ppo_net_pass<false, MAX_OUT, PANELS_CRITIC>(a, smem, blockIdx.x - G, G);
}

// Sum over the G partial rows of one net for 32 consecutive bucket elements per CTA (8 warps): warp w adds rows
// w, w+8, ... (coalesced 128-byte loads, 8 independent loads in flight per thread), the 8 partial sums are combined in
// warp order -> a fixed summation order (deterministic), ~2 us instead of ~12 us for the G = 132 sequential loads per thread.
constexpr int RED_W = 8, RED_NT = 32 * RED_W;
__device__ __forceinline__ float reduce_partials(const float* __restrict__ partials, int net, int G, int stride, int el,
                                                 float (*part)[32]) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    float s0 = 0.f, s1 = 0.f;
    if (el < stride) {
        const float* p = partials + (size_t)net * G * stride + el;
        int g = w;
#pragma unroll 4
        for (; g + RED_W < G; g += 2 * RED_W) { s0 += p[(size_t)g * stride]; s1 += p[(size_t)(g + RED_W) * stride]; }
        if (g < G) s0 += p[(size_t)g * stride];
    }
    part[w][lane] = s0 + s1;
    __syncthreads();
    float t = 0.f;
    if (w == 0) {
#pragma unroll
        for (int k = 0; k < RED_W; ++k) t += part[k][lane];
    }
    return t;   // valid in warp 0
}

// folded[net][i] = sum over the G partial rows of that net
__global__ void __launch_bounds__(RED_NT) ppo_reduce_kernel(const float* __restrict__ partials, float* __restrict__ folded, int G, int stride) {
    __shared__ float part[RED_W][32];
    const int net = blockIdx.y, el = blockIdx.x * 32 + (threadIdx.x & 31);
    const float s = reduce_partials(partials, net, G, stride, el, part);
    if (threadIdx.x < 32 && el < stride) folded[(size_t)net * stride + el] = s;
}

// ---- gradient-bucket exchange over NVLink peer memory, fused into the reduce and optimiser kernels -------------------
// Every rank owns a symmetric allocation mapped into all peers: floats [parity 2][source rank W][net 2][stride], then
// uint32 arrival flags [3][ORL_PEER_MAX_WORLD], then doubles [parity 2][ORL_PEER_SMALL_MAX] (orl_peer_sum_f64).
// Update number e of a net (1-based) uses half (e-1)&1.  PUSH: ppo_reduce_peer_kernel (76 CTAs) stores this rank's
// bucket straight into slot [half][my rank] of EVERY rank's allocation - posted NVLink writes, no round trip.  The apply
// CTA of that net then (a) publishes "my bucket for update e has been written everywhere" into every peer's flag word
// [net][my rank] (fence.sys + st.release.sys; the pushes are ordered before it by the kernel boundary), (b) waits until
// all W flag words of its own copy show >= e (ld.acquire.sys), (c) sums the W slots of its OWN copy in rank order - local
// reads, the same order on every rank, so all ranks hold bit-identical sums - and continues as the single-GPU optimiser.
// Two halves suffice: a rank pushes into half h again in update e+2, after its apply of e+1 saw every peer's flag e+1,
// and a peer raises flag e+1 only after its apply of e (the last reader of its half h) has retired.
__global__ void __launch_bounds__(RED_NT) ppo_reduce_peer_kernel(const float* __restrict__ partials, const OrlPeerArgs pa, int G, int stride) {
    __shared__ float part[RED_W][32];
    const int net = blockIdx.y, el = blockIdx.x * 32 + (threadIdx.x & 31);
    const float s = reduce_partials(partials, net, G, stride, el, part);
    if (threadIdx.x < 32 && el < stride) {
        const size_t off = ((size_t)(pa.epochs[net] & 1u) * pa.world + pa.rank) * 2u * stride + (size_t)net * stride + el;
        for (int q = 0; q < pa.world; ++q) reinterpret_cast<float*>(pa.peer_buffers[q])[off] = s;
    }
}

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ float4 ld_peer4(const float* p) {
    float4 v;
    asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint64_t global_ns() {
    uint64_t t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

__host__ __device__ __forceinline__ size_t peer_flag_word(int world, int stride) { return (size_t)4 * world * stride; }

// signal every peer's flag word [slot][my rank] with `e`, then wait until all W words of my own copy show >= e
__device__ __forceinline__ void peer_handshake(const OrlPeerArgs& pa, int slot, uint32_t e, size_t flag_word) {
    const int tid = threadIdx.x, W = pa.world;
    if (tid < W) {
        __threadfence_system();
        uint32_t* remote = reinterpret_cast<uint32_t*>(pa.peer_buffers[tid]) + flag_word + slot * ORL_PEER_MAX_WORLD + pa.rank;
        st_release_sys(remote, e);
        const uint32_t* mine = reinterpret_cast<const uint32_t*>(pa.peer_buffers[pa.rank]) + flag_word + slot * ORL_PEER_MAX_WORLD + tid;
        const uint64_t t0 = global_ns();
        unsigned spins = 0;
        while ((int32_t)(ld_acquire_sys(mine) - e) < 0) {
            if ((++spins & 1023u) == 0 && global_ns() - t0 > (uint64_t)pa.timeout_ms * 1000000ull) {
                atomicExch(pa.error_flag, 1 + tid);   // peer `tid` never arrived: the host raises on the next read-back
                break;
            }
        }
        __threadfence_system();
    }
    __syncthreads();
}

__device__ const float* peer_gather(const OrlPeerArgs& pa, int net, int stride) {
    const int tid = threadIdx.x, W = pa.world;
    const uint32_t e = pa.epochs[net] + 1u;
    peer_handshake(pa, net, e, peer_flag_word(W, stride));
    // the W slots of this rank's own copy (written by the peers; L1 is bypassed: ld.relaxed.sys)
    const float* base = pa.local_buffer + (size_t)((e - 1u) & 1u) * W * 2u * stride + (size_t)net * stride;
    float* out = pa.summed + (size_t)net * stride;
    for (int i = tid * 4; i < stride; i += blockDim.x * 4) {
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int q0 = 0; q0 < W; q0 += 8) {
            float4 v[8];
#pragma unroll
            for (int q = 0; q < 8; ++q)
                if (q0 + q < W) v[q] = ld_peer4(base + (size_t)(q0 + q) * 2u * stride + i);
#pragma unroll
            for (int q = 0; q < 8; ++q)
                if (q0 + q < W) { s.x += v[q].x; s.y += v[q].y; s.z += v[q].z; s.w += v[q].w; }
        }
        *reinterpret_cast<float4*>(out + i) = s;
    }
    __syncthreads();
    return out;
}

// SUM of n <= ORL_PEER_SMALL_MAX doubles over all ranks, in place (the once-per-iteration rollout moments): one CTA
__global__ void __launch_bounds__(64) peer_sum_f64_kernel(const OrlPeerArgs pa, double* __restrict__ data, int n, int stride) {
    const int tid = threadIdx.x, W = pa.world;
    const uint32_t e = pa.epochs[2] + 1u;
    const size_t flag_word = peer_flag_word(W, stride);
    const size_t small_byte = flag_word * 4 + (size_t)3 * ORL_PEER_MAX_WORLD * 4 + (size_t)((e - 1u) & 1u) * ORL_PEER_SMALL_MAX * 8;
    double* mine = reinterpret_cast<double*>(reinterpret_cast<char*>(pa.peer_buffers[pa.rank]) + small_byte);
    if (tid < n) mine[tid] = data[tid];
    __syncthreads();
    peer_handshake(pa, 2, e, flag_word);
    if (tid < n) {
        double s = 0.0;
        for (int q = 0; q < W; ++q) {
            double v;
            asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v)
                         : "l"(reinterpret_cast<const double*>(reinterpret_cast<const char*>(pa.peer_buffers[q]) + small_byte) + tid) : "memory");
            s += v;
        }
        data[tid] = s;
    }
    if (tid == 0) pa.epochs[2] = e;
}

template <bool PEER>
__global__ void __launch_bounds__(1024) ppo_apply_kernel(const OrlPpoArgs a, const OrlPeerArgs pa) {
    const int net = blockIdx.x;  // 0 policy, 1 critic
    const int d = net == 0 ? a.obs_dim : a.critic_obs_dim;
    const int n = net == 0 ? a.n_actions : 1;
    const int stride = ppo_stride(a.obs_dim, a.critic_obs_dim, a.n_actions);
    const NetOffsets po = net_offsets(d, n, net == 0 && a.head_kind == ORL_HEAD_GAUSSIAN);
    const FoldOffsets fo = fold_offsets(d, n);
    float* params = net == 0 ? a.policy_params : a.critic_params;
    float* am = net == 0 ? a.policy_adam_m : a.critic_adam_m;
    float* av = net == 0 ? a.policy_adam_v : a.critic_adam_v;
    float* grads = a.grads + (size_t)net * ppo_grads_stride(a.obs_dim, a.critic_obs_dim, a.n_actions);
    const int tid = threadIdx.x;
    const float* f = PEER ? peer_gather(pa, net, stride) : a.folded + (size_t)net * stride;

    float sq = 0.f;
    for (int i = tid; i < po.total; i += blockDim.x) {
        const float g = unfolded_grad(params, po, fo, f, i);
        grads[i] = g;
        sq = fmaf(g, g, sq);
    }
    const float norm = block_l2_norm(sq);
    adam_step(a, net, params, am, av, grads, po.total, clip_factor(a, norm));   // after every thread's unfolding reads of params
    if (tid == 0) {
        if (PEER) {
            pa.epochs[net] += 1u;
            // a peer timed out: poison the logged scalars so that the host's one read-back sees it (it then reads error_flag)
            if (*reinterpret_cast<volatile int32_t*>(pa.error_flag) != 0) a.train_info[net == 0 ? 2 : 0] = __int_as_float(0x7fc00000);
        }
        const float* ls = f + stride - N_LOSS;
        if (net == 0) add_policy_info(a, ls, norm);
        else add_value_info(a, ls[0], norm);
    }
}

__global__ void minibatch_stats_kernel(const int64_t* __restrict__ idx, int64_t rows, const float* __restrict__ returns,
                                       const float* __restrict__ active, double* __restrict__ out) {
    double s0 = 0, s1 = 0, s2 = 0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < rows; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t g = idx[i];
        const double r = returns[g];
        s0 += r; s1 += r * r; s2 += active[g];
    }
    __shared__ double red[3][8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    s0 = warp_sum(s0); s1 = warp_sum(s1); s2 = warp_sum(s2);
    if (lane == 0) { red[0][warp] = s0; red[1][warp] = s1; red[2][warp] = s2; }
    __syncthreads();
    if (threadIdx.x < 3) {
        double t = 0;
        for (int wv = 0; wv < (int)(blockDim.x >> 5); ++wv) t += red[threadIdx.x][wv];
        atomicAdd(out + threadIdx.x, t);
    }
}

size_t fwdbwd_smem_bytes(int d, int dc) {
    const int dm = std::max(d, dc);
    const int ldx = orl::pad4(dm) + 4;
    const size_t floats = orl::smem_weights_floats(dm, true) + (size_t)P_M * ldx + 3 * (size_t)P_M * orl::LDA +
                          (size_t)P_M * DLW + 4 * P_M + 32 + 4 * P_M /* row_idx as 2 floats each */ + 16;
    return floats * sizeof(float);
}
// the wide policy pass (no separate dL tile) or the critic pass, whichever needs more
size_t fwdbwd_wide_smem_bytes(int d, int dc) {
    const size_t rest = (size_t)4 * P_M + 32 + 4 * P_M + 16;
    const size_t pol = orl::smem_weights_floats<orl::MAX_OUT_WIDE>(d, true) + (size_t)P_M * (orl::pad4(d) + 4) + 3 * (size_t)P_M * orl::LDA + rest;
    const size_t cri = orl::smem_weights_floats(dc, true) + (size_t)P_M * (orl::pad4(dc) + 4) + 3 * (size_t)P_M * orl::LDA + (size_t)P_M * DLW + rest;
    return std::max(pol, cri) * sizeof(float);
}

// The arguments ppo_apply_kernel runs on: both DiagGaussian kinds have one parameter layout (logstd[n] after bh) and one
// folded layout, and the kernel finds logstd from head_kind == ORL_HEAD_GAUSSIAN; so ORL_HEAD_GAUSSIAN_WIDE runs as that.
OrlPpoArgs apply_args(const OrlPpoArgs& a) {
    OrlPpoArgs b = a;
    if (b.head_kind == ORL_HEAD_GAUSSIAN_WIDE) b.head_kind = ORL_HEAD_GAUSSIAN;
    return b;
}

int check_ppo_args(const OrlPpoArgs& a) {
    ORL_CHECK_ARG(a.obs_dim > 0 && a.obs_dim <= orl::MAX_OBS_WIDE && a.critic_obs_dim > 0 && a.critic_obs_dim <= orl::MAX_OBS_WIDE,
                  "obs dims must be in 1..256");
    ORL_CHECK_ARG(a.n_actions > 0 && a.n_actions <= orl::MAX_OUT_WIDE, "n_actions must be in 1..64");
    ORL_CHECK_ARG(a.n_actions <= orl::MAX_OUT || a.head_kind == ORL_HEAD_CATEGORICAL || a.head_kind == ORL_HEAD_GAUSSIAN_WIDE,
                  "n_actions must be in 1..8 for Gaussian heads (1..64 for Categorical heads)");
    ORL_CHECK_ARG(a.activation_id >= 0 && a.activation_id <= 3, "activation_id");
    ORL_CHECK_ARG(a.grid_per_net > 0, "grid_per_net");
    ORL_CHECK_ARG(a.batch_rows > 0, "batch_rows");
    ORL_CHECK_ARG(a.policy_params && a.critic_params && a.partials && a.folded && a.grads && a.train_info, "null buffer");
    return 0;
}

}  // namespace

namespace orl {
int ppo_stride_host(int obs_dim, int critic_obs_dim, int n_actions) { return ppo_stride(obs_dim, critic_obs_dim, n_actions); }
int launch_ppo_fwdbwd_tc(const OrlPpoArgs& a, cudaStream_t st);
}  // namespace orl

extern "C" int orl_ppo_stride(int obs_dim, int critic_obs_dim, int n_actions) {
    return ppo_stride(obs_dim, critic_obs_dim, n_actions);
}

extern "C" int orl_ppo_grads_stride(int obs_dim, int critic_obs_dim, int n_actions) {
    return ppo_grads_stride(obs_dim, critic_obs_dim, n_actions);
}

extern "C" int orl_net_param_count(int obs_dim, int n_out) { return orl::net_offsets(obs_dim, n_out).total; }

extern "C" int orl_ppo_fwdbwd(const OrlPpoArgs* args, void* stream) {
    ORL_CHECK_ARG(args, "args");
    const OrlPpoArgs& a = *args;
    if (int e = check_ppo_args(a)) return e;
    ORL_CHECK_ARG(a.policy_obs && a.critic_obs && a.actions && a.old_log_probs && a.advantages && a.value_preds &&
                      a.returns && a.active_masks && a.gae_stats && a.mb_stats, "null rollout buffer");
    ORL_CHECK_ARG(!(a.flags & ORL_PPO_VALUENORM) || a.vn_state, "vn_state required with VALUENORM");
    ORL_CHECK_ARG(a.indices || (a.row_begin >= 0 && a.row_begin + a.batch_rows <= a.total_rows), "row range");
    ORL_CHECK_ARG(a.head_kind == ORL_HEAD_CATEGORICAL || a.head_kind == ORL_HEAD_GAUSSIAN || a.head_kind == ORL_HEAD_GAUSSIAN_WIDE,
                  "head_kind");
    if (a.flags & ORL_PPO_TF32) {
        ORL_CHECK_ARG(a.head_kind != ORL_HEAD_GAUSSIAN_WIDE, "ORL_PPO_TENSORCORE: ORL_HEAD_GAUSSIAN_WIDE is not supported");
        ORL_CHECK_ARG(a.n_actions <= orl::MAX_OUT, "ORL_PPO_TENSORCORE: n_actions must be in 1..8");
        ORL_CHECK_ARG(a.obs_dim <= orl::OBS_PANEL && a.critic_obs_dim <= orl::OBS_PANEL, "ORL_PPO_TENSORCORE: obs dims must be in 1..64");
        if (a.head_kind != ORL_HEAD_CATEGORICAL) {
            orl::set_last_error("orl_ppo_fwdbwd: ORL_PPO_TENSORCORE supports categorical heads only");
            return ORL_ERR_UNSUPPORTED;
        }
        return orl::launch_ppo_fwdbwd_tc(a, reinterpret_cast<cudaStream_t>(stream));
    }
    const bool wide = a.n_actions > orl::MAX_OUT;
    // a panelled pass uses the buffers of the d = 64 layout
    const int ds = std::min(a.obs_dim, orl::OBS_PANEL), dcs = std::min(a.critic_obs_dim, orl::OBS_PANEL);
    const size_t smem = wide ? fwdbwd_wide_smem_bytes(ds, dcs) : fwdbwd_smem_bytes(ds, dcs);
    const bool pp = a.obs_dim > orl::OBS_PANEL, pc = a.critic_obs_dim > orl::OBS_PANEL;
    void (*const kern)(OrlPpoArgs) =
        !pp && !pc ? (wide ? ppo_fwdbwd_kernel<orl::MAX_OUT_WIDE, false, false> : ppo_fwdbwd_kernel<orl::MAX_OUT, false, false>)
        : wide ? (pp && pc ? ppo_fwdbwd_kernel<orl::MAX_OUT_WIDE, true, true>
                  : pp ? ppo_fwdbwd_kernel<orl::MAX_OUT_WIDE, true, false> : ppo_fwdbwd_kernel<orl::MAX_OUT_WIDE, false, true>)
               : (pp && pc ? ppo_fwdbwd_kernel<orl::MAX_OUT, true, true>
                  : pp ? ppo_fwdbwd_kernel<orl::MAX_OUT, true, false> : ppo_fwdbwd_kernel<orl::MAX_OUT, false, true>);
    if (a.head_kind == ORL_HEAD_GAUSSIAN_WIDE) {   // the wide layout whatever the width (fwdbwd_wide_smem_bytes)
        void (*const gk)(OrlPpoArgs) = pp && pc ? ppo_fwdbwd_gaussian_wide_kernel<true, true>
                                       : pp ? ppo_fwdbwd_gaussian_wide_kernel<true, false>
                                       : pc ? ppo_fwdbwd_gaussian_wide_kernel<false, true> : ppo_fwdbwd_gaussian_wide_kernel<false, false>;
        const size_t gsmem = fwdbwd_wide_smem_bytes(ds, dcs);   // 226 240 B at d = dc = 256 (the d = 64 layout)
        if (gsmem > 227 * 1024) {
            orl::set_last_error("orl_ppo_fwdbwd: the wide DiagGaussian pass needs %zu bytes of shared memory", gsmem);
            return ORL_ERR_UNSUPPORTED;
        }
        if (int e = orl::allow_dynamic_smem(gk, 227 * 1024)) return e;
        gk<<<2 * a.grid_per_net, P_NT, gsmem, reinterpret_cast<cudaStream_t>(stream)>>>(a);
        ORL_LAUNCH_CHECK("ppo_fwdbwd_gaussian_wide_kernel");
        return 0;
    }
    if (int e = orl::allow_dynamic_smem(kern, 227 * 1024)) return e;
    kern<<<2 * a.grid_per_net, P_NT, smem, reinterpret_cast<cudaStream_t>(stream)>>>(a);
    ORL_LAUNCH_CHECK("ppo_fwdbwd_kernel");
    return 0;
}

extern "C" int orl_ppo_reduce(const OrlPpoArgs* args, void* stream) {
    ORL_CHECK_ARG(args, "args");
    const OrlPpoArgs& a = *args;
    if (int e = check_ppo_args(a)) return e;
    const int stride = orl_ppo_stride(a.obs_dim, a.critic_obs_dim, a.n_actions);
    dim3 grid((stride + 31) / 32, 2);
    ppo_reduce_kernel<<<grid, RED_NT, 0, reinterpret_cast<cudaStream_t>(stream)>>>(a.partials, a.folded, a.grid_per_net, stride);
    ORL_LAUNCH_CHECK("ppo_reduce_kernel");
    return 0;
}

static int check_peer_args(const OrlPeerArgs& pa) {
    ORL_CHECK_ARG(pa.world >= 2 && pa.world <= ORL_PEER_MAX_WORLD && pa.rank >= 0 && pa.rank < pa.world, "peer world / rank");
    ORL_CHECK_ARG(pa.peer_buffers && pa.local_buffer && pa.epochs && pa.error_flag && pa.summed, "null peer buffer");
    ORL_CHECK_ARG(pa.timeout_ms > 0, "timeout_ms");
    return 0;
}

extern "C" long long orl_ppo_peer_bucket_bytes(int obs_dim, int critic_obs_dim, int n_actions, int world) {
    const int stride = orl_ppo_stride(obs_dim, critic_obs_dim, n_actions);
    return (long long)peer_flag_word(world, stride) * sizeof(float) + (long long)3 * ORL_PEER_MAX_WORLD * sizeof(uint32_t) +
           (long long)2 * ORL_PEER_SMALL_MAX * sizeof(double);
}

extern "C" int orl_peer_sum_f64(const OrlPeerArgs* peer, int stride, double* data, int n, void* stream) {
    ORL_CHECK_ARG(peer && data && stride > 0 && stride % 4 == 0, "args");
    if (int e = check_peer_args(*peer)) return e;
    ORL_CHECK_ARG(n > 0 && n <= ORL_PEER_SMALL_MAX, "n must be in 1..ORL_PEER_SMALL_MAX");
    peer_sum_f64_kernel<<<1, 64, 0, reinterpret_cast<cudaStream_t>(stream)>>>(*peer, data, n, stride);
    ORL_LAUNCH_CHECK("peer_sum_f64_kernel");
    return 0;
}

extern "C" int orl_ppo_reduce_peer(const OrlPpoArgs* args, const OrlPeerArgs* peer, void* stream) {
    ORL_CHECK_ARG(args && peer, "args");
    const OrlPpoArgs& a = *args;
    if (int e = check_ppo_args(a)) return e;
    if (int e = check_peer_args(*peer)) return e;
    const int stride = orl_ppo_stride(a.obs_dim, a.critic_obs_dim, a.n_actions);
    dim3 grid((stride + 31) / 32, 2);
    ppo_reduce_peer_kernel<<<grid, RED_NT, 0, reinterpret_cast<cudaStream_t>(stream)>>>(a.partials, *peer, a.grid_per_net, stride);
    ORL_LAUNCH_CHECK("ppo_reduce_kernel(peer)");
    return 0;
}

extern "C" int orl_ppo_apply_peer(const OrlPpoArgs* args, const OrlPeerArgs* peer, void* stream) {
    ORL_CHECK_ARG(args && peer, "args");
    const OrlPpoArgs& a = *args;
    if (int e = check_ppo_args(a)) return e;
    if (int e = check_peer_args(*peer)) return e;
    ORL_CHECK_ARG(a.policy_adam_m && a.policy_adam_v && a.critic_adam_m && a.critic_adam_v && a.adam_steps && a.lrs,
                  "null optimiser state");
    ORL_CHECK_ARG(a.mb_stats, "mb_stats");
    ppo_apply_kernel<true><<<2, 1024, 0, reinterpret_cast<cudaStream_t>(stream)>>>(apply_args(a), *peer);
    ORL_LAUNCH_CHECK("ppo_apply_kernel(peer)");
    return 0;
}

extern "C" int orl_ppo_apply(const OrlPpoArgs* args, void* stream) {
    ORL_CHECK_ARG(args, "args");
    const OrlPpoArgs& a = *args;
    if (int e = check_ppo_args(a)) return e;
    ORL_CHECK_ARG(a.policy_adam_m && a.policy_adam_v && a.critic_adam_m && a.critic_adam_v && a.adam_steps && a.lrs,
                  "null optimiser state");
    ORL_CHECK_ARG(a.mb_stats, "mb_stats");
    ppo_apply_kernel<false><<<2, 1024, 0, reinterpret_cast<cudaStream_t>(stream)>>>(apply_args(a), OrlPeerArgs{});
    ORL_LAUNCH_CHECK("ppo_apply_kernel");
    return 0;
}

extern "C" int orl_minibatch_stats(const int64_t* indices, int64_t batch_rows, const float* returns,
                                   const float* active_masks, double* mb_stats_out, void* stream) {
    ORL_CHECK_ARG(indices && returns && active_masks && mb_stats_out && batch_rows > 0, "null buffer / rows");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    int e = orl::check_cuda(cudaMemsetAsync(mb_stats_out, 0, 3 * sizeof(double), st), "memset mb_stats");
    if (e) return e;
    const int grid = (int)std::min<int64_t>((batch_rows + 255) / 256, 4LL * orl::sm_count());
    minibatch_stats_kernel<<<grid, 256, 0, st>>>(indices, batch_rows, returns, active_masks, mb_stats_out);
    ORL_LAUNCH_CHECK("minibatch_stats_kernel");
    return 0;
}
