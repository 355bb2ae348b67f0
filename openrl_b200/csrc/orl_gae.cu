// GAE / discounted-return backward scan over the (T, B) rollout buffer, fused with the
// advantage construction and the moments its normalisation needs.
//
// Reference semantics: ReplayData.compute_returns, openrl/buffers/replay_data.py:320-423
// (8 branches) and PPOAlgorithm.train_ppo, openrl/algorithms/ppo.py:384-399.
//
// HBM-bound streaming scan: the B columns are independent, T is sequential.  One thread owns
// VEC adjacent columns (128-bit loads when VEC == 4) and walks t = T-1 .. 0; loads of a chunk of
// U timesteps are issued before the dependent gae chain so U*arrays requests are in flight per
// thread.  Algorithmic traffic: 16 B / element (rewards, value_preds, masks in; returns out),
// +4 B with bad_masks, +4 B advantages out, +4 B active_masks in (stats).
//
// Every float op is an explicit round-to-nearest intrinsic in the reference's numpy float32
// evaluation order (no FMA contraction) so the result is bit-exact with the reference.
#include "orl_common.cuh"

namespace {

template <int VEC> struct Vec;
template <> struct Vec<1> { float v[1]; };
template <> struct alignas(16) Vec<4> { float v[4]; };

template <int VEC>
__device__ __forceinline__ Vec<VEC> ldv(const float* __restrict__ p) {
    Vec<VEC> r;
    if constexpr (VEC == 4) {
        const float4 q = __ldg(reinterpret_cast<const float4*>(p));
        r.v[0] = q.x; r.v[1] = q.y; r.v[2] = q.z; r.v[3] = q.w;
    } else {
        r.v[0] = __ldg(p);
    }
    return r;
}
template <int VEC>
__device__ __forceinline__ void stv(float* __restrict__ p, const Vec<VEC>& r) {
    if constexpr (VEC == 4) {
        *reinterpret_cast<float4*>(p) = make_float4(r.v[0], r.v[1], r.v[2], r.v[3]);
    } else {
        *p = r.v[0];
    }
}

struct GaeParams {
    const float* rewards;
    float* value_preds;
    const float* masks;
    const float* bad_masks;
    const float* active_masks;
    const float* next_value;
    const float* vn_state;
    float* returns;
    float* advantages;
    double* stats;
    int T, B;
    float gamma;       // float32(gamma)
    float gamma_lambda;  // float32(gamma * gae_lambda) with the product taken in double
};

template <int VEC, int U, bool USE_GAE, bool PTL, bool DENORM, bool ADV, bool STATS>
__global__ void __launch_bounds__(128) gae_scan_kernel(const GaeParams p) {
    const int col = (blockIdx.x * blockDim.x + threadIdx.x) * VEC;
    const int T = p.T, B = p.B;
    const bool valid = col < B;

    float vn_mean = 0.f, vn_std = 1.f;
    if (DENORM) {
        const orl::VnScalars s = orl::vn_mean_std(p.vn_state);
        vn_mean = s.mean; vn_std = s.std;
    }
    auto denorm = [&](float v) -> float {
        return DENORM ? __fadd_rn(__fmul_rn(v, vn_std), vn_mean) : v;
    };

    double s_adv = 0, s_adv2 = 0, s_act_adv = 0, s_act_adv2 = 0, s_act_n = 0, s_ret = 0, s_ret2 = 0;

    if (valid) {
        // bootstrap row
        Vec<VEC> nv = ldv<VEC>(p.next_value + col);
        if (USE_GAE) stv<VEC>(p.value_preds + (size_t)T * B + col, nv);
        else stv<VEC>(p.returns + (size_t)T * B + col, nv);

        float carry[VEC];     // gae (USE_GAE) or returns[t+1] (!USE_GAE)
        float v1d[VEC];       // denorm(value_preds[t+1])
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
            carry[i] = USE_GAE ? 0.f : nv.v[i];
            v1d[i] = denorm(nv.v[i]);
        }

        for (int t_hi = T; t_hi > 0; t_hi -= U) {
            Vec<VEC> r[U], v[U], m[U], bad[U], act[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int t = t_hi - 1 - u;
                if (t >= 0) {
                    const size_t o = (size_t)t * B + col;
                    r[u] = ldv<VEC>(p.rewards + o);
                    v[u] = ldv<VEC>(p.value_preds + o);
                    m[u] = ldv<VEC>(p.masks + o + B);
                    if (PTL) bad[u] = ldv<VEC>(p.bad_masks + o + B);
                    if (STATS && p.active_masks) act[u] = ldv<VEC>(p.active_masks + o);
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int t = t_hi - 1 - u;
                if (t >= 0) {
                    Vec<VEC> ret, adv;
#pragma unroll
                    for (int i = 0; i < VEC; ++i) {
                        const float v0d = denorm(v[u].v[i]);
                        const float m1 = m[u].v[i];
                        float out;
                        if (USE_GAE) {
                            // delta = r + gamma*V'(t+1)*m(t+1) - V'(t)
                            const float delta = __fsub_rn(
                                __fadd_rn(r[u].v[i], __fmul_rn(__fmul_rn(p.gamma, v1d[i]), m1)), v0d);
                            float g;
                            if (PTL && DENORM) {
                                // replay_data.py:337-339: gamma*lambda*gae*mask
                                g = __fadd_rn(delta, __fmul_rn(__fmul_rn(p.gamma_lambda, carry[i]), m1));
                            } else {
                                // replay_data.py:352-355 / 395-398 / 410-413: gamma*lambda*mask*gae
                                g = __fadd_rn(delta, __fmul_rn(__fmul_rn(p.gamma_lambda, m1), carry[i]));
                            }
                            if (PTL) g = __fmul_rn(g, bad[u].v[i]);
                            carry[i] = g;
                            out = __fadd_rn(g, v0d);
                        } else {
                            // returns[t] = returns[t+1]*gamma*m(t+1) + r  (replay_data.py:419-422)
                            float x = __fadd_rn(__fmul_rn(__fmul_rn(carry[i], p.gamma), m1), r[u].v[i]);
                            if (PTL) {
                                const float b1 = bad[u].v[i];
                                // (...)*bad + (1-bad)*V'(t)   (replay_data.py:362-380)
                                x = __fadd_rn(__fmul_rn(x, b1), __fmul_rn(__fsub_rn(1.0f, b1), v0d));
                            }
                            carry[i] = x;
                            out = x;
                        }
                        ret.v[i] = out;
                        v1d[i] = v0d;
                        if (ADV || STATS) {
                            const float a = __fsub_rn(out, v0d);
                            adv.v[i] = a;
                            if (STATS) {
                                const double ad = (double)a;
                                s_adv += ad; s_adv2 += ad * ad;
                                const bool on = p.active_masks ? (act[u].v[i] != 0.0f) : true;
                                if (on) { s_act_adv += ad; s_act_adv2 += ad * ad; s_act_n += 1.0; }
                                const double rd = (double)out;
                                s_ret += rd; s_ret2 += rd * rd;
                            }
                        }
                    }
                    const size_t o = (size_t)t * B + col;
                    stv<VEC>(p.returns + o, ret);
                    if (ADV) stv<VEC>(p.advantages + o, adv);
                }
            }
        }
    }

    if (STATS) {
        __shared__ double red[7][4];
        double vals[7] = {s_adv, s_adv2, s_act_adv, s_act_adv2, s_act_n, s_ret, s_ret2};
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
        for (int k = 0; k < 7; ++k) {
            const double w = orl::warp_sum(vals[k]);
            if (lane == 0) red[k][warp] = w;
        }
        __syncthreads();
        if (threadIdx.x < 7) {
            const int k = threadIdx.x;
            const double tot = red[k][0] + red[k][1] + red[k][2] + red[k][3];
            // stats index map: see ORL_GS_*
            const int idx = (k == 0) ? ORL_GS_ADV_SUM : (k == 1) ? ORL_GS_ADV_SQSUM
                          : (k == 2) ? ORL_GS_ADV_ACT_SUM : (k == 3) ? ORL_GS_ADV_ACT_SQSUM
                          : (k == 4) ? ORL_GS_ACT_COUNT : (k == 5) ? ORL_GS_RET_SUM : ORL_GS_RET_SQSUM;
            if (tot != 0.0) atomicAdd(p.stats + idx, tot);
        }
        if (blockIdx.x == 0 && threadIdx.x == 0) p.stats[ORL_GS_COUNT] = (double)T * (double)B;
    }
}


// ---- small-B variant (default GAE branch: use_gae, no proper-time-limits) -----------------------
// With few columns the streaming kernel above is latency-bound: T dependent steps, each waiting on
// DRAM.  Here a CTA owns 32 columns and splits the work into (A) a fully parallel pass over all
// (t, column) elements that loads the inputs with every thread and computes the step-local terms
// delta_t and k_t = gamma*lambda*m_{t+1} into shared memory, (B) the serial recurrence
// g_t = delta_t + k_t*g_{t+1} from shared memory (2 dependent float ops per step, one thread per
// column), (C) a parallel epilogue (returns, advantages, moments, coalesced stores).  Same float32
// operation order per element as the streaming kernel, hence still bit-exact.
constexpr int TILE_COLS = 32, TILE_THREADS = 1024, TILE_WARPS = TILE_THREADS / 32, TILE_BATCH = 4;

template <bool DENORM, bool ADV, bool STATS>
__global__ void __launch_bounds__(TILE_THREADS) gae_tile_kernel(const GaeParams p) {
    extern __shared__ float tsm[];
    const int T = p.T, B = p.B;
    float* sdelta = tsm;                 // [T][32], overwritten by g in phase B
    float* sk = tsm + (size_t)T * TILE_COLS;
    const int col0 = blockIdx.x * TILE_COLS;
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
    const int col = col0 + lane;
    const bool valid = col < B;
    float vn_mean = 0.f, vn_std = 1.f;
    if (DENORM) { const orl::VnScalars s = orl::vn_mean_std(p.vn_state); vn_mean = s.mean; vn_std = s.std; }
    auto denorm = [&](float v) -> float { return DENORM ? __fadd_rn(__fmul_rn(v, vn_std), vn_mean) : v; };

    // bootstrap row (USE_GAE: value_preds[T] <- next_value); read next_value BEFORE it may be overwritten
    float nv = 0.f;
    if (valid && wrp == 0) nv = __ldg(p.next_value + col);
    // phase A: every warp takes rows t = wrp, wrp + 32, ...; the loads of TILE_BATCH rows are issued
    // together so their DRAM latencies overlap
    for (int t0 = wrp; t0 < T; t0 += TILE_WARPS * TILE_BATCH) {
        float r[TILE_BATCH], v0[TILE_BATCH], v1[TILE_BATCH], m1[TILE_BATCH];
#pragma unroll
        for (int u = 0; u < TILE_BATCH; ++u) {
            const int t = t0 + u * TILE_WARPS;
            if (valid && t < T) {
                const size_t o = (size_t)t * B + col;
                r[u] = __ldg(p.rewards + o); v0[u] = p.value_preds[o]; m1[u] = __ldg(p.masks + o + B);
                v1[u] = (t == T - 1) ? __ldg(p.next_value + col) : p.value_preds[o + B];
            }
        }
#pragma unroll
        for (int u = 0; u < TILE_BATCH; ++u) {
            const int t = t0 + u * TILE_WARPS;
            if (valid && t < T) {
                const float v0d = denorm(v0[u]), v1d = denorm(v1[u]);
                sdelta[t * TILE_COLS + lane] = __fsub_rn(__fadd_rn(r[u], __fmul_rn(__fmul_rn(p.gamma, v1d), m1[u])), v0d);
                sk[t * TILE_COLS + lane] = __fmul_rn(p.gamma_lambda, m1[u]);
            }
        }
    }
    __syncthreads();
    if (wrp == 0 && valid) {
        p.value_preds[(size_t)T * B + col] = nv;
        float g = 0.f;
#pragma unroll 8
        for (int t = T - 1; t >= 0; --t) {
            g = __fadd_rn(sdelta[t * TILE_COLS + lane], __fmul_rn(sk[t * TILE_COLS + lane], g));
            sdelta[t * TILE_COLS + lane] = g;
        }
    }
    __syncthreads();
    // phase C
    double s_adv = 0, s_adv2 = 0, s_act_adv = 0, s_act_adv2 = 0, s_act_n = 0, s_ret = 0, s_ret2 = 0;
    for (int t0 = wrp; t0 < T; t0 += TILE_WARPS * TILE_BATCH) {
        float v0[TILE_BATCH], am[TILE_BATCH];
#pragma unroll
        for (int u = 0; u < TILE_BATCH; ++u) {
            const int t = t0 + u * TILE_WARPS;
            if (valid && t < T) {
                const size_t o = (size_t)t * B + col;
                v0[u] = p.value_preds[o];
                am[u] = (STATS && p.active_masks) ? __ldg(p.active_masks + o) : 1.0f;
            }
        }
#pragma unroll
        for (int u = 0; u < TILE_BATCH; ++u) {
            const int t = t0 + u * TILE_WARPS;
            if (valid && t < T) {
                const size_t o = (size_t)t * B + col;
                const float v0d = denorm(v0[u]);
                const float g = sdelta[t * TILE_COLS + lane];
                const float ret = __fadd_rn(g, v0d);
                p.returns[o] = ret;
                if (ADV || STATS) {
                    const float a = __fsub_rn(ret, v0d);
                    if (ADV) p.advantages[o] = a;
                    if (STATS) {
                        const double ad = (double)a, rd = (double)ret;
                        s_adv += ad; s_adv2 += ad * ad; s_ret += rd; s_ret2 += rd * rd;
                        if (am[u] != 0.0f) { s_act_adv += ad; s_act_adv2 += ad * ad; s_act_n += 1.0; }
                    }
                }
            }
        }
    }
    if (STATS) {
        __shared__ double red[7][TILE_THREADS / 32];
        double vals[7] = {s_adv, s_adv2, s_act_adv, s_act_adv2, s_act_n, s_ret, s_ret2};
#pragma unroll
        for (int k = 0; k < 7; ++k) { const double w = orl::warp_sum(vals[k]); if (lane == 0) red[k][wrp] = w; }
        __syncthreads();
        if (threadIdx.x < 7) {
            const int k = threadIdx.x;
            double tot = 0;
            for (int w = 0; w < TILE_THREADS / 32; ++w) tot += red[k][w];
            const int idx = (k == 0) ? ORL_GS_ADV_SUM : (k == 1) ? ORL_GS_ADV_SQSUM : (k == 2) ? ORL_GS_ADV_ACT_SUM
                          : (k == 3) ? ORL_GS_ADV_ACT_SQSUM : (k == 4) ? ORL_GS_ACT_COUNT : (k == 5) ? ORL_GS_RET_SUM : ORL_GS_RET_SQSUM;
            if (tot != 0.0) atomicAdd(p.stats + idx, tot);
        }
        if (blockIdx.x == 0 && threadIdx.x == 0) p.stats[ORL_GS_COUNT] = (double)T * (double)B;
    }
}

template <bool DENORM>
int launch_gae_tile(const GaeParams& p, cudaStream_t st) {
    const int grid = (p.B + TILE_COLS - 1) / TILE_COLS;
    const size_t smem = (size_t)p.T * TILE_COLS * 2 * sizeof(float);
    const bool adv = p.advantages != nullptr, stats = p.stats != nullptr;
    if (stats) {
        int e = orl::check_cuda(cudaMemsetAsync(p.stats, 0, sizeof(double) * ORL_GAE_NSTATS, st), "memset stats");
        if (e) return e;
    }
    const auto kern = adv ? (stats ? gae_tile_kernel<DENORM, true, true> : gae_tile_kernel<DENORM, true, false>)
                          : (stats ? gae_tile_kernel<DENORM, false, true> : gae_tile_kernel<DENORM, false, false>);
    if (int e = orl::allow_dynamic_smem(kern, 200 * 1024)) return e;
    kern<<<grid, TILE_THREADS, smem, st>>>(p);
    ORL_LAUNCH_CHECK("gae_tile_kernel");
    return 0;
}

template <int VEC, int U, bool USE_GAE, bool PTL, bool DENORM>
int launch_gae2(const GaeParams& p, cudaStream_t st) {
    const int threads = 128;
    const int cols = (p.B + VEC - 1) / VEC;
    const int grid = (cols + threads - 1) / threads;
    const bool adv = p.advantages != nullptr, stats = p.stats != nullptr;
    if (stats) {
        int e = orl::check_cuda(cudaMemsetAsync(p.stats, 0, sizeof(double) * ORL_GAE_NSTATS, st), "memset stats");
        if (e) return e;
    }
    if (adv && stats) gae_scan_kernel<VEC, U, USE_GAE, PTL, DENORM, true, true><<<grid, threads, 0, st>>>(p);
    else if (adv) gae_scan_kernel<VEC, U, USE_GAE, PTL, DENORM, true, false><<<grid, threads, 0, st>>>(p);
    else if (stats) gae_scan_kernel<VEC, U, USE_GAE, PTL, DENORM, false, true><<<grid, threads, 0, st>>>(p);
    else gae_scan_kernel<VEC, U, USE_GAE, PTL, DENORM, false, false><<<grid, threads, 0, st>>>(p);
    ORL_LAUNCH_CHECK("gae_scan_kernel");
    return 0;
}

template <int VEC, int U>
int launch_gae(const GaeParams& p, int flags, cudaStream_t st) {
    const bool g = flags & ORL_GAE_USE_GAE, t = flags & ORL_GAE_PROPER_TIME_LIMITS, d = flags & ORL_GAE_DENORM;
    if (g) {
        if (t) return d ? launch_gae2<VEC, U, true, true, true>(p, st) : launch_gae2<VEC, U, true, true, false>(p, st);
        return d ? launch_gae2<VEC, U, true, false, true>(p, st) : launch_gae2<VEC, U, true, false, false>(p, st);
    }
    if (t) return d ? launch_gae2<VEC, U, false, true, true>(p, st) : launch_gae2<VEC, U, false, true, false>(p, st);
    // !gae & !ptl: the returns ignore the normaliser (replay_data.py:417-423) — the kernel's return
    // formula does not touch V in that branch — but the fused advantage still subtracts the
    // DENORMALISED value (ppo.py:384-399), so DENORM is honoured
    return d ? launch_gae2<VEC, U, false, false, true>(p, st) : launch_gae2<VEC, U, false, false, false>(p, st);
}

bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15u) == 0; }

}  // namespace

extern "C" int orl_gae(const float* rewards, float* value_preds, const float* masks,
                       const float* bad_masks, const float* active_masks, const float* next_value,
                       const float* vn_state, float* returns, float* advantages, double* stats,
                       int T, int B, double gamma, double gae_lambda, int flags, void* stream) {
    ORL_CHECK_ARG(rewards && value_preds && masks && next_value && returns, "null buffer");
    ORL_CHECK_ARG(T > 0 && B > 0, "T and B must be positive");
    ORL_CHECK_ARG(!(flags & ORL_GAE_PROPER_TIME_LIMITS) || bad_masks, "bad_masks required with PROPER_TIME_LIMITS");
    ORL_CHECK_ARG(!(flags & ORL_GAE_DENORM) || vn_state, "vn_state required with DENORM");
    GaeParams p;
    p.rewards = rewards; p.value_preds = value_preds; p.masks = masks; p.bad_masks = bad_masks;
    p.active_masks = active_masks; p.next_value = next_value; p.vn_state = vn_state;
    p.returns = returns; p.advantages = advantages; p.stats = stats; p.T = T; p.B = B;
    p.gamma = (float)gamma;
    p.gamma_lambda = (float)(gamma * gae_lambda);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const bool vec_ok = (B % 4 == 0) && aligned16(rewards) && aligned16(value_preds) && aligned16(masks) &&
                        aligned16(next_value) && aligned16(returns) && (!bad_masks || aligned16(bad_masks)) &&
                        (!active_masks || aligned16(active_masks)) && (!advantages || aligned16(advantages));
    // 128-bit columns only when there are enough of them to fill the machine (>= 2 waves of
    // 128-thread CTAs on every SM); otherwise scalar columns keep more threads in flight.
    const long long min_cols_for_vec = 2LL * orl::sm_count() * 16 * 128;
    if (vec_ok && (long long)(B / 4) >= min_cols_for_vec) return launch_gae<4, 4>(p, flags, st);
    // few columns: tile kernel (parallel load + short serial chain from shared memory) for the default branch
    const bool tile_branch = (flags & ORL_GAE_USE_GAE) && !(flags & ORL_GAE_PROPER_TIME_LIMITS);
    if (tile_branch && (long long)B < 16LL * orl::sm_count() * 128 && (size_t)T * TILE_COLS * 8 <= 160 * 1024)
        return (flags & ORL_GAE_DENORM) ? launch_gae_tile<true>(p, st) : launch_gae_tile<false>(p, st);
    return launch_gae<1, 8>(p, flags, st);
}
