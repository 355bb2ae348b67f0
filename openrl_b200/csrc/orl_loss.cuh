// The PPO loss maths, in one place: the categorical log-softmax and log-prob that the rollout sampler (orl_envstep.cuh)
// and policy_eval_kernel share with the updates, the DiagGaussian log-prob and entropy of policy_eval_kernel and the
// FFMA update, and the per-minibatch constants, categorical row loss and value row loss of every update kernel
// (ppo_net_pass in orl_ppo.cu, tc_net_pass in orl_ppo_tc.cu, the chunk and JRPO kernels of orl_rnn.cu,
// share_fwdbwd_kernel in orl_share.cu).  The DiagGaussian row loss serves ppo_net_pass (the FFMA update) and the
// shared model's share_fwdbwd_kernel: Box action spaces run those two updates.
#pragma once
#include "orl_mlp.cuh"

namespace orl {

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

// log_softmax_n of a row's logits with the masked-out actions (mask row entry 0, nullable) at -6e4; returns the
// masked-out actions as a bit set
__device__ __forceinline__ unsigned masked_log_softmax(float (&logit)[MAX_OUT], int n, const float* mask_row,
                                                       float (&nl)[MAX_OUT], float (&pr)[MAX_OUT]) {
    unsigned masked = 0;
    if (mask_row) {
#pragma unroll
        for (int j = 0; j < MAX_OUT; ++j)
            if (j < n && mask_row[j] == 0.f) { logit[j] = -6e4f; masked |= 1u << j; }
    }
    log_softmax_n(logit, n, nl, pr);
    return masked;
}

// log-prob of action `act`; an action outside [0, n) gets nl[0]
__device__ __forceinline__ float log_prob_of(const float (&nl)[MAX_OUT], int n, int act) {
    float lp = nl[0];
#pragma unroll
    for (int j = 1; j < MAX_OUT; ++j) if (j < n && j == act) lp = nl[j];
    return lp;
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

struct AdvNorm { float m0, s0, m1, s1; bool two_stage; };
__device__ __forceinline__ AdvNorm make_adv_norm(const double* __restrict__ gs, bool use_adv_normalize) {
    // ppo.py:402-409
    AdvNorm r;
    const double n_all = gs[ORL_GS_COUNT], n_act = gs[ORL_GS_ACT_COUNT];
    const double mean_all = gs[ORL_GS_ADV_SUM] / n_all;
    const double var_all = fmax(gs[ORL_GS_ADV_SQSUM] / n_all - mean_all * mean_all, 0.0);
    double mean_act = gs[ORL_GS_ADV_ACT_SUM] / n_act;
    const double var_act = fmax(gs[ORL_GS_ADV_ACT_SQSUM] / n_act - mean_act * mean_act, 0.0);
    double std_act = sqrt(var_act);
    r.two_stage = use_adv_normalize;
    r.m0 = 0.f; r.s0 = 1.f;
    if (use_adv_normalize) {
        const double s0 = (double)((float)sqrt(var_all)) + 1e-5;
        r.m0 = (float)mean_all;
        r.s0 = (float)s0;
        mean_act = (mean_act - mean_all) / s0;
        std_act = std_act / s0;
    }
    r.m1 = (float)mean_act;
    r.s1 = (float)((double)((float)std_act) + 1e-5);
    return r;
}
__device__ __forceinline__ float apply_adv_norm(const AdvNorm& r, float a) {
    if (r.two_stage) a = (a - r.m0) / r.s0;
    return (a - r.m1) / r.s1;
}

// ValueNorm.update (valuenorm.py:59-76) applied to the old state with this minibatch's moments.
__device__ __forceinline__ void vn_updated(const float* __restrict__ vn_state, const double* __restrict__ mb_stats,
                                           double batch_rows, double beta_d, float (&out)[3]) {
    const float bm = (float)(mb_stats[0] / batch_rows);
    const float bsq = (float)(mb_stats[1] / batch_rows);
    const float beta = (float)beta_d;
    const float omw = (float)(1.0 - beta_d);
    out[0] = __fadd_rn(__fmul_rn(vn_state[0], beta), __fmul_rn(bm, omw));
    out[1] = __fadd_rn(__fmul_rn(vn_state[1], beta), __fmul_rn(bsq, omw));
    out[2] = __fadd_rn(__fmul_rn(vn_state[2], beta), __fmul_rn(1.0f, omw));
}

// Rows behind the 1/rows loss weights, the reported ratio mean and the ValueNorm batch moments: the global minibatch
// (norm_rows) when ranks share the update, else this call's rows (feed-forward) or chunk steps (recurrent).
__device__ __forceinline__ double loss_rows(const OrlPpoArgs& a) { return (double)(a.norm_rows > 0 ? a.norm_rows : a.batch_rows); }
__device__ __forceinline__ double loss_rows(const OrlRnnArgs& a) {
    return a.norm_rows > 0 ? (double)a.norm_rows : (double)a.n_chunks * a.chunk_length;
}

// Per-minibatch constants of an update kernel, built once per kernel: the row weights 1/rows and 1/sum(active), the
// advantage normalisation, and the ValueNorm mean / std after this minibatch's update (0 / 1 without ORL_PPO_VALUENORM).
struct MbConsts {
    float inv_rows, inv_act;
    AdvNorm adv;
    float vn_mean, vn_std;
    // loss weight of a row: active / sum(active) with the active-mask option, else 1 / rows
    __device__ __forceinline__ float weight(bool use_active_masks, float active) const {
        return use_active_masks ? active * inv_act : inv_rows;
    }
};
template <class Args>
__device__ __forceinline__ MbConsts mb_consts(const Args& a) {
    MbConsts c;
    const double rows = loss_rows(a);
    c.inv_rows = (float)(1.0 / rows);
    c.inv_act = (float)(1.0 / a.mb_stats[2]);
    c.adv = make_adv_norm(a.gae_stats, a.flags & ORL_PPO_ADV_NORMALIZE);
    c.vn_mean = 0.f; c.vn_std = 1.f;
    if (a.flags & ORL_PPO_VALUENORM) {
        float st[3];
        vn_updated(a.vn_state, a.mb_stats, rows, a.vn_beta, st);
        const VnScalars s = vn_mean_std(st);
        c.vn_mean = s.mean; c.vn_std = s.std;
    }
    return c;
}

// entropy of a categorical row (act.py:160-168)
template <int NOUT = MAX_OUT>
__device__ __forceinline__ float categorical_entropy(const float (&nl)[MAX_OUT], const float (&pr)[MAX_OUT], int n) {
    float ent = 0.f;
#pragma unroll
    for (int j = 0; j < NOUT; ++j) if (j < n) ent -= pr[j] * nl[j];
    return ent;
}

// dL/dlogits of a categorical row from d(loss)/d(logp) `dlp` and the entropy weight `went` (entropy_coef x row
// weight).  Writes the unmasked entries j < n only; the masked-out actions (bits of `masked`) get no gradient.
template <int NOUT = MAX_OUT>
__device__ __forceinline__ void categorical_dlogits(float dlp, float went, int act, int n, unsigned masked,
                                                    const float (&nl)[MAX_OUT], const float (&pr)[MAX_OUT], float ent,
                                                    float (&dl)[MAX_OUT]) {
#pragma unroll
    for (int j = 0; j < NOUT; ++j)
        if (j < n && !((masked >> j) & 1u)) dl[j] = dlp * ((j == act ? 1.f : 0.f) - pr[j]) + went * pr[j] * (nl[j] + ent);
}

// Policy loss of one categorical row (ppo.py:300-319, entropy act.py:160-168): masks the logits in place, writes
// dL/dlogits (entries as categorical_dlogits) and returns the unweighted policy loss and entropy and the ratio.
struct CatRow { float loss, ent, ratio; };
template <int NOUT = MAX_OUT, class Args>
__device__ __forceinline__ CatRow categorical_row(const Args& a, float (&logit)[MAX_OUT], int n, const float* mask_row,
                                                  int act, float old_lp, float adv, float wrow, float (&dl)[MAX_OUT]) {
    float nl[MAX_OUT], pr[MAX_OUT];
    const unsigned masked = masked_log_softmax(logit, n, mask_row, nl, pr);
    const PgTerm pg = pg_term(log_prob_of(nl, n, act), old_lp, adv, a.clip_param, a.flags, a.dual_clip_coeff);
    const float ent = categorical_entropy<NOUT>(nl, pr, n);
    categorical_dlogits<NOUT>(pg.dlogp * wrow, a.entropy_coef * wrow, act, n, masked, nl, pr, ent, dl);
    return CatRow{pg.loss, ent, pg.ratio};
}

// ---- the wide Categorical head (NB = 64): one row's logits x[0..n) in shared memory, owned by one thread -------------------
// The same maths as log_softmax_n / categorical_row, streamed over the row instead of held in per-thread arrays (a 64-entry
// array per thread would spill): a first pass masks (-6e4) and takes the max, a second the sum of exponentials, and every
// later pass recomputes nl[j] = x[j] - lse and p[j] = exp(nl[j] - mx2) / s2 on the fly.  mx2 = max_j (x[j] - lse) is
// mx - lse: rounding is monotone, so the max of the rounded differences is the rounded difference of the max.
struct WideSoftmax {
    float lse, mx2, s2;
    uint64_t masked;   // masked-out actions
    __device__ __forceinline__ float nl(const float* x, int j) const { return x[j] - lse; }
    __device__ __forceinline__ float pr(const float* x, int j) const { return expf(x[j] - lse - mx2) / s2; }
};
__device__ __forceinline__ WideSoftmax wide_log_softmax(float* x, int n, const float* mask_row) {
    WideSoftmax r;
    r.masked = 0;
    if (mask_row) {
        for (int j = 0; j < n; ++j)
            if (mask_row[j] == 0.f) { x[j] = -6e4f; r.masked |= 1ull << j; }
    }
    float mx = x[0];
    for (int j = 1; j < n; ++j) mx = fmaxf(mx, x[j]);
    float s = 0.f;
    for (int j = 0; j < n; ++j) s += expf(x[j] - mx);
    r.lse = mx + logf(s);
    r.mx2 = mx - r.lse;
    float s2 = 0.f;
    for (int j = 0; j < n; ++j) s2 += expf(x[j] - r.lse - r.mx2);
    r.s2 = s2;
    return r;
}
__device__ __forceinline__ float wide_log_prob_of(const WideSoftmax& sm, const float* x, int n, int act) {
    return sm.nl(x, (act >= 0 && act < n) ? act : 0);
}
__device__ __forceinline__ float wide_entropy(const WideSoftmax& sm, const float* x, int n) {
    float ent = 0.f;
    for (int j = 0; j < n; ++j) ent -= sm.pr(x, j) * sm.nl(x, j);
    return ent;
}

// categorical_row of a wide head: masks the row's logits, then overwrites x[0..pad4(n)) with dL/dlogits (0 for the
// masked-out actions and the padding), the K = pad4(n) operand of dn3 = dL . Whf and GH += dL^T n3.
template <class Args>
__device__ __forceinline__ CatRow wide_categorical_row(const Args& a, float* x, int n, const float* mask_row, int act,
                                                       float old_lp, float adv, float wrow) {
    const WideSoftmax sm = wide_log_softmax(x, n, mask_row);
    const PgTerm pg = pg_term(wide_log_prob_of(sm, x, n, act), old_lp, adv, a.clip_param, a.flags, a.dual_clip_coeff);
    const float ent = wide_entropy(sm, x, n);
    const float dlp = pg.dlogp * wrow, went = a.entropy_coef * wrow;
    for (int j = 0; j < n; ++j) {
        const float p = sm.pr(x, j), nl = sm.nl(x, j);
        x[j] = ((sm.masked >> j) & 1ull) ? 0.f : dlp * ((j == act ? 1.f : 0.f) - p) + went * p * (nl + ent);
    }
    for (int j = n; j < pad4(n); ++j) x[j] = 0.f;
    return CatRow{pg.loss, ent, pg.ratio};
}

// DiagGaussian head (distributions.py:34-47, 75-98): Normal.log_prob of one dimension at distance diff = x - mean,
// -diff^2 / (2 var) - log(std) - log(sqrt(2 pi)), and Normal.entropy of one dimension, 0.5 + 0.5 log(2 pi) + log(std)
__device__ __forceinline__ float gaussian_log_prob(float diff, float std, float logstd) {
    return -(diff * diff) / (2.0f * (std * std)) - logstd - 0.9189385332046727f;
}
__device__ __forceinline__ float gaussian_entropy(float logstd) { return 1.4189385332046727f + logstd; }

// Policy loss of one DiagGaussian row (act.py:150-158; ppo.py:307-319: a ratio per dimension, the surrogate summed over
// the dimensions).  act / old_lp are the row's n entries; wrow weights the loss, went the entropy.  Adds each
// dimension's weighted loss, weighted entropy and ratio / n to loss / ent / ratio in dimension order, so the caller's
// running sums round as one loop over its rows' dimensions; writes dL/dmean to dl[j] and adds dL/dlogstd to dls[j].
template <class Args>
__device__ __forceinline__ void gaussian_row(const Args& a, const float (&mean)[MAX_OUT], int n, const float* logstd,
                                             const float* act, const float* old_lp, float adv, float wrow, float went,
                                             float (&dl)[MAX_OUT], float (&dls)[MAX_OUT], float& loss, float& ent,
                                             float& ratio) {
#pragma unroll
    for (int j = 0; j < MAX_OUT; ++j) {
        if (j < n) {
            const float ls = logstd[j], std = expf(ls), var = std * std, diff = act[j] - mean[j];
            const PgTerm pg = pg_term(gaussian_log_prob(diff, std, ls), old_lp[j], adv, a.clip_param, a.flags, a.dual_clip_coeff);
            loss += pg.loss * wrow;
            ent += gaussian_entropy(ls) * went;
            ratio += pg.ratio / (float)n;
            const float dlp = pg.dlogp * wrow;
            dl[j] = dlp * diff / var;
            dls[j] += dlp * (diff * diff / var - 1.0f) - a.entropy_coef * went;
        }
    }
}

__device__ __forceinline__ float huber(float e, float d) { return fabsf(e) <= d ? 0.5f * e * e : d * (fabsf(e) - 0.5f * d); }
__device__ __forceinline__ float huber_grad(float e, float d) { return fabsf(e) <= d ? e : (e > 0.f ? d : -d); }

// Clipped value loss of one row (ppo.py:344-386 cal_value_loss): returns the loss and d(loss)/d(value).
struct ValueTerm { float loss, dv; };
__device__ __forceinline__ ValueTerm value_term(float v, float vp, float target, float clip, float delta, int flags) {
    const float diff = v - vp;
    const float clipped = vp + fminf(fmaxf(diff, -clip), clip);
    const float e_c = target - clipped, e_o = target - v;
    const bool hub = flags & ORL_PPO_HUBER;
    const float l_c = hub ? huber(e_c, delta) : 0.5f * e_c * e_c;
    const float l_o = hub ? huber(e_o, delta) : 0.5f * e_o * e_o;
    const float gc = hub ? huber_grad(e_c, delta) : e_c;
    const float go = hub ? huber_grad(e_o, delta) : e_o;
    ValueTerm o; o.loss = l_o; o.dv = -go;
    if (flags & ORL_PPO_CLIP_VALUE) {
        const bool inrange = diff >= -clip && diff <= clip;
        const float dc = inrange ? -gc : 0.f;
        if (l_o > l_c) { o.loss = l_o; o.dv = -go; }
        else if (l_c > l_o) { o.loss = l_c; o.dv = dc; }
        else { o.loss = l_o; o.dv = 0.5f * (-go) + 0.5f * dc; }
    }
    return o;
}

}  // namespace orl
