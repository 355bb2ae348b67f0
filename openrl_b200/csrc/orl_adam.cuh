// The optimiser step of every PPO update (ppo_apply_kernel in orl_ppo.cu, rnn_apply_kernel in orl_rnn.cu,
// share_apply_kernel in orl_share.cu), run by one CTA per parameter vector: clip_grad_norm_ (the block L2 norm and the
// clip factor), torch.optim.Adam (ppo.py:120-158), and the train_info sums with the ValueNorm commit.
#pragma once
#include "orl_loss.cuh"

namespace orl {

// L2 norm over the CTA of the per-thread sums of squares `sq` (warp sums, then shared memory); valid in every thread
__device__ __forceinline__ float block_l2_norm(float sq) {
    __shared__ float red[32];
    __shared__ float s_norm;
    const int tid = threadIdx.x;
    const float s = warp_sum(sq);
    if ((tid & 31) == 0) red[tid >> 5] = s;
    __syncthreads();
    if (tid < 32) {
        float v = (tid < (int)(blockDim.x >> 5)) ? red[tid] : 0.f;
        v = warp_sum(v);
        if (tid == 0) s_norm = sqrtf(v);
    }
    __syncthreads();
    return s_norm;
}

// clip_grad_norm_(max_grad_norm) factor of a gradient whose L2 norm is `norm`; 1 without ORL_PPO_MAX_GRAD_NORM
template <class Args>
__device__ __forceinline__ float clip_factor(const Args& a, float norm) {
    return (a.flags & ORL_PPO_MAX_GRAD_NORM) ? fminf(a.max_grad_norm / (norm + 1e-6f), 1.0f) : 1.f;
}

// One Adam step on grads * clip with lr = lrs[slot]; advances adam_steps[slot].  Every thread of the CTA calls it.  Its
// barrier also orders every earlier read of `params` by the CTA before the first update of them.
template <class Args>
__device__ __forceinline__ void adam_step(const Args& a, int slot, float* params, float* am, float* av,
                                          const float* grads, int total, float clip) {
    const int tid = threadIdx.x;
    const int step = a.adam_steps[slot] + 1;
    __shared__ float s_adam[2];
    if (tid == (int)blockDim.x - 1) {   // the two double-precision pow() once per CTA (f64 is slow here), not once per thread
        const double bc1 = 1.0 - pow((double)a.adam_beta1, (double)step);
        const double bc2 = 1.0 - pow((double)a.adam_beta2, (double)step);
        s_adam[0] = (float)((double)a.lrs[slot] / bc1);
        s_adam[1] = (float)sqrt(bc2);
    }
    __syncthreads();
    const float step_size = s_adam[0], bc2_sqrt = s_adam[1];
    for (int i = tid; i < total; i += blockDim.x) {
        float g = grads[i] * clip;
        const float pv = params[i];
        if (a.weight_decay != 0.f) g = fmaf(a.weight_decay, pv, g);
        const float m = am[i] + (g - am[i]) * (1.f - a.adam_beta1);                  // exp_avg.lerp_(grad, 1-beta1)
        const float v = fmaf(av[i], a.adam_beta2, (g * g) * (1.f - a.adam_beta2));  // mul_(beta2).addcmul_(g,g,1-beta2)
        am[i] = m; av[i] = v;
        params[i] = pv - step_size * (m / (sqrtf(v) / bc2_sqrt + a.adam_eps));
    }
    if (tid == 0) a.adam_steps[slot] = step;
}

// train_info += {policy_loss, dist_entropy, actor_grad_norm, ratio mean} (slots 2-5) from the minibatch's loss sums
// {policy, entropy, ratio}.  One thread.
template <class Args>
__device__ __forceinline__ void add_policy_info(const Args& a, const float* loss, float norm) {
    a.train_info[2] += loss[0];
    a.train_info[3] += loss[1];
    a.train_info[4] += norm;
    a.train_info[5] += loss[2] / (float)loss_rows(a);
}

// train_info += {value_loss, critic_grad_norm} (slots 0-1) and, with ORL_PPO_VALUENORM, commits the minibatch's
// ValueNorm update.  One thread.
template <class Args>
__device__ __forceinline__ void add_value_info(const Args& a, float value_loss, float norm) {
    a.train_info[0] += value_loss;
    a.train_info[1] += norm;
    if (a.flags & ORL_PPO_VALUENORM) {
        float st[3];
        vn_updated(a.vn_state, a.mb_stats, loss_rows(a), a.vn_beta, st);
        a.vn_state[0] = st[0]; a.vn_state[1] = st[1]; a.vn_state[2] = st[2];
    }
}

}  // namespace orl
