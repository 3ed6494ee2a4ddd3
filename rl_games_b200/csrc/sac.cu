// Soft Actor-Critic (sac_agent.py): device-resident replay buffer, squashed-Gaussian head, twin-critic TD loss, actor / temperature
// loss with the backward through the squash, and the Polyak target update.  The MLP GEMMs are b200rl_linear_* (fp32) or
// b200rl_linear_*_tc (mixed precision); the optimiser steps are b200rl_adam_step_f32.  Every random draw is Philox keyed by
// (seed, call site) with the row in the low counter word and a device-resident u64 counter in the high word, so an update reads no
// host state and can be replayed from a CUDA graph; the caller bumps the counter (b200rl_bump_u64) once per update / env step.
#include "common.cuh"

namespace {

constexpr int SAC_THREADS = 256;
constexpr int SAC_RED_THREADS = 1024;

__device__ __forceinline__ uint64_t sac_hi(const uint64_t* ctr, int site) {
    return ((ctr ? *ctr : 0ull) << 8) | (uint64_t)site;
}
__device__ __forceinline__ uint64_t sac_key(uint64_t seed, int site) {
    return seed ^ (0xA0761D6478BD642Full * (uint64_t)(site + 1));
}
// j-th standard normal of row r at this call site (four normals per Philox block, j = 4q + k)
__device__ __forceinline__ float sac_normal(uint64_t seed, const uint64_t* ctr, int site, int64_t r, int j) {
    const Philox4 p = philox4x32_10((uint64_t)r | ((uint64_t)(j >> 2) << 40), sac_hi(ctr, site), sac_key(seed, site));
    float n0, n1, n2, n3;
    box_muller(p.x, p.y, n0, n1);
    box_muller(p.z, p.w, n2, n3);
    const int k = j & 3;
    return k == 0 ? n0 : k == 1 ? n1 : k == 2 ? n2 : n3;
}
// uniform in [0, 1) (torch.rand's range)
__device__ __forceinline__ float sac_uniform(uint64_t seed, const uint64_t* ctr, int site, int64_t r, int j) {
    const Philox4 p = philox4x32_10((uint64_t)r | ((uint64_t)(j >> 2) << 40), sac_hi(ctr, site), sac_key(seed, site));
    const int k = j & 3;
    const uint32_t u = k == 0 ? p.x : k == 1 ? p.y : k == 2 ? p.z : p.w;
    return (float)(u >> 8) * (1.0f / 16777216.0f);
}

// ---------------------------------------------------------------------------------------------------------------- replay insert
// Phase 1 (one CTA): which rows of this env step are written and where, the ring head / fill, and the episode accounting of
// _store_transitions.  next_step autoreset: a row whose previous step ended an episode is the reset step's filler and is skipped;
// live rows keep their order (block-wide exclusive prefix count), which is the reference's nonzero + index_select.
__global__ void __launch_bounds__(SAC_RED_THREADS) replay_plan_kernel(
        const float* __restrict__ reward, const uint8_t* __restrict__ dones, const uint8_t* __restrict__ time_outs, int value_bootstrap,
        int next_step, uint8_t* __restrict__ prev_dones, int N, int capacity, int64_t* __restrict__ rb_state, int* __restrict__ slot,
        uint8_t* __restrict__ term_out, uint8_t* __restrict__ trunc_out, float* __restrict__ ep_state, double* __restrict__ meter,
        int games_to_track) {
    __shared__ int warp_tot[32];
    __shared__ int base_s;
    __shared__ double sm[64];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    const int64_t head0 = rb_state[0];
    if (tid == 0) base_s = 0;
    double rsum = 0.0, lsum = 0.0;
    int ndone = 0;
    __syncthreads();
    for (int c0 = 0; c0 < N; c0 += blockDim.x) {
        const int r = c0 + tid;
        const bool in = r < N;
        const bool d = in && dones[r] != 0;
        const bool live = in && (!next_step || prev_dones[r] == 0);
        // exclusive prefix count of live rows (ballot within the warp, then across warps)
        const unsigned b = __ballot_sync(0xffffffffu, live);
        if (lane == 0) warp_tot[warp] = __popc(b);
        __syncthreads();
        int before = 0, chunk_tot = 0;
        for (int w = 0; w < nw; ++w) {
            const int t = warp_tot[w];
            before += w < warp ? t : 0;
            chunk_tot += t;
        }
        const int rank = base_s + before + __popc(b & ((1u << lane) - 1u));
        if (in) {
            const bool tr = value_bootstrap && time_outs && time_outs[r] != 0;
            term_out[r] = (uint8_t)(d && !tr);
            trunc_out[r] = (uint8_t)tr;
            slot[r] = live ? (int)((head0 + rank) % capacity) : -1;
            // episode accounting: current_rewards / current_lengths (live rows only under next_step), meters on done live rows
            float cr = ep_state[r], cl = ep_state[N + r];
            if (live) { cr += reward[r]; cl += 1.0f; }
            if (d && live) { rsum += (double)cr; lsum += (double)cl; ++ndone; }
            if (d) { cr = 0.0f; cl = 0.0f; }
            ep_state[r] = cr; ep_state[N + r] = cl;
        }
        __syncthreads();
        if (tid == 0) base_s += chunk_tot;
        __syncthreads();
        if (in && next_step) prev_dones[r] = (uint8_t)d;
    }
    if (!next_step)
        for (int r = tid; r < N; r += blockDim.x) prev_dones[r] = dones[r] != 0;
    double v[2] = {rsum, lsum};
    block_sum_d<2>(v, sm);
    double nd[1] = {(double)ndone};
    block_sum_d<1>(nd, sm);
    if (tid == 0) {
        const int n = base_s;
        rb_state[0] = (head0 + n) % capacity;
        rb_state[1] = min((int64_t)capacity, rb_state[1] + n);
        // torch_ext.AverageMeter.update on the done rows' accumulators
        const int k = (int)nd[0];
        if (k > 0) {
            const int size = min(k, games_to_track);
            const int old = (int)min((double)(games_to_track - size), meter[2]);
            const double tot = (double)(old + size);
            meter[0] = (meter[0] * old + (v[0] / k) * size) / tot;
            meter[1] = (meter[1] * old + (v[1] / k) * size) / tot;
            meter[2] = tot;
        }
    }
}

// Phase 2 (grid): copy each written row into its slot.  same_step autoreset: a truncated row's next_obs is the final observation
// (final_obs when the env reports it, else the s_t proxy obs).
__global__ void replay_copy_kernel(const float* __restrict__ obs, const float* __restrict__ action, const float* __restrict__ reward,
                                   const float* __restrict__ next_obs, const float* __restrict__ final_obs, int next_step, int N, int D, int A,
                                   const int* __restrict__ slot, const uint8_t* __restrict__ term, const uint8_t* __restrict__ trunc,
                                   float* __restrict__ rb_obs, float* __restrict__ rb_act, float* __restrict__ rb_rew,
                                   float* __restrict__ rb_next, uint8_t* __restrict__ rb_term, uint8_t* __restrict__ rb_trunc) {
    const int W = 2 * D + A + 1;
    const int64_t total = (int64_t)N * W;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int r = (int)(i / W), c = (int)(i - (int64_t)r * W);
        const int s = slot[r];
        if (s < 0) continue;
        if (c < D) {
            rb_obs[(int64_t)s * D + c] = obs[(int64_t)r * D + c];
        } else if (c < 2 * D) {
            const int j = c - D;
            const bool sub = !next_step && trunc[r];
            rb_next[(int64_t)s * D + j] = sub ? (final_obs ? final_obs[(int64_t)r * D + j] : obs[(int64_t)r * D + j]) : next_obs[(int64_t)r * D + j];
        } else if (c < 2 * D + A) {
            const int j = c - 2 * D;
            rb_act[(int64_t)s * A + j] = action[(int64_t)r * A + j];
        } else {
            rb_rew[s] = reward[r];
            rb_term[s] = term[r];
            rb_trunc[s] = trunc[r];
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------- replay sample
// idx[b] uniform over the current fill (or from a tape); gathers normalised obs into x_cur[:, :D] and x_pi[:, :D], the stored action
// into x_cur[:, D:D+A], normalised next_obs into x_next[:, :D], reward and not_done.  Rows of x_* are D + A wide.
__global__ void replay_sample_kernel(const float* __restrict__ rb_obs, const float* __restrict__ rb_act, const float* __restrict__ rb_rew,
                                     const float* __restrict__ rb_next, const uint8_t* __restrict__ rb_term, const int64_t* __restrict__ rb_state,
                                     int capacity, int D, int A, int B, const int64_t* __restrict__ idx_tape, uint64_t seed,
                                     const uint64_t* __restrict__ ctr, const float* __restrict__ norm_mean, const float* __restrict__ norm_std,
                                     float* __restrict__ x_cur, float* __restrict__ x_pi, float* __restrict__ x_next, float* __restrict__ reward,
                                     float* __restrict__ not_done, int64_t* __restrict__ idx_out) {
    const int W = 2 * D + A + 1, ld = D + A;
    const int64_t total = (int64_t)B * W;
    const int64_t fill = max((int64_t)1, rb_state[1]);
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int b = (int)(i / W), c = (int)(i - (int64_t)b * W);
        int64_t k;
        if (idx_tape) {
            k = idx_tape[b];
        } else {
            const Philox4 p = philox4x32_10((uint64_t)b, sac_hi(ctr, 2), sac_key(seed, 2));
            const uint64_t u = ((uint64_t)p.x << 32) | p.y;
            k = (int64_t)(((unsigned __int128)u * (unsigned __int128)(uint64_t)fill) >> 64);
        }
        if (c < D) {
            float x = rb_obs[k * D + c];
            if (norm_mean) x = fminf(fmaxf(__fdiv_rn(x - norm_mean[c], norm_std[c]), -5.0f), 5.0f);
            x_cur[(int64_t)b * ld + c] = x;
            x_pi[(int64_t)b * ld + c] = x;
        } else if (c < 2 * D) {
            const int j = c - D;
            float x = rb_next[k * D + j];
            if (norm_mean) x = fminf(fmaxf(__fdiv_rn(x - norm_mean[j], norm_std[j]), -5.0f), 5.0f);
            x_next[(int64_t)b * ld + j] = x;
        } else if (c < 2 * D + A) {
            const int j = c - 2 * D;
            x_cur[(int64_t)b * ld + D + j] = rb_act[k * A + j];
        } else {
            reward[b] = rb_rew[k];
            not_done[b] = rb_term[k] ? 0.0f : 1.0f;
            if (idx_out) idx_out[b] = k;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------- squashed Gaussian
struct SquashArgs {
    const float* head; int A; float ls_lo, ls_hi; const float* noise; uint64_t seed; const uint64_t* ctr; int site;
    const float* scale; const float* bias; const float* low; const float* high; float log_scale_sum;
    float* dst; int64_t dst_ld; float* eps_out; float* logp;
};

__device__ __forceinline__ void bounded_logstd(float raw, float lo, float hi, float& t, float& ls) {
    t = tanhf(raw);
    ls = lo + 0.5f * (hi - lo) * (t + 1.0f);
}

// DiagGaussianActor.forward + SquashedNormal.rsample + _env_log_prob + rescale_actions, one thread per row
__global__ void squash_fwd_kernel(SquashArgs a, int M) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= M) return;
    const int A = a.A;
    const float* h = a.head + (int64_t)r * 2 * A;
    float lp = 0.0f;
    for (int j = 0; j < A; ++j) {
        const float mu = h[j];
        float t, ls;
        bounded_logstd(h[A + j], a.ls_lo, a.ls_hi, t, ls);
        const float sd = expf(ls);
        const float e = a.noise ? a.noise[(int64_t)r * A + j] : sac_normal(a.seed, a.ctr, a.site, r, j);
        const float x = mu + e * sd;
        const float y = tanhf(x);
        if (a.logp) {
            const float d = x - mu;
            const float nlp = -(d * d) / (2.0f * (sd * sd)) - logf(sd) - 0.91893853320467274f;      // log(sqrt(2 pi))
            const float sp = (-2.0f * x) > 20.0f ? -2.0f * x : log1pf(expf(-2.0f * x));           // softplus(-2x), torch threshold 20
            const float jac = 2.0f * (0.69314718055994531f - x - sp);
            lp += (0.0f - jac) + nlp;
        }
        if (a.eps_out) a.eps_out[(int64_t)r * A + j] = e;
        if (a.dst) {
            const float v = fminf(fmaxf(y * a.scale[j] + a.bias[j], a.low[j]), a.high[j]);
            a.dst[(int64_t)r * a.dst_ld + j] = v;
        }
    }
    if (a.logp) a.logp[r] = lp - a.log_scale_sum;
}

// warmup exploration (play_steps' random_exploration): action = low + (high - low) * U[0, 1)
__global__ void uniform_actions_kernel(const float* __restrict__ low, const float* __restrict__ high, const float* __restrict__ u_tape,
                                       uint64_t seed, const uint64_t* __restrict__ ctr, float* __restrict__ out, int N, int A) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= (int64_t)N * A) return;
    const int r = (int)(i / A), j = (int)(i - (int64_t)r * A);
    const float u = u_tape ? u_tape[i] : sac_uniform(seed, ctr, 4, r, j);
    out[i] = __fadd_rn(low[j], __fmul_rn(__fsub_rn(high[j], low[j]), u));     // torch's rounding: no fused multiply-add
}

// ---------------------------------------------------------------------------------------------------------------- critic loss
// target = r + not_done * gamma * (min(Q1t, Q2t) - alpha * logp'),  L = 0.5 (mse(Q1, target) + mse(Q2, target)).
// stats[0..2] = critic_loss, critic1_loss, critic2_loss; dq1 / dq2 = dL/dQ.
__global__ void __launch_bounds__(SAC_RED_THREADS) critic_loss_kernel(const float* __restrict__ q1, const float* __restrict__ q2,
                                                                      const float* __restrict__ q1t, const float* __restrict__ q2t,
                                                                      const float* __restrict__ logp_next, const float* __restrict__ reward,
                                                                      const float* __restrict__ not_done, const float* __restrict__ log_alpha,
                                                                      float gamma, int B, float* __restrict__ dq1, float* __restrict__ dq2,
                                                                      float* __restrict__ stats) {
    __shared__ double sm[64];
    const float alpha = expf(*log_alpha);
    const float inv = 1.0f / (float)B;
    double acc[2] = {0.0, 0.0};
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        const float tv = fminf(q1t[b], q2t[b]) - alpha * logp_next[b];
        const float tq = reward[b] + not_done[b] * gamma * tv;
        const float e1 = q1[b] - tq, e2 = q2[b] - tq;
        acc[0] += (double)e1 * e1;
        acc[1] += (double)e2 * e2;
        dq1[b] = e1 * inv;          // d(0.5 * mean(e^2)) / dq = e / B
        dq2[b] = e2 * inv;
    }
    block_sum_d<2>(acc, sm);
    if (threadIdx.x == 0) {
        const float l1 = (float)(acc[0] / B), l2 = (float)(acc[1] / B);
        stats[0] = 0.5f * (l1 + l2);
        stats[1] = l1;
        stats[2] = l2;
    }
}

// ---------------------------------------------------------------------------------------------------------------- actor / alpha loss
// L_actor = mean(max(alpha, min_alpha) * logp - min(Q1, Q2)); torch.min(a, b)'s backward splits a tie's gradient in halves.
// L_alpha = mean(alpha * (-logp - target_entropy)) (logp detached) -> d log_alpha = alpha * mean(-logp - target_entropy).
// stats[3] = actor_loss, stats[4] = entropy (-mean logp), stats[6] = alpha_loss; dq1 / dq2 = dL_actor/dQ.
__global__ void __launch_bounds__(SAC_RED_THREADS) actor_loss_kernel(const float* __restrict__ q1, const float* __restrict__ q2,
                                                                     const float* __restrict__ logp, const float* __restrict__ log_alpha,
                                                                     float min_alpha, float target_entropy, int learnable, int B,
                                                                     float* __restrict__ dq1, float* __restrict__ dq2,
                                                                     float* __restrict__ d_log_alpha, float* __restrict__ stats) {
    __shared__ double sm[96];
    const float alpha = expf(*log_alpha);
    const float ac = fmaxf(alpha, min_alpha);
    const float inv = 1.0f / (float)B;
    double acc[3] = {0.0, 0.0, 0.0};
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        const float a = q1[b], c = q2[b], lp = logp[b];
        acc[0] += (double)(ac * lp - fminf(a, c));
        acc[1] += (double)lp;
        acc[2] += (double)(-lp - target_entropy);
        const float g = -inv;
        dq1[b] = a < c ? g : a == c ? 0.5f * g : 0.0f;
        dq2[b] = c < a ? g : a == c ? 0.5f * g : 0.0f;
    }
    block_sum_d<3>(acc, sm);
    if (threadIdx.x == 0) {
        stats[3] = (float)(acc[0] / B);
        stats[4] = (float)(-acc[1] / B);
        const float m = (float)(acc[2] / B);
        stats[6] = learnable ? alpha * m : 0.0f;
        if (learnable && d_log_alpha) d_log_alpha[0] = alpha * m;
    }
}

// backward of squash_fwd for the actor pass: dL/d(action) = dxa1 + dxa2 (the two critics' input-gradient action columns), plus
// max(alpha, min_alpha) / B * dlogp/d(.) ; writes d_head [M, 2A] = dL/d(mu, raw log_std)
__global__ void squash_bwd_kernel(const float* __restrict__ head, const float* __restrict__ eps, int A, float ls_lo, float ls_hi,
                                  const float* __restrict__ scale, const float* __restrict__ bias, const float* __restrict__ low,
                                  const float* __restrict__ high, const float* __restrict__ dxa1, const float* __restrict__ dxa2, int64_t dx_ld,
                                  const float* __restrict__ log_alpha, float min_alpha, int M, float* __restrict__ d_head) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= M) return;
    const float g_lp = fmaxf(expf(*log_alpha), min_alpha) / (float)M;
    const float* h = head + (int64_t)r * 2 * A;
    for (int j = 0; j < A; ++j) {
        const float mu = h[j];
        float t, ls;
        bounded_logstd(h[A + j], ls_lo, ls_hi, t, ls);
        const float sd = expf(ls);
        const float e = eps[(int64_t)r * A + j];
        const float x = mu + e * sd;
        const float y = tanhf(x);
        const float pre = y * scale[j] + bias[j];
        const float da_env = dxa1[(int64_t)r * dx_ld + j] + dxa2[(int64_t)r * dx_ld + j];
        const float da = (pre >= low[j] && pre <= high[j]) ? da_env * scale[j] : 0.0f;     // clamp's backward
        const float d = x - mu;
        const float var = sd * sd;
        // logp = sum_j [ -d^2 / (2 var) - log sd - log sqrt(2 pi) - 2 (log 2 - x - softplus(-2x)) ]
        const float dx = da * (1.0f - y * y) + g_lp * (-d / var + 2.0f * y);
        const float dmu = dx + g_lp * (d / var);
        const float dsd = dx * e + g_lp * ((d * d) / (var * sd) - 1.0f / sd);
        const float dls = dsd * sd;
        d_head[(int64_t)r * 2 * A + j] = dmu;
        d_head[(int64_t)r * 2 * A + A + j] = dls * 0.5f * (ls_hi - ls_lo) * (1.0f - t * t);
    }
}

// ---------------------------------------------------------------------------------------------------------------- Polyak
// target <- target.lerp(src, tau), torch's lerp formula (weight < 0.5: self + w (end - self), else end - (end - self)(1 - w))
__global__ void polyak_kernel(float* __restrict__ target, const float* __restrict__ src, int n, float tau,
                              const float* __restrict__ log_alpha, float* __restrict__ alpha_stat) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const float t = target[i], s = src[i], d = s - t;
        target[i] = tau < 0.5f ? t + tau * d : s - d * (1.0f - tau);
    }
    if (i == 0 && alpha_stat) alpha_stat[0] = expf(*log_alpha);
}

inline int blocks_for(int64_t n, int t) {
    int64_t b = (n + t - 1) / t;
    if (b > 132 * 16) b = 132 * 16;
    return (int)(b < 1 ? 1 : b);
}

}  // namespace

B200RL_EXPORT int b200rl_sac_replay_insert_f32(const float* obs, const float* action, const float* reward, const float* next_obs,
                                               const float* final_obs, const uint8_t* dones, const uint8_t* time_outs, int value_bootstrap,
                                               int next_step, uint8_t* prev_dones, int N, int D, int A, int capacity, float* rb_obs,
                                               float* rb_act, float* rb_rew, float* rb_next, uint8_t* rb_term, uint8_t* rb_trunc,
                                               int64_t* rb_state, int* slot, uint8_t* term_scratch, uint8_t* trunc_scratch,
                                               float* ep_state, double* meter, int games_to_track, void* stream) {
    if (!obs || !action || !reward || !next_obs || !dones || !prev_dones || !rb_obs || !rb_act || !rb_rew || !rb_next || !rb_term ||
        !rb_trunc || !rb_state || !slot || !term_scratch || !trunc_scratch || !ep_state || !meter)
        return B200RL_EINVAL;
    if (N <= 0 || D <= 0 || A <= 0 || capacity < N || games_to_track <= 0) return B200RL_EINVAL;
    cudaStream_t s = as_stream(stream);
    replay_plan_kernel<<<1, SAC_RED_THREADS, 0, s>>>(reward, dones, time_outs, value_bootstrap, next_step, prev_dones, N, capacity, rb_state,
                                                     slot, term_scratch, trunc_scratch, ep_state, meter, games_to_track);
    B200RL_LAUNCH_CHECK();
    replay_copy_kernel<<<blocks_for((int64_t)N * (2 * D + A + 1), SAC_THREADS), SAC_THREADS, 0, s>>>(
        obs, action, reward, next_obs, final_obs, next_step, N, D, A, slot, term_scratch, trunc_scratch, rb_obs, rb_act, rb_rew, rb_next,
        rb_term, rb_trunc);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_sac_replay_sample_f32(const float* rb_obs, const float* rb_act, const float* rb_rew, const float* rb_next,
                                               const uint8_t* rb_term, const int64_t* rb_state, int capacity, int D, int A, int B,
                                               const int64_t* idx_tape, uint64_t seed, const uint64_t* rng_ctr, const float* norm_mean,
                                               const float* norm_std, float* x_cur, float* x_pi, float* x_next, float* reward,
                                               float* not_done, int64_t* idx_out, void* stream) {
    if (!rb_obs || !rb_act || !rb_rew || !rb_next || !rb_term || !rb_state || !x_cur || !x_pi || !x_next || !reward || !not_done)
        return B200RL_EINVAL;
    if (capacity <= 0 || D <= 0 || A <= 0 || B <= 0 || (!idx_tape && !rng_ctr) || ((norm_mean != nullptr) != (norm_std != nullptr)))
        return B200RL_EINVAL;
    replay_sample_kernel<<<blocks_for((int64_t)B * (2 * D + A + 1), SAC_THREADS), SAC_THREADS, 0, as_stream(stream)>>>(
        rb_obs, rb_act, rb_rew, rb_next, rb_term, rb_state, capacity, D, A, B, idx_tape, seed, rng_ctr, norm_mean, norm_std, x_cur, x_pi,
        x_next, reward, not_done, idx_out);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_sac_squash_fwd_f32(const float* head, int M, int A, float log_std_min, float log_std_max, const float* noise,
                                            uint64_t seed, const uint64_t* rng_ctr, int rng_site, const float* act_scale,
                                            const float* act_bias, const float* act_low, const float* act_high, float log_action_scale_sum,
                                            float* dst, int64_t dst_ld, float* eps_out, float* logp, void* stream) {
    if (!head || M <= 0 || A <= 0 || (!noise && !rng_ctr) || rng_site < 0 || rng_site > 255) return B200RL_EINVAL;
    if (dst && (!act_scale || !act_bias || !act_low || !act_high || dst_ld < A)) return B200RL_EINVAL;
    SquashArgs a{head, A, log_std_min, log_std_max, noise, seed, rng_ctr, rng_site, act_scale, act_bias, act_low, act_high,
                 log_action_scale_sum, dst, dst_ld, eps_out, logp};
    squash_fwd_kernel<<<(M + 127) / 128, 128, 0, as_stream(stream)>>>(a, M);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_sac_uniform_actions_f32(const float* act_low, const float* act_high, const float* u_tape, uint64_t seed,
                                                 const uint64_t* rng_ctr, float* out, int N, int A, void* stream) {
    if (!act_low || !act_high || !out || N <= 0 || A <= 0 || (!u_tape && !rng_ctr)) return B200RL_EINVAL;
    const int64_t n = (int64_t)N * A;
    uniform_actions_kernel<<<(int)((n + SAC_THREADS - 1) / SAC_THREADS), SAC_THREADS, 0, as_stream(stream)>>>(act_low, act_high, u_tape,
                                                                                                              seed, rng_ctr, out, N, A);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_sac_critic_loss_f32(const float* q1, const float* q2, const float* q1t, const float* q2t, const float* logp_next,
                                             const float* reward, const float* not_done, const float* log_alpha, float gamma, int B,
                                             float* dq1, float* dq2, float* stats, void* stream) {
    if (!q1 || !q2 || !q1t || !q2t || !logp_next || !reward || !not_done || !log_alpha || !dq1 || !dq2 || !stats || B <= 0)
        return B200RL_EINVAL;
    critic_loss_kernel<<<1, SAC_RED_THREADS, 0, as_stream(stream)>>>(q1, q2, q1t, q2t, logp_next, reward, not_done, log_alpha, gamma, B, dq1,
                                                                     dq2, stats);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_sac_actor_loss_f32(const float* q1, const float* q2, const float* logp, const float* log_alpha, float min_alpha,
                                            float target_entropy, int learnable_temperature, int B, float* dq1, float* dq2,
                                            float* d_log_alpha, float* stats, void* stream) {
    if (!q1 || !q2 || !logp || !log_alpha || !dq1 || !dq2 || !stats || B <= 0 || (learnable_temperature && !d_log_alpha))
        return B200RL_EINVAL;
    actor_loss_kernel<<<1, SAC_RED_THREADS, 0, as_stream(stream)>>>(q1, q2, logp, log_alpha, min_alpha, target_entropy, learnable_temperature,
                                                                    B, dq1, dq2, d_log_alpha, stats);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_sac_squash_bwd_f32(const float* head, const float* eps, int M, int A, float log_std_min, float log_std_max,
                                            const float* act_scale, const float* act_bias, const float* act_low, const float* act_high,
                                            const float* dxa1, const float* dxa2, int64_t dx_ld, const float* log_alpha, float min_alpha,
                                            float* d_head, void* stream) {
    if (!head || !eps || !act_scale || !act_bias || !act_low || !act_high || !dxa1 || !dxa2 || !log_alpha || !d_head || M <= 0 || A <= 0 ||
        dx_ld < A)
        return B200RL_EINVAL;
    squash_bwd_kernel<<<(M + 127) / 128, 128, 0, as_stream(stream)>>>(head, eps, A, log_std_min, log_std_max, act_scale, act_bias, act_low,
                                                                      act_high, dxa1, dxa2, dx_ld, log_alpha, min_alpha, M, d_head);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_sac_polyak_f32(float* target, const float* src, int n, float tau, const float* log_alpha, float* alpha_stat,
                                        void* stream) {
    if (!target || !src || n <= 0 || (alpha_stat && !log_alpha)) return B200RL_EINVAL;
    polyak_kernel<<<(n + SAC_THREADS - 1) / SAC_THREADS, SAC_THREADS, 0, as_stream(stream)>>>(target, src, n, tau, log_alpha, alpha_stat);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}
