// Categorical (discrete-action) policy head for PPO -- SURVEY.md 8a row a15 (a2c_discrete.py:92-209, models.py:95-125,
// common/extensions/distributions.py:23-44).
//
// Parity tests: tests/test_discrete_gpu.py (through the C ABI, against oracle/ppo_discrete_oracle.py, which is pinned to the real
// reference by golden vectors).
//
// Narrow kernels: one thread per row, for layouts of at most CAT_MAXH heads of at most CAT_MAXK actions.  Wide kernels (second half
// of this file): one CTA per row and one warp per head, for every other layout.  Both are HBM/latency bound, no tensor-core work.
#include <math.h>
#include "common.cuh"

namespace {

constexpr int CAT_MAXK = 64;

struct CatLossDev { float e_clip, critic_coef, entropy_coef; int clip_value, smooth, ppo; };

// ---- per-row arithmetic: __host__ __device__ so that the SAME code is exercised on the CPU by the host test entry points at the
//      end of this file (tests/test_discrete_rows_cpu.py) -- the kernels below only add indexing and the block reduction ----------

// masked log-softmax pieces of one row: legal-max m, lse = m + log(sum exp(z - m)); masked logits count as -1e8 (distributions.py:29)
__host__ __device__ inline void cat_lse(const float* z, const uint8_t* mask, int K, float& lse) {
    float m = -3.0e38f;
    for (int k = 0; k < K; ++k) {
        const float v = (mask && !mask[k]) ? -1e8f : z[k];
        m = fmaxf(m, v);
    }
    float s = 0.f;
    for (int k = 0; k < K; ++k) {
        const float v = (mask && !mask[k]) ? -1e8f : z[k];
        s += expf(v - m);
    }
    lse = m + logf(s);
}

// one categorical per head (a single Discrete(K) space is one head; a Tuple space = ModelA2CMultiDiscrete, models.py:128-206):
// logits / action masks of the heads are concatenated along the row, neglogp and entropy are sums over the heads
constexpr int CAT_MAXH = 8;
struct CatHeads { int n; int size[CAT_MAXH]; int off[CAT_MAXH]; };

// action_j = #{k : cdf_k <= u_j}, clamped to the last action of non-zero probability (oracle.sample_inverse_cdf); returns sum_j neglogp_j
__host__ __device__ inline float cat_sample_row(const float* z, const uint8_t* mk, const CatHeads& hd, const float* u, int64_t u_stride,
                                                int64_t* actions) {
    float nlp = 0.f;
    for (int j = 0; j < hd.n; ++j) {
        const float* zj = z + hd.off[j];
        const uint8_t* mj = mk ? mk + hd.off[j] : nullptr;
        const int K = hd.size[j];
        float lse;
        cat_lse(zj, mj, K, lse);
        const float uj = u[(int64_t)j * u_stride];
        float cdf = 0.f;
        int count = 0, last = 0;
        for (int k = 0; k < K; ++k) {
            const float v = (mj && !mj[k]) ? -1e8f : zj[k];
            const float p = expf(v - lse);
            cdf += p;
            if (cdf <= uj) ++count;
            if (p > 0.f) last = k;
        }
        const int a = count < last ? count : last;
        const float va = (mj && !mj[a]) ? -1e8f : zj[a];
        nlp += -(va - lse);
        actions[j] = (int64_t)a;
    }
    return nlp;
}

struct CatRowOut { float a_loss, c_loss, ent, kl, clipped, d_value; };

// the per-row scalars once a row's neglogp and entropy (sums over its heads) are known: actor loss and g_a = d(actor)/d(neglogp), which
// the logit gradients scale by; critic loss and d(critic)/d(value)
__host__ __device__ inline void cat_row_scalars(float nlp, float val, float old_nlp, float adv, float old_v, float ret, const CatLossDev& c,
                                                float& a_loss, float& g_a, float& c_loss, float& dc) {
    // actor loss + d/dnlp (common_losses.py:41-82)
    if (c.ppo) {
        const float ratio = expf(old_nlp - nlp);
        const float mi = 1.0f - c.e_clip, mx = 1.0f + c.e_clip;
        float clamped, dcl;
        if (c.smooth) {
            const float s = 1.0f / (1.0f + expf((-(ratio - mi) / (mx - mi) + 0.5f) * 4.0f));
            clamped = s * (mx - mi) + mi;
            dcl = 4.0f * s * (1.0f - s);
        } else {
            clamped = fminf(fmaxf(ratio, mi), mx);
            dcl = (ratio >= mi && ratio <= mx) ? 1.0f : 0.0f;
        }
        const float t1 = -(adv * ratio), t2 = -(adv * clamped);
        a_loss = fmaxf(t1, t2);
        const float d1 = adv * ratio, d2 = adv * dcl * ratio;             // d(-adv * f(ratio))/dnlp = adv * f'(ratio) * ratio
        g_a = (t1 > t2) ? d1 : ((t1 < t2) ? d2 : 0.5f * (d1 + d2));
    } else {
        a_loss = nlp * adv;
        g_a = adv;
    }
    // critic loss + d/dvalue (common_losses.py:7-38)
    if (c.clip_value) {
        const float delta = val - old_v;
        const float vpc = old_v + fminf(fmaxf(delta, -c.e_clip), c.e_clip);
        const float e1 = val - ret, e2 = vpc - ret;
        const float l1 = e1 * e1, l2 = e2 * e2;
        c_loss = fmaxf(l1, l2);
        const float g1 = 2.0f * e1, g2 = (delta >= -c.e_clip && delta <= c.e_clip) ? 2.0f * e2 : 0.0f;
        dc = (l1 > l2) ? g1 : ((l1 < l2) ? g2 : 0.5f * (g1 + g2));
    } else {
        const float e1 = ret - val;
        c_loss = e1 * e1;
        dc = -2.0f * e1;
    }
}

__host__ __device__ inline CatRowOut cat_row_out(float a_loss, float c_loss, float ent, float dl, float w, float dc, const CatLossDev& c) {
    CatRowOut o;
    o.a_loss = a_loss; o.c_loss = c_loss; o.ent = ent;
    o.kl = 0.5f * dl * dl;                                                // a2c_discrete.py:189
    o.clipped = (fabsf(expf(dl) - 1.0f) > c.e_clip) ? 1.f : 0.f;
    o.d_value = w * 0.5f * c.critic_coef * dc;
    return o;
}

// loss pieces of one row and the gradient of  w * (a + 0.5 * critic_coef * c - entropy_coef * H)  w.r.t. its logits (dz[sum K_j]) / value
__host__ __device__ inline CatRowOut cat_loss_row(const float* z, const uint8_t* mk, const CatHeads& hd, const int64_t* actions, float val,
                                                  float old_nlp, float adv, float old_v, float ret, float w, const CatLossDev& c, float* dz) {
    float lse[CAT_MAXH], entj[CAT_MAXH];
    float nlp = 0.f, ent = 0.f;
    for (int j = 0; j < hd.n; ++j) {
        const float* zj = z + hd.off[j];
        const uint8_t* mj = mk ? mk + hd.off[j] : nullptr;
        cat_lse(zj, mj, hd.size[j], lse[j]);
        const int a = (int)actions[j];
        const float za = (mj && !mj[a]) ? -1e8f : zj[a];
        nlp += -(za - lse[j]);
        // entropy: -sum p log p over legal actions (distributions.py:38-44; unmasked: torch Categorical.entropy)
        float e = 0.f;
        for (int k = 0; k < hd.size[j]; ++k) {
            if (mj && !mj[k]) continue;
            const float lp = zj[k] - lse[j];
            e -= expf(lp) * lp;
        }
        entj[j] = e;
        ent += e;
    }
    float a_loss, g_a, c_loss, dc;
    cat_row_scalars(nlp, val, old_nlp, adv, old_v, ret, c, a_loss, g_a, c_loss, dc);
    const float dl = old_nlp - nlp;
    // gradients, head by head: dnlp/dz_k = p_k - [k == a_j];   dH/dz_k = -p_k (log p_k + H_j)   (a2c_discrete.py:163-165)
    for (int j = 0; j < hd.n; ++j) {
        const float* zj = z + hd.off[j];
        const uint8_t* mj = mk ? mk + hd.off[j] : nullptr;
        const int a = (int)actions[j];
        for (int k = 0; k < hd.size[j]; ++k) {
            float g = 0.f;
            if (!(mj && !mj[k])) {
                const float lp = zj[k] - lse[j], p = expf(lp);
                g = w * (g_a * (p - (k == a ? 1.0f : 0.0f)) + c.entropy_coef * p * (lp + entj[j]));
            }
            dz[hd.off[j] + k] = g;
        }
    }
    return cat_row_out(a_loss, c_loss, ent, dl, w, dc, c);
}

// ---- per-THREAD bodies: everything a kernel thread does except the block reduction, __host__ __device__ so that the arena
//      addressing (row strides, chunk mapping, mask / action layouts) is exercised on the CPU too (host test entry points
//      b200rl_hosttest_categorical_*_arena, tests/test_discrete_rows_cpu.py) ------------------------------------------------------
__host__ __device__ inline int64_t chunk_row_hd(int m, int rows_per_chunk, int64_t chunk_stride) {
    const int c = m / rows_per_chunk;
    return (int64_t)c * chunk_stride + (m - c * rows_per_chunk);
}

struct CatSampleArgs {
    const float* logits; int ld; int K; CatHeads hd; const float* value_raw; int value_ld; const uint8_t* action_masks;
    const float* u_tape; uint64_t seed; const uint64_t* rng_epoch_dev; uint32_t step_index; const double* vms_mean; const double* vms_var;
    int normalize_value; int64_t* actions; float* neglogp; float* values; const uint8_t* dones_cur; uint8_t* dones_out;
    const float* prev_dones; float* valid_out; int N; int values_only;
};

// rollout: sample (inverse CDF, one uniform per row and head), neglogp, de-normalised value.
// actions: int64 [N, n_heads]; u_tape (optional): float [n_heads, N]
__host__ __device__ inline void cat_sample_thread(const CatSampleArgs& a, int e) {
    // value: denorm_value (running_mean_std.py:104-106): sqrt(var + eps) * clamp(v, -5, 5) + mean
    float val = a.value_raw[(int64_t)e * a.value_ld];
    if (a.normalize_value) {
        const float m = (float)a.vms_mean[0];
#ifdef __CUDA_ARCH__
        const float s = __fsqrt_rn(__fadd_rn((float)a.vms_var[0], 1e-5f));
        val = __fadd_rn(__fmul_rn(s, fminf(fmaxf(val, -5.0f), 5.0f)), m);
#else
        const float s = sqrtf((float)a.vms_var[0] + 1e-5f);
        val = s * fminf(fmaxf(val, -5.0f), 5.0f) + m;
#endif
    }
    a.values[e] = val;
    if (a.values_only) return;
    float ubuf[CAT_MAXH];
    const float* u = ubuf;
    int64_t ustride = 1;
    if (a.u_tape) {
        u = a.u_tape + e;
        ustride = a.N;
    } else {
#ifdef __CUDA_ARCH__
        const uint64_t ep = a.rng_epoch_dev ? *a.rng_epoch_dev : 0ull;
        for (int j = 0; j < a.hd.n; ++j) {
            const Philox4 r = philox4x32_10((uint64_t)e, (ep << 20) | ((uint64_t)a.step_index << 4) | (uint64_t)(8 + j), a.seed);
            ubuf[j] = (float)(r.x >> 8) * (1.0f / 16777216.0f);           // [0, 1)
        }
#else
        for (int j = 0; j < a.hd.n; ++j) ubuf[j] = 0.5f;                  // the host test always supplies the uniform tape
#endif
    }
    a.neglogp[e] = cat_sample_row(a.logits + (int64_t)e * a.ld, a.action_masks ? a.action_masks + (int64_t)e * a.K : nullptr, a.hd, u, ustride,
                                  a.actions + (int64_t)e * a.hd.n);
    if (a.dones_out) a.dones_out[e] = a.dones_cur[e];
    if (a.valid_out) a.valid_out[e] = a.prev_dones ? (1.0f - a.prev_dones[e]) : 1.0f;
}

__global__ void __launch_bounds__(256) categorical_sample_kernel(const CatSampleArgs a) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < a.N) cat_sample_thread(a, e);
}

// training: loss pieces + gradients at the logits / value for one minibatch
struct CatLossArgs {
    const float* logits; int ld; int K; CatHeads hd; const float* values; int value_ld; const int64_t* actions;
    const uint8_t* action_masks; const float* old_values_n; const float* returns_n; const float* old_neglogp; const float* advs_n;
    const float* mask; int rows_per_chunk; int64_t chunk_stride; int M; CatLossDev c; const float* inv_count_dev; float* d_logits; int d_ld;
    float* d_value; int dv_ld;
};

// acc: sum w*a_loss, sum w*c_loss, sum w*entropy, sum w*kl, sum mask, sum mask*clipped, sum w
__host__ __device__ inline void cat_loss_thread(const CatLossArgs& a, int m, double (&acc)[7]) {
    const int64_t ar = chunk_row_hd(m, a.rows_per_chunk, a.chunk_stride);
    const float mkr = a.mask ? a.mask[ar] : 1.0f;
    const float inv_cnt = a.inv_count_dev ? a.inv_count_dev[0] : (1.0f / (float)a.M);
    const float w = mkr * inv_cnt;
    const CatRowOut o = cat_loss_row(a.logits + (int64_t)m * a.ld, a.action_masks ? a.action_masks + ar * a.K : nullptr, a.hd,
                                     a.actions + ar * a.hd.n, a.values[(int64_t)m * a.value_ld], a.old_neglogp[ar], a.advs_n[ar],
                                     a.old_values_n[ar], a.returns_n[ar], w, a.c, a.d_logits + (int64_t)m * a.d_ld);
    a.d_value[(int64_t)m * a.dv_ld] = o.d_value;
    acc[0] = (double)w * o.a_loss; acc[1] = (double)w * o.c_loss; acc[2] = (double)w * o.ent; acc[3] = (double)w * o.kl;
    acc[4] = mkr; acc[5] = mkr * o.clipped; acc[6] = w;
}

// partial row (8 doubles per block): the seven sums above, 0
__global__ void __launch_bounds__(256) categorical_loss_kernel(const CatLossArgs a, double* __restrict__ partials) {
    __shared__ double sm[32 * 7];
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    double acc[7] = {0, 0, 0, 0, 0, 0, 0};
    if (m < a.M) cat_loss_thread(a, m, acc);
    block_sum_d<7>(acc, sm);
    if (threadIdx.x == 0) {
        double* p = partials + (int64_t)blockIdx.x * 8;
#pragma unroll
        for (int i = 0; i < 7; ++i) p[i] = acc[i];
        p[7] = 0.0;
    }
}

// head table from the host: sizes of n_heads heads (NULL / 0 = one head of K actions); returns false on a bad table
static bool make_heads(int K, int n_heads, const int* head_sizes_host, CatHeads& hd) {
    if (n_heads <= 0 || !head_sizes_host) { hd.n = 1; hd.size[0] = K; hd.off[0] = 0; return K > 0 && K <= CAT_MAXK; }
    if (n_heads > CAT_MAXH) return false;
    hd.n = n_heads;
    int off = 0;
    for (int j = 0; j < n_heads; ++j) {
        if (head_sizes_host[j] <= 0 || head_sizes_host[j] > CAT_MAXK) return false;
        hd.size[j] = head_sizes_host[j]; hd.off[j] = off; off += head_sizes_host[j];
    }
    return off == K;
}

// ---- wide heads: any number of heads of any size ----------------------------------------------------------------------------------
// One CTA per row, WIDE_WARPS(n_heads) warps; warp w takes heads w, w + W, w + 2W, ... of its row and sums their neglogp / entropy in
// that order, then thread 0 adds the W warp sums in warp order: a fixed order per layout, no atomics, so repeated runs give the same
// bits.  Head j covers logits [off[j], off[j + 1]) of the row, off being the device table head_offsets_dev [n_heads + 1] (NULL: one
// head of K actions).  Every row index is 64-bit.
constexpr int CATW_MAXWARPS = 8;
__host__ __device__ inline int wide_warps(int n_heads) { return n_heads < CATW_MAXWARPS ? n_heads : CATW_MAXWARPS; }

__device__ __forceinline__ float cat_logit(const float* z, const uint8_t* mk, int k) { return (mk && !mk[k]) ? -1e8f : z[k]; }

// (max, sum of exp(v - max)) of two partial log-sum-exps; an empty side has max = -inf
__device__ __forceinline__ void lse_merge(float& m, float& s, float om, float os) {
    const float mm = fmaxf(m, om);
    s = (m == -INFINITY ? 0.f : s * expf(m - mm)) + (om == -INFINITY ? 0.f : os * expf(om - mm));
    m = mm;
}

// masked log-sum-exp of one head: each lane runs an online log-sum-exp over actions lane, lane + 32, ..., then a butterfly merges the
// lanes (each merge is symmetric, so every lane ends with the same bits)
__device__ __forceinline__ float warp_lse(const float* z, const uint8_t* mk, int K, int lane) {
    float m = -INFINITY, s = 0.f;
    for (int k = lane; k < K; k += 32) {
        const float v = cat_logit(z, mk, k);
        if (v > m) { s = s * expf(m - v) + 1.0f; m = v; }
        else s += expf(v - m);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, m, o), os = __shfl_xor_sync(0xffffffffu, s, o);
        lse_merge(m, s, om, os);
    }
    return m + logf(s);
}

__device__ __forceinline__ void wide_head(const int* off, int K, int j, int& o, int& n) {
    if (off) { o = off[j]; n = off[j + 1] - o; }
    else { o = 0; n = K; }
}

// fixed-order sum of the W warp values v (lane 0 of each warp) through sm[W]: every thread returns the same sum
__device__ __forceinline__ float wide_row_sum(float v, float* sm) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    if (lane == 0) sm[warp] = v;
    __syncthreads();
    float t = 0.f;
    for (int i = 0; i < nw; ++i) t += sm[i];
    __syncthreads();
    return t;
}

// rollout: one uniform per head, from the tape u_tape [n_heads, N] or Philox.  Philox counter of head j of row e:
// ctr_lo = e | (j >> 3) << 32, ctr_hi = epoch << 20 | step << 4 | (8 + (j & 7)); for j < 8 that is the narrow kernel's counter.
// The cdf of a head is summed 32 actions at a time: cdf_k = carry + S(k), S = the inclusive Hillis-Steele warp scan of p over the
// chunk [32c, 32c + 32) (step d = 1, 2, 4, 8, 16: x_l += x_{l-d} for l >= d), carry = the cdf at the previous chunk's last action
// (0 for the first chunk).  action = #{k : cdf_k <= u}, clamped to the last action with p > 0, as cat_sample_row.
__global__ void __launch_bounds__(256) categorical_sample_wide_kernel(const CatSampleArgs a, int n_heads, const int* __restrict__ off) {
    __shared__ float sm[CATW_MAXWARPS];
    const int64_t e = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const float* z = a.logits + e * a.ld;
    const uint8_t* mk = a.action_masks ? a.action_masks + e * a.K : nullptr;
    const uint64_t ep = (!a.u_tape && a.rng_epoch_dev) ? *a.rng_epoch_dev : 0ull;
    float nlp = 0.f;
    for (int j = warp; j < n_heads; j += nw) {
        int o, K;
        wide_head(off, a.K, j, o, K);
        const float* zj = z + o;
        const uint8_t* mj = mk ? mk + o : nullptr;
        const float lse = warp_lse(zj, mj, K, lane);
        float u;
        if (a.u_tape) {
            u = a.u_tape[(int64_t)j * a.N + e];
        } else {
            const Philox4 r = philox4x32_10((uint64_t)e | ((uint64_t)(j >> 3) << 32),
                                            (ep << 20) | ((uint64_t)a.step_index << 4) | (uint64_t)(8 + (j & 7)), a.seed);
            u = (float)(r.x >> 8) * (1.0f / 16777216.0f);                  // [0, 1)
        }
        float carry = 0.f;
        int count = 0, last = 0;
        for (int base = 0; base < K; base += 32) {
            const int k = base + lane;
            const float p = k < K ? expf(cat_logit(zj, mj, k) - lse) : 0.f;
            float x = p;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const float y = __shfl_up_sync(0xffffffffu, x, d);
                if (lane >= d) x += y;
            }
            const float cdf = carry + x;
            count += __popc(__ballot_sync(0xffffffffu, k < K && cdf <= u));
            if (k < K && p > 0.f) last = k;
            carry = __shfl_sync(0xffffffffu, cdf, 31);
        }
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) last = max(last, __shfl_xor_sync(0xffffffffu, last, s));
        const int act = count < last ? count : last;
        if (lane == 0) {
            nlp += -(cat_logit(zj, mj, act) - lse);
            a.actions[e * n_heads + j] = (int64_t)act;
        }
    }
    nlp = wide_row_sum(nlp, sm);
    if (threadIdx.x == 0) {
        float val = a.value_raw[e * a.value_ld];
        if (a.normalize_value) {
            const float m = (float)a.vms_mean[0];
            const float s = __fsqrt_rn(__fadd_rn((float)a.vms_var[0], 1e-5f));
            val = __fadd_rn(__fmul_rn(s, fminf(fmaxf(val, -5.0f), 5.0f)), m);
        }
        a.values[e] = val;
        a.neglogp[e] = nlp;
        if (a.dones_out) a.dones_out[e] = a.dones_cur[e];
        if (a.valid_out) a.valid_out[e] = a.prev_dones ? (1.0f - a.prev_dones[e]) : 1.0f;
    }
}

// training: pass 1 finds each head's log-sum-exp and entropy and parks them in the head's first two gradient slots (a head of one action
// has a zero gradient and parks nothing); the row's neglogp and entropy give g_a (cat_row_scalars); pass 2 reads the two values back and
// writes the head's gradient over them.  The warp that parks a head's values is the warp that reads them back.
// Partial rows: one per row (8 doubles, as categorical_loss_kernel's per-block rows).
__global__ void __launch_bounds__(256) categorical_loss_wide_kernel(const CatLossArgs a, int n_heads, const int* __restrict__ off,
                                                                    double* __restrict__ partials) {
    __shared__ float sm[CATW_MAXWARPS];
    __shared__ float sg[2];
    const int m = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const int64_t ar = chunk_row(m, a.rows_per_chunk, a.chunk_stride);
    const float* z = a.logits + (int64_t)m * a.ld;
    const uint8_t* mk = a.action_masks ? a.action_masks + ar * a.K : nullptr;
    const int64_t* act = a.actions + ar * n_heads;
    float* dz = a.d_logits + (int64_t)m * a.d_ld;
    // the row's scalars are read up front: 64-bit row offsets kept alive across thread 0's section would be spilled
    float mkr = 1.0f, val = 0.f, old_nlp = 0.f, adv = 0.f, old_v = 0.f, ret = 0.f;
    if (threadIdx.x == 0) {
        mkr = a.mask ? a.mask[ar] : 1.0f;
        val = a.values[(int64_t)m * a.value_ld];
        old_nlp = a.old_neglogp[ar]; adv = a.advs_n[ar]; old_v = a.old_values_n[ar]; ret = a.returns_n[ar];
    }
    float nlp = 0.f, ent = 0.f;
    for (int j = warp; j < n_heads; j += nw) {
        int o, K;
        wide_head(off, a.K, j, o, K);
        const float* zj = z + o;
        const uint8_t* mj = mk ? mk + o : nullptr;
        const float lse = warp_lse(zj, mj, K, lane);
        float e = 0.f;                                                    // -sum p log p over legal actions (distributions.py:38-44)
        for (int k = lane; k < K; k += 32) {
            if (mj && !mj[k]) continue;
            const float lp = zj[k] - lse;
            e -= expf(lp) * lp;
        }
        e = warp_sum(e);
        if (lane == 0) {
            nlp += -(cat_logit(zj, mj, (int)act[j]) - lse);
            ent += e;
            if (K > 1) { dz[o] = lse; dz[o + 1] = e; }
        }
    }
    nlp = wide_row_sum(nlp, sm);
    ent = wide_row_sum(ent, sm);
    if (threadIdx.x == 0) {
        const float inv_cnt = a.inv_count_dev ? a.inv_count_dev[0] : (1.0f / (float)a.M);
        const float w = mkr * inv_cnt;
        float a_loss, g_a, c_loss, dc;
        cat_row_scalars(nlp, val, old_nlp, adv, old_v, ret, a.c, a_loss, g_a, c_loss, dc);
        const CatRowOut r = cat_row_out(a_loss, c_loss, ent, old_nlp - nlp, w, dc, a.c);
        a.d_value[(int64_t)m * a.dv_ld] = r.d_value;
        double* p = partials + (int64_t)m * 8;
        p[0] = (double)w * r.a_loss; p[1] = (double)w * r.c_loss; p[2] = (double)w * r.ent; p[3] = (double)w * r.kl;
        p[4] = mkr; p[5] = mkr * r.clipped; p[6] = w; p[7] = 0.0;
        sg[0] = w; sg[1] = g_a;
    }
    __syncthreads();
    const float w = sg[0], g_a = sg[1], ce = a.c.entropy_coef;
    for (int j = warp; j < n_heads; j += nw) {
        int o, K;
        wide_head(off, a.K, j, o, K);
        if (K == 1) {
            if (lane == 0) dz[o] = 0.f;
            continue;
        }
        const float lse = dz[o], e = dz[o + 1];
        __syncwarp();
        const float* zj = z + o;
        const uint8_t* mj = mk ? mk + o : nullptr;
        const int aj = (int)act[j];
        for (int k = lane; k < K; k += 32) {
            float g = 0.f;
            if (!(mj && !mj[k])) {
                const float lp = zj[k] - lse, p = expf(lp);
                g = w * (g_a * (p - (k == aj ? 1.0f : 0.0f)) + ce * p * (lp + e));
            }
            dz[o + k] = g;
        }
    }
}

// checks a wide layout against its host copy of the head sizes (n_heads <= 0 or NULL sizes: one head of K actions); heads = its head count
static bool wide_heads_ok(int K, int n_heads, const int* head_sizes_host, const int* head_offsets_dev, int& heads) {
    if (n_heads <= 0 || !head_sizes_host) { heads = 1; return K > 0; }
    if (!head_offsets_dev) return false;
    int64_t tot = 0;
    for (int j = 0; j < n_heads; ++j) {
        if (head_sizes_host[j] <= 0) return false;
        tot += head_sizes_host[j];
    }
    heads = n_heads;
    return tot == K;
}

}  // namespace

B200RL_EXPORT int b200rl_categorical_sample_f32(const float* logits, int ld, int K, int n_heads, const int* head_sizes_host,
                                                const float* value_raw, int value_ld,
                                                const uint8_t* action_masks, const float* u_tape, uint64_t seed,
                                                const uint64_t* rng_epoch_dev, uint32_t step_index, const double* vms_mean,
                                                const double* vms_var, int normalize_value, int64_t* actions, float* neglogp,
                                                float* values, const uint8_t* dones_cur, uint8_t* dones_out, const float* prev_dones,
                                                float* valid_out, int N, int values_only, void* stream) {
    if (!value_raw || !values || N <= 0 || value_ld <= 0) return B200RL_EINVAL;
    CatHeads hd{};
    if (!values_only && (!logits || !actions || !neglogp || ld < K || !make_heads(K, n_heads, head_sizes_host, hd))) return B200RL_EINVAL;
    if (normalize_value && (!vms_mean || !vms_var)) return B200RL_EINVAL;
    if (dones_out && !dones_cur) return B200RL_EINVAL;
    const CatSampleArgs a{logits, ld, K, hd, value_raw, value_ld, action_masks, u_tape, seed, rng_epoch_dev, step_index, vms_mean, vms_var,
                          normalize_value, actions, neglogp, values, dones_cur, dones_out, prev_dones, valid_out, N, values_only};
    categorical_sample_kernel<<<(N + 255) / 256, 256, 0, as_stream(stream)>>>(a);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_categorical_loss_f32(const float* logits, int ld, int K, int n_heads, const int* head_sizes_host,
                                              const float* values, int value_ld,
                                              const int64_t* actions, const uint8_t* action_masks, const float* old_values_n,
                                              const float* returns_n, const float* old_neglogp, const float* advs_n, const float* mask,
                                              int rows_per_chunk, int64_t chunk_stride, int M, const b200rl_cat_loss_cfg* cfg_host,
                                              const float* inv_count_dev, float* d_logits, int d_ld, float* d_value, int dv_ld,
                                              double* partials, int max_partials, int* n_blocks_out_host, void* stream) {
    if (!logits || !values || !actions || !old_values_n || !returns_n || !old_neglogp || !advs_n || !cfg_host || !d_logits || !d_value ||
        !partials)
        return B200RL_EINVAL;
    CatHeads hd{};
    if (M <= 0 || ld < K || d_ld < K || value_ld <= 0 || dv_ld <= 0 || rows_per_chunk <= 0 || !make_heads(K, n_heads, head_sizes_host, hd))
        return B200RL_EINVAL;
    const int blocks = (M + 255) / 256;
    if (n_blocks_out_host) *n_blocks_out_host = blocks;
    if (blocks > max_partials) return B200RL_EINVAL;
    CatLossDev c{cfg_host->e_clip, cfg_host->critic_coef, cfg_host->entropy_coef, cfg_host->clip_value, cfg_host->use_smooth_clamp,
                 cfg_host->ppo};
    const CatLossArgs a{logits, ld, K, hd, values, value_ld, actions, action_masks, old_values_n, returns_n, old_neglogp, advs_n, mask,
                        rows_per_chunk, chunk_stride, M, c, inv_count_dev, d_logits, d_ld, d_value, dv_ld};
    categorical_loss_kernel<<<blocks, 256, 0, as_stream(stream)>>>(a, partials);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_categorical_sample_wide_f32(const float* logits, int ld, int K, int n_heads, const int* head_sizes_host,
                                                     const int* head_offsets_dev, const float* value_raw, int value_ld,
                                                     const uint8_t* action_masks, const float* u_tape, uint64_t seed,
                                                     const uint64_t* rng_epoch_dev, uint32_t step_index, const double* vms_mean,
                                                     const double* vms_var, int normalize_value, int64_t* actions, float* neglogp,
                                                     float* values, const uint8_t* dones_cur, uint8_t* dones_out, const float* prev_dones,
                                                     float* valid_out, int N, void* stream) {
    int heads = 0;
    if (!logits || !value_raw || !values || !actions || !neglogp || N <= 0 || value_ld <= 0 || ld < K ||
        !wide_heads_ok(K, n_heads, head_sizes_host, head_offsets_dev, heads))
        return B200RL_EINVAL;
    if (normalize_value && (!vms_mean || !vms_var)) return B200RL_EINVAL;
    if (dones_out && !dones_cur) return B200RL_EINVAL;
    const CatSampleArgs a{logits, ld, K, CatHeads{}, value_raw, value_ld, action_masks, u_tape, seed, rng_epoch_dev, step_index, vms_mean,
                          vms_var, normalize_value, actions, neglogp, values, dones_cur, dones_out, prev_dones, valid_out, N, 0};
    categorical_sample_wide_kernel<<<N, 32 * wide_warps(heads), 0, as_stream(stream)>>>(a, heads, heads > 1 ? head_offsets_dev : nullptr);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_categorical_loss_wide_f32(const float* logits, int ld, int K, int n_heads, const int* head_sizes_host,
                                                   const int* head_offsets_dev, const float* values, int value_ld,
                                                   const int64_t* actions, const uint8_t* action_masks, const float* old_values_n,
                                                   const float* returns_n, const float* old_neglogp, const float* advs_n, const float* mask,
                                                   int rows_per_chunk, int64_t chunk_stride, int M, const b200rl_cat_loss_cfg* cfg_host,
                                                   const float* inv_count_dev, float* d_logits, int d_ld, float* d_value, int dv_ld,
                                                   double* partials, int max_partials, int* n_blocks_out_host, void* stream) {
    if (!logits || !values || !actions || !old_values_n || !returns_n || !old_neglogp || !advs_n || !cfg_host || !d_logits || !d_value ||
        !partials)
        return B200RL_EINVAL;
    int heads = 0;
    if (M <= 0 || ld < K || d_ld < K || value_ld <= 0 || dv_ld <= 0 || rows_per_chunk <= 0 ||
        !wide_heads_ok(K, n_heads, head_sizes_host, head_offsets_dev, heads))
        return B200RL_EINVAL;
    if (n_blocks_out_host) *n_blocks_out_host = M;
    if (M > max_partials) return B200RL_EINVAL;
    CatLossDev c{cfg_host->e_clip, cfg_host->critic_coef, cfg_host->entropy_coef, cfg_host->clip_value, cfg_host->use_smooth_clamp,
                 cfg_host->ppo};
    const CatLossArgs a{logits, ld, K, CatHeads{}, values, value_ld, actions, action_masks, old_values_n, returns_n, old_neglogp, advs_n,
                        mask, rows_per_chunk, chunk_stride, M, c, inv_count_dev, d_logits, d_ld, d_value, dv_ld};
    categorical_loss_wide_kernel<<<M, 32 * wide_warps(heads), 0, as_stream(stream)>>>(a, heads, heads > 1 ? head_offsets_dev : nullptr,
                                                                                      partials);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

#ifdef B200RL_TEST_HOOKS   // test-only host entry points: compiled into tests/libb200rl_testhooks.so (csrc/build.py), not into the product library
// ---- host test entry points: the per-row functions above, run on the CPU over HOST arrays (no GPU involved).  Test infrastructure for
//      tests/test_discrete_rows_cpu.py; not declared in include/b200rl.h and never called by the product. -----------------------------
B200RL_EXPORT int b200rl_hosttest_categorical_sample_rows(const float* logits, int K, int n_heads, const int* head_sizes, const uint8_t* masks,
                                                         const float* u /* [n_heads, N] */, int N, int64_t* actions /* [N, n_heads] */,
                                                         float* neglogp) {
    CatHeads hd{};
    if (!make_heads(K, n_heads, head_sizes, hd)) return B200RL_EINVAL;
    for (int e = 0; e < N; ++e)
        neglogp[e] = cat_sample_row(logits + (int64_t)e * K, masks ? masks + (int64_t)e * K : nullptr, hd, u + e, N, actions + (int64_t)e * hd.n);
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_hosttest_categorical_loss_rows(const float* logits, int K, int n_heads, const int* head_sizes, const float* values,
                                                       const int64_t* actions /* [M, n_heads] */,
                                                       const uint8_t* masks, const float* old_values_n, const float* returns_n,
                                                       const float* old_neglogp, const float* advs_n, const float* w, int M,
                                                       const b200rl_cat_loss_cfg* cfg, float* d_logits, float* d_value, double* sums4) {
    CatLossDev c{cfg->e_clip, cfg->critic_coef, cfg->entropy_coef, cfg->clip_value, cfg->use_smooth_clamp, cfg->ppo};
    CatHeads hd{};
    if (!make_heads(K, n_heads, head_sizes, hd)) return B200RL_EINVAL;
    double acc[4] = {0, 0, 0, 0};
    for (int m = 0; m < M; ++m) {
        const CatRowOut o = cat_loss_row(logits + (int64_t)m * K, masks ? masks + (int64_t)m * K : nullptr, hd, actions + (int64_t)m * hd.n, values[m],
                                         old_neglogp[m], advs_n[m], old_values_n[m], returns_n[m], w[m], c, d_logits + (int64_t)m * K);
        d_value[m] = o.d_value;
        acc[0] += (double)w[m] * o.a_loss; acc[1] += (double)w[m] * o.c_loss; acc[2] += (double)w[m] * o.ent; acc[3] += (double)w[m] * o.kl;
    }
    for (int i = 0; i < 4; ++i) sums4[i] = acc[i];
    return B200RL_OK;
}

// the kernels' per-thread bodies over HOST arrays laid out like the device arena (same arguments as the C-ABI entry points, no stream):
// arena addressing and strides on the CPU.  One partial row (8 doubles) for the loss.
B200RL_EXPORT int b200rl_hosttest_categorical_sample_arena(const float* logits, int ld, int K, int n_heads, const int* head_sizes,
                                                          const float* value_raw, int value_ld, const uint8_t* action_masks, const float* u_tape,
                                                          const double* vms_mean, const double* vms_var, int normalize_value, int64_t* actions,
                                                          float* neglogp, float* values, const uint8_t* dones_cur, uint8_t* dones_out,
                                                          const float* prev_dones, float* valid_out, int N, int values_only) {
    CatHeads hd{};
    if (!values_only && !make_heads(K, n_heads, head_sizes, hd)) return B200RL_EINVAL;
    const CatSampleArgs a{logits, ld, K, hd, value_raw, value_ld, action_masks, u_tape, 0ull, nullptr, 0u, vms_mean, vms_var,
                          normalize_value, actions, neglogp, values, dones_cur, dones_out, prev_dones, valid_out, N, values_only};
    for (int e = 0; e < N; ++e) cat_sample_thread(a, e);
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_hosttest_categorical_loss_arena(const float* logits, int ld, int K, int n_heads, const int* head_sizes,
                                                        const float* values, int value_ld, const int64_t* actions, const uint8_t* action_masks,
                                                        const float* old_values_n, const float* returns_n, const float* old_neglogp,
                                                        const float* advs_n, const float* mask, int rows_per_chunk, int64_t chunk_stride, int M,
                                                        const b200rl_cat_loss_cfg* cfg, const float* inv_count, float* d_logits, int d_ld,
                                                        float* d_value, int dv_ld, double* partial8) {
    CatHeads hd{};
    if (!make_heads(K, n_heads, head_sizes, hd)) return B200RL_EINVAL;
    const CatLossDev c{cfg->e_clip, cfg->critic_coef, cfg->entropy_coef, cfg->clip_value, cfg->use_smooth_clamp, cfg->ppo};
    const CatLossArgs a{logits, ld, K, hd, values, value_ld, actions, action_masks, old_values_n, returns_n, old_neglogp, advs_n, mask,
                        rows_per_chunk, chunk_stride, M, c, inv_count, d_logits, d_ld, d_value, dv_ld};
    double tot[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int m = 0; m < M; ++m) {
        double acc[7] = {0, 0, 0, 0, 0, 0, 0};
        cat_loss_thread(a, m, acc);
        for (int i = 0; i < 7; ++i) tot[i] += acc[i];
    }
    for (int i = 0; i < 8; ++i) partial8[i] = tot[i];
    return B200RL_OK;
}
#endif  // B200RL_TEST_HOOKS
