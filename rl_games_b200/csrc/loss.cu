// PPO loss head: head GEMM (mu, value) + distribution math + clipped-surrogate / value / bound losses +
// analytic KL + the backward pass of all of it down to d(last hidden activation), fused in one kernel.
// Replaces a2c_continuous.py:97-134 (calc_losses), :241-257, common_losses.py:16-82, torch_ext.py:27-36,
// :157-170, models.py:335-364 and ~135 eager launches + loss.backward() for this part of the graph.
// One thread per sample; the [128 x Hl] activation tile and the head weights are staged in shared memory;
// scalar statistics go through warp-shuffle reductions into per-block fp64 partials (deterministic).
#include "common.cuh"
#include "loss_math.cuh"

namespace {

constexpr int LT = 128;       // threads (= samples) per block
constexpr int MAXA = 32;      // max action dim + 1 supported by the register tiles
constexpr int NSC = LOSS_NSC; // scalar partial slots before the dlogstd block
constexpr int MAXA_SD = 16;   // state-dependent sigma: value + up to 15 mu rows, up to 15 raw-sigma rows

// SD = state-dependent sigma: the head has 1 + 2A rows (value, mu, raw sigma), sigma is per row (sigma_param) and the raw-sigma
// gradient of each row goes to d_head[1 + A + j] and into d_alast instead of into the dlogstd partial slots (those stay 0).
template <int MA, bool SD>
__device__ __forceinline__ void ppo_head_loss_body(
    const float* __restrict__ a_last, int Hl, const float* __restrict__ Wh, const float* __restrict__ bh,
    const float* __restrict__ logstd, const float* __restrict__ actions, float* __restrict__ old_mu,
    float* __restrict__ old_sigma, const float* __restrict__ old_values_n, const float* __restrict__ returns_n,
    const float* __restrict__ old_neglogp, const float* __restrict__ advs_n, const float* __restrict__ mask,
    int rows_per_chunk, int64_t chunk_stride, int M, int A, const LossCfgDev& cfg, const float* __restrict__ inv_count_dev,
    float* __restrict__ d_head, float* __restrict__ d_alast, int act_last,
    float* __restrict__ mu_out, float* __restrict__ value_out, float* __restrict__ neglogp_out,
    double* __restrict__ partials, const SigmaCfgDev& scfg, const float* __restrict__ entropy_coef_dev) {
    extern __shared__ float smf[];
    const int AH = A + 1;
    const int HR = SD ? 1 + 2 * A : AH;              // head rows
    float* tile = smf;                               // [LT][Hl+1]
    float* sW = tile + LT * (Hl + 1);                // [HR][Hl]
    float* sB = sW + HR * Hl;                        // [HR]
    float* sSig = sB + HR;                           // sigma, logstd, 1/sigma, log(sigma): 4*A (fixed sigma)
    float* sRed = sSig + 4 * A;                      // [LT/32][NSC + A]
    const int tid = threadIdx.x;
    const int m0 = blockIdx.x * LT;
    const int rows = min(LT, M - m0);
    // ---- stage tile + head weights ----
    for (int i = tid; i < rows * Hl; i += LT) {
        const int r = i / Hl, k = i - r * Hl;
        tile[r * (Hl + 1) + k] = __ldg(a_last + (int64_t)(m0 + r) * Hl + k);
    }
    for (int i = tid; i < HR * Hl; i += LT) sW[i] = __ldg(Wh + i);
    if (tid < HR) sB[tid] = __ldg(bh + tid);
    if (!SD && tid < A) loss_fill_sigma(sSig, logstd, A, tid);
    __syncthreads();

    float sc[NSC];
#pragma unroll
    for (int i = 0; i < NSC; ++i) sc[i] = 0.f;
    float dls[MA];
#pragma unroll
    for (int j = 0; j < MA; ++j) dls[j] = 0.f;
    float dh[MA];   // dh[0] = dvalue, dh[1+j] = dmu_j

    const int m = m0 + tid;
    const bool live = tid < rows;
    if (live) {
        float head[MA], raw[MA];
#pragma unroll
        for (int j = 0; j < MA; ++j) {
            head[j] = (j < AH) ? sB[j] : 0.f;
            if (SD) raw[j] = (j < A) ? sB[AH + j] : 0.f;
        }
        const float* row = tile + tid * (Hl + 1);
        for (int k = 0; k < Hl; ++k) {
            const float a = row[k];
#pragma unroll
            for (int j = 0; j < MA; ++j) {
                if (j < AH) head[j] = fmaf(a, sW[j * Hl + k], head[j]);
                if (SD && j < A) raw[j] = fmaf(a, sW[(AH + j) * Hl + k], raw[j]);
            }
        }
        RowSigma<MA> rs;
        if (SD) {
#pragma unroll
            for (int j = 0; j < MA; ++j) {
                rs.sg[j] = 1.f; rs.ls[j] = 0.f; rs.dr[j] = 0.f;
                if (j < A) sigma_param(raw[j], scfg, rs.sg[j], rs.ls[j], rs.dr[j]);
            }
        }
        const int64_t ar = chunk_row(m, rows_per_chunk, chunk_stride);
        const float inv_cnt = inv_count_dev ? __ldg(inv_count_dev) : (1.0f / (float)M);
        LossArena la{actions, old_mu, old_sigma, old_values_n, returns_n, old_neglogp, advs_n, mask};
        LossRow<MA> lrow;
        loss_row_load<MA>(la, ar, A, lrow);
        const float nlp = SD ? ppo_sample_loss<MA, false, true>(head, A, sSig, la, ar, lrow, inv_cnt, cfg, dh, dls, sc, &rs,
                                                                __ldg(entropy_coef_dev))
                             : ppo_sample_loss<MA, false>(head, A, sSig, la, ar, lrow, inv_cnt, cfg, dh, dls, sc);
        if (mu_out) {
#pragma unroll
            for (int j = 0; j < MA - 1; ++j)
                if (j < A) mu_out[(int64_t)m * A + j] = head[1 + j];
        }
        if (value_out) value_out[m] = head[0];
        if (neglogp_out) neglogp_out[m] = nlp;
        // ---- d(head) out, d(a_last) into the tile (row owned by this thread) ----
#pragma unroll
        for (int j = 0; j < MA; ++j) {
            if (j < AH) d_head[(int64_t)m * HR + j] = dh[j];
            if (SD && j < A) d_head[(int64_t)m * HR + AH + j] = dls[j];
        }
        float* rw = tile + tid * (Hl + 1);
        for (int k = 0; k < Hl; ++k) {
            float g = 0.f;
#pragma unroll
            for (int j = 0; j < MA; ++j) {
                if (j < AH) g = fmaf(dh[j], sW[j * Hl + k], g);
                if (SD && j < A) g = fmaf(dls[j], sW[(AH + j) * Hl + k], g);
            }
            rw[k] = g * act_bwd_from_out(rw[k], act_last);
        }
    }
    // ---- block reduction of the scalars: warp shuffles -> smem -> fp64 partial row ----
    const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (int i = 0; i < NSC; ++i) sc[i] = warp_sum(sc[i]);
    if (!SD) {
#pragma unroll
        for (int j = 0; j < MA; ++j)
            if (j < A) dls[j] = warp_sum(dls[j]);
    }
    if (lane == 0) {
#pragma unroll
        for (int i = 0; i < NSC; ++i) sRed[warp * (NSC + A) + i] = sc[i];
#pragma unroll
        for (int j = 0; j < MA; ++j)
            if (j < A) sRed[warp * (NSC + A) + NSC + j] = SD ? 0.f : dls[j];
    }
    __syncthreads();
    if (tid < NSC + A) {
        double s = 0.0;
        for (int wv = 0; wv < LT / 32; ++wv) s += (double)sRed[wv * (NSC + A) + tid];
        partials[(int64_t)blockIdx.x * (NSC + MAXA) + tid] = s;
    }
    // ---- coalesced store of d(a_last) ----
    for (int i = tid; i < rows * Hl; i += LT) {
        const int r = i / Hl, k = i - r * Hl;
        d_alast[(int64_t)(m0 + r) * Hl + k] = tile[r * (Hl + 1) + k];
    }
}

__global__ void __launch_bounds__(LT) ppo_head_loss_kernel(
    const float* __restrict__ a_last, int Hl, const float* __restrict__ Wh, const float* __restrict__ bh,
    const float* __restrict__ logstd, const float* __restrict__ actions, float* __restrict__ old_mu,
    float* __restrict__ old_sigma, const float* __restrict__ old_values_n, const float* __restrict__ returns_n,
    const float* __restrict__ old_neglogp, const float* __restrict__ advs_n, const float* __restrict__ mask,
    int rows_per_chunk, int64_t chunk_stride, int M, int A, LossCfgDev cfg, const float* __restrict__ inv_count_dev,
    float* __restrict__ d_head, float* __restrict__ d_alast, int act_last,
    float* __restrict__ mu_out, float* __restrict__ value_out, float* __restrict__ neglogp_out,
    double* __restrict__ partials) {
    ppo_head_loss_body<MAXA, false>(a_last, Hl, Wh, bh, logstd, actions, old_mu, old_sigma, old_values_n, returns_n, old_neglogp, advs_n,
                                    mask, rows_per_chunk, chunk_stride, M, A, cfg, inv_count_dev, d_head, d_alast, act_last, mu_out,
                                    value_out, neglogp_out, partials, SigmaCfgDev{}, nullptr);
}

// state-dependent sigma (A <= 15): 1 + 2A head rows
__global__ void __launch_bounds__(LT) ppo_head_loss_sd_kernel(
    const float* __restrict__ a_last, int Hl, const float* __restrict__ Wh, const float* __restrict__ bh,
    const float* __restrict__ actions, float* __restrict__ old_mu,
    float* __restrict__ old_sigma, const float* __restrict__ old_values_n, const float* __restrict__ returns_n,
    const float* __restrict__ old_neglogp, const float* __restrict__ advs_n, const float* __restrict__ mask,
    int rows_per_chunk, int64_t chunk_stride, int M, int A, LossCfgDev cfg, const float* __restrict__ inv_count_dev,
    float* __restrict__ d_head, float* __restrict__ d_alast, int act_last,
    float* __restrict__ mu_out, float* __restrict__ value_out, float* __restrict__ neglogp_out,
    double* __restrict__ partials, SigmaCfgDev scfg, const float* __restrict__ entropy_coef_dev) {
    ppo_head_loss_body<MAXA_SD, true>(a_last, Hl, Wh, bh, nullptr, actions, old_mu, old_sigma, old_values_n, returns_n, old_neglogp, advs_n,
                                      mask, rows_per_chunk, chunk_stride, M, A, cfg, inv_count_dev, d_head, d_alast, act_last, mu_out,
                                      value_out, neglogp_out, partials, scfg, entropy_coef_dev);
}

__global__ void __launch_bounds__(256) ppo_loss_finalize_kernel(const double* __restrict__ partials, int n_partials, int A,
                                                               const float* __restrict__ entropy_coef_dev,
                                                               float* __restrict__ stats, float* __restrict__ d_logstd, float* __restrict__ kl_out) {
    __shared__ double sm[256];
    const int slots = NSC + A;
    // thread layout: slot = tid % 64 (slots <= 40), lane group = tid / 64 (4 groups) -- fixed order => deterministic
    const int slot = threadIdx.x & 63, grp = threadIdx.x >> 6;
    double s = 0.0;
    if (slot < slots)
        for (int p = grp; p < n_partials; p += 4) s += partials[(int64_t)p * (NSC + MAXA) + slot];
    sm[threadIdx.x] = s;
    __syncthreads();
    if (grp == 0 && slot < slots) {
        const double t = (sm[slot] + sm[64 + slot]) + (sm[128 + slot] + sm[192 + slot]);
        sm[slot] = t;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        stats[B200RL_STAT_ALOSS] = (float)sm[0];
        stats[B200RL_STAT_CLOSS] = (float)sm[1];
        stats[B200RL_STAT_ENTROPY] = (float)sm[2];
        stats[B200RL_STAT_BLOSS] = (float)sm[3];
        stats[B200RL_STAT_KL] = (float)sm[4];
        if (kl_out) *kl_out = (float)sm[4];
        stats[B200RL_STAT_SUMMASK] = (float)sm[5];
        stats[B200RL_STAT_CLIPFRAC] = (float)(sm[6] / fmax(sm[5], 1.0));
    }
    if (threadIdx.x < A) {
        const double ec = (double)__ldg(entropy_coef_dev);
        d_logstd[threadIdx.x] = (float)(sm[NSC + threadIdx.x] - ec * sm[7]);
    }
}

// One launch for the two tiny post-backward steps: blocks [0, gridDim-2] sum the split partials of the flat gradient
// (deterministic, fixed order), the last block finalises the loss partials (stats, d_logstd, KL slot).
__global__ void __launch_bounds__(256) reduce_finalize_kernel(const float* __restrict__ part, float* __restrict__ out, int n, int n_splits,
                                                             int64_t split_stride, const double* __restrict__ partials, int n_partials,
                                                             int A, const float* __restrict__ entropy_coef_dev, float* __restrict__ stats,
                                                             float* __restrict__ d_logstd, float* __restrict__ kl_out) {
    pdl_sync();
    if (blockIdx.x + 1 < gridDim.x) {
        const int i = blockIdx.x * blockDim.x + threadIdx.x;
        if (i >= n) return;
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
        int k = 0;
        for (; k + 3 < n_splits; k += 4) {
            s0 += __ldg(part + (int64_t)k * split_stride + i);
            s1 += __ldg(part + (int64_t)(k + 1) * split_stride + i);
            s2 += __ldg(part + (int64_t)(k + 2) * split_stride + i);
            s3 += __ldg(part + (int64_t)(k + 3) * split_stride + i);
        }
        for (; k < n_splits; ++k) s0 += __ldg(part + (int64_t)k * split_stride + i);
        out[i] = (s0 + s1) + (s2 + s3);
        return;
    }
    __shared__ double sm[256];
    const int slots = NSC + A;
    const int slot = threadIdx.x & 63, grp = threadIdx.x >> 6;
    double s = 0.0;
    if (slot < slots)
        for (int p = grp; p < n_partials; p += 4) s += partials[(int64_t)p * (NSC + MAXA) + slot];
    sm[threadIdx.x] = s;
    __syncthreads();
    if (grp == 0 && slot < slots) sm[slot] = (sm[slot] + sm[64 + slot]) + (sm[128 + slot] + sm[192 + slot]);
    __syncthreads();
    if (threadIdx.x == 0) {
        stats[B200RL_STAT_ALOSS] = (float)sm[0];
        stats[B200RL_STAT_CLOSS] = (float)sm[1];
        stats[B200RL_STAT_ENTROPY] = (float)sm[2];
        stats[B200RL_STAT_BLOSS] = (float)sm[3];
        stats[B200RL_STAT_KL] = (float)sm[4];
        if (kl_out) *kl_out = (float)sm[4];
        stats[B200RL_STAT_SUMMASK] = (float)sm[5];
        stats[B200RL_STAT_CLIPFRAC] = (float)(sm[6] / fmax(sm[5], 1.0));
    }
    if (threadIdx.x < A) {
        const double ec = (double)__ldg(entropy_coef_dev);
        d_logstd[threadIdx.x] = (float)(sm[NSC + threadIdx.x] - ec * sm[7]);
    }
}

// inv_count[i] = 1 / max(sum of mask over minibatch i, 1)   (torch_ext.py:157-170 apply_masks)
__global__ void __launch_bounds__(256) mask_inv_counts_kernel(const float* __restrict__ mask, int H, int N, int envs_per_mb,
                                                             float* __restrict__ inv_count) {
    __shared__ double sm[32];
    const int mb = blockIdx.x;
    const int e0 = mb * envs_per_mb;
    double acc[1] = {0.0};
    for (int i = threadIdx.x; i < H * envs_per_mb; i += blockDim.x) {
        const int t = i / envs_per_mb, e = e0 + (i - t * envs_per_mb);
        acc[0] += (double)__ldg(mask + (int64_t)t * N + e);
    }
    block_sum_d<1>(acc, sm);
    if (threadIdx.x == 0) inv_count[mb] = (float)(1.0 / fmax(acc[0], 1.0));
}

}  // namespace

B200RL_EXPORT int b200rl_ppo_head_loss_f32(const float* a_last, int Hl, const float* W_head, const float* b_head,
                                           const float* logstd, const float* actions, float* old_mu, float* old_sigma,
                                           const float* old_values_n, const float* returns_n, const float* old_neglogp,
                                           const float* advs_n, const float* mask,
                                           int rows_per_chunk, int64_t chunk_stride, int M, int A,
                                           const b200rl_loss_cfg* cfg_host, const float* inv_count_dev,
                                           float* d_head, float* d_alast, int act_last,
                                           float* mu_out, float* value_out, float* neglogp_out,
                                           double* partials, int max_partials, int* n_blocks_out_host, void* stream) {
    if (!a_last || !W_head || !b_head || !logstd || !actions || !old_mu || !old_sigma || !old_values_n || !returns_n ||
        !old_neglogp || !advs_n || !cfg_host || !d_head || !d_alast || !partials)
        return B200RL_EINVAL;
    if (M <= 0 || A <= 0 || A + 1 > MAXA || Hl <= 0 || rows_per_chunk <= 0) return B200RL_EINVAL;
    const int blocks = (M + LT - 1) / LT;
    if (n_blocks_out_host) *n_blocks_out_host = blocks;
    if (blocks > max_partials) return B200RL_EINVAL;
    const size_t smem = sizeof(float) * ((size_t)LT * (Hl + 1) + (size_t)(A + 1) * Hl + (A + 1) + 4 * A + (LT / 32) * (NSC + A));
    if (smem > 200 * 1024) return B200RL_EUNSUPPORTED;
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(ppo_head_loss_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return (int)e;
    }
    LossCfgDev c;
    c.e_clip = cfg_host->e_clip; c.critic_coef = cfg_host->critic_coef; c.bounds_coef = cfg_host->bounds_loss_coef;
    c.has_bounds = cfg_host->has_bounds_loss; c.bound_type = cfg_host->bound_loss_type; c.clip_value = cfg_host->clip_value;
    c.smooth = cfg_host->use_smooth_clamp; c.ppo = cfg_host->ppo;
    c.log_lo = log1pf(-cfg_host->e_clip); c.log_hi = log1pf(cfg_host->e_clip);
    ppo_head_loss_kernel<<<blocks, LT, smem, as_stream(stream)>>>(
        a_last, Hl, W_head, b_head, logstd, actions, old_mu, old_sigma, old_values_n, returns_n, old_neglogp, advs_n, mask,
        rows_per_chunk, chunk_stride, M, A, c, inv_count_dev, d_head, d_alast, act_last, mu_out, value_out, neglogp_out, partials);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_ppo_head_loss_sd_f32(const float* a_last, int Hl, const float* W_head, const float* b_head,
                                              const b200rl_sigma_cfg* sigma_cfg_host, const float* entropy_coef_dev,
                                              const float* actions, float* old_mu, float* old_sigma,
                                              const float* old_values_n, const float* returns_n, const float* old_neglogp,
                                              const float* advs_n, const float* mask,
                                              int rows_per_chunk, int64_t chunk_stride, int M, int A,
                                              const b200rl_loss_cfg* cfg_host, const float* inv_count_dev,
                                              float* d_head, float* d_alast, int act_last,
                                              float* mu_out, float* value_out, float* neglogp_out,
                                              double* partials, int max_partials, int* n_blocks_out_host, void* stream) {
    if (!a_last || !W_head || !b_head || !sigma_cfg_host || !entropy_coef_dev || !actions || !old_mu || !old_sigma || !old_values_n ||
        !returns_n || !old_neglogp || !advs_n || !cfg_host || !d_head || !d_alast || !partials)
        return B200RL_EINVAL;
    if (M <= 0 || A <= 0 || A + 1 > MAXA_SD || Hl <= 0 || rows_per_chunk <= 0) return B200RL_EINVAL;
    if (sigma_cfg_host->parametrization < SIGMA_EXP || sigma_cfg_host->parametrization > SIGMA_LINEAR) return B200RL_EINVAL;
    const int blocks = (M + LT - 1) / LT;
    if (n_blocks_out_host) *n_blocks_out_host = blocks;
    if (blocks > max_partials) return B200RL_EINVAL;
    const int HR = 1 + 2 * A;
    const size_t smem = sizeof(float) * ((size_t)LT * (Hl + 1) + (size_t)HR * Hl + HR + 4 * A + (LT / 32) * (NSC + A));
    if (smem > 200 * 1024) return B200RL_EUNSUPPORTED;
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(ppo_head_loss_sd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return (int)e;
    }
    LossCfgDev c;
    c.e_clip = cfg_host->e_clip; c.critic_coef = cfg_host->critic_coef; c.bounds_coef = cfg_host->bounds_loss_coef;
    c.has_bounds = cfg_host->has_bounds_loss; c.bound_type = cfg_host->bound_loss_type; c.clip_value = cfg_host->clip_value;
    c.smooth = cfg_host->use_smooth_clamp; c.ppo = cfg_host->ppo;
    c.log_lo = log1pf(-cfg_host->e_clip); c.log_hi = log1pf(cfg_host->e_clip);
    ppo_head_loss_sd_kernel<<<blocks, LT, smem, as_stream(stream)>>>(
        a_last, Hl, W_head, b_head, actions, old_mu, old_sigma, old_values_n, returns_n, old_neglogp, advs_n, mask,
        rows_per_chunk, chunk_stride, M, A, c, inv_count_dev, d_head, d_alast, act_last, mu_out, value_out, neglogp_out, partials,
        sigma_cfg_dev(*sigma_cfg_host), entropy_coef_dev);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

#ifdef B200RL_TEST_HOOKS   // test-only host entry point: compiled into tests/libb200rl_testhooks.so (csrc/build.py), not into the product library
// the sigma parametrisation row function (loss_math.cuh sigma_param) over host arrays
B200RL_EXPORT int b200rl_hosttest_sigma_param(const float* raw, int n, const b200rl_sigma_cfg* cfg, float* sigma, float* logstd,
                                              float* dlogstd_draw) {
    const SigmaCfgDev c = sigma_cfg_dev(*cfg);
    for (int i = 0; i < n; ++i) sigma_param(raw[i], c, sigma[i], logstd[i], dlogstd_draw[i]);
    return B200RL_OK;
}
#endif  // B200RL_TEST_HOOKS

B200RL_EXPORT int b200rl_ppo_loss_finalize(const double* partials, int n_partials, int A, const float* entropy_coef_dev,
                                           float* stats, float* d_logstd, float* kl_out, void* stream) {
    if (!partials || !entropy_coef_dev || !stats || !d_logstd || n_partials <= 0 || A <= 0 || A + 1 > MAXA) return B200RL_EINVAL;
    ppo_loss_finalize_kernel<<<1, 256, 0, as_stream(stream)>>>(partials, n_partials, A, entropy_coef_dev, stats, d_logstd, kl_out);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_reduce_finalize(const float* part, float* out, int n, int n_splits, int64_t split_stride,
                                         const double* partials, int n_partials, int A, const float* entropy_coef_dev,
                                         float* stats, float* d_logstd, float* kl_out, void* stream) {
    if (!part || !out || n <= 0 || n_splits <= 0 || !partials || !entropy_coef_dev || !stats || !d_logstd || n_partials <= 0 || A <= 0 ||
        A + 1 > MAXA)
        return B200RL_EINVAL;
    cudaError_t le = launch_k(reduce_finalize_kernel, dim3((n + 255) / 256 + 1), dim3(256), 0, as_stream(stream), part, out, n, n_splits,
                              split_stride, partials, n_partials, A, entropy_coef_dev, stats, d_logstd, kl_out);
    if (le != cudaSuccess) return (int)le;
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_mask_inv_counts_f32(const float* mask, int H, int N, int envs_per_mb, float* inv_count, void* stream) {
    if (!mask || !inv_count || H <= 0 || N <= 0 || envs_per_mb <= 0 || N % envs_per_mb != 0) return B200RL_EINVAL;
    mask_inv_counts_kernel<<<N / envs_per_mb, 256, 0, as_stream(stream)>>>(mask, H, N, envs_per_mb, inv_count);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_loss_partial_stride(void) { return NSC + MAXA; }
