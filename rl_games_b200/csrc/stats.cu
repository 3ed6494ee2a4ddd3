// Running mean/std + batch preparation kernels (HBM-bound scan/reduce work, no tensor cores).
//   prepare_batch  -- a2c_common.py:1586-1660 (prepare_dataset): value normaliser update (values THEN
//                     returns), normalise/clamp, advantage normalisation (unmasked :1634, masked
//                     torch_ext.py:172-191).  Consumes the block partials written by gae_fused_kernel.
//   moments_update -- running_mean_std.py:55-114 training-mode update of the obs normaliser on one
//                     minibatch (rows given as time-major chunks of the arena).
//   normalize      -- running_mean_std.py:104-113 (eval forward / denorm).
// Running statistics are fp64 + int64 count like the reference; batch moments are accumulated in fp64.
#include "common.cuh"

namespace {

__device__ __forceinline__ void chan_merge(double& mean, double& var, double& count_f, double bm, double bv, double n) {
    // running_mean_std.py:55-67
    const double tot = count_f + n;
    const double delta = bm - mean;
    const double new_mean = mean + delta * n / tot;
    const double M2 = var * count_f + bv * n + delta * delta * count_f * n / tot;
    mean = new_mean; var = M2 / tot; count_f = tot;
}

__device__ __forceinline__ float norm_clamp(float x, float mean, float std) {
    const float y = __fdiv_rn(__fsub_rn(x, mean), std);
    return fminf(fmaxf(y, -5.0f), 5.0f);
}

template <bool MASKED>
__global__ void __launch_bounds__(256) prepare_batch_kernel(
    const float* __restrict__ values, const float* __restrict__ returns,
    const float* __restrict__ mask, const double* __restrict__ partials, int n_partials,
    double* vms_mean, double* vms_var, int64_t* vms_count,
    float* __restrict__ old_values_n, float* __restrict__ returns_n, float* __restrict__ advs_n,
    int B, int normalize_value, int normalize_advantage, int freeze_stats) {
    __shared__ double sm[32 * 7];
    double acc[7] = {0, 0, 0, 0, 0, 0, 0};
    for (int p = threadIdx.x; p < n_partials; p += blockDim.x) {
#pragma unroll
        for (int i = 0; i < 7; ++i) acc[i] += partials[(int64_t)p * 8 + i];
    }
    block_sum_d<7>(acc, sm);
    const double n = acc[0];
    // ---- value normaliser (values, then returns) ----
    // Unmasked path (a2c_common.py:1616-1620): `values = vms(values)` updates with the values and normalises
    // them with THAT intermediate state; `returns = vms(returns)` then updates again and uses the final state.
    // Masked path (:1605-1615): both updates first, then both tensors are normalised with the final state.
    double mean = vms_mean[0], var = vms_var[0], cnt = (double)vms_count[0];
    double mean_v = mean, var_v = var;
    if (normalize_value && !freeze_stats && n > 0.0) {
        const double mv = acc[1] / n, vv = fmax(acc[2] / n - mv * mv, 0.0);
        chan_merge(mean, var, cnt, mv, vv, n);
        mean_v = mean; var_v = var;
        const double mr = acc[3] / n, vr = fmax(acc[4] / n - mr * mr, 0.0);
        chan_merge(mean, var, cnt, mr, vr, n);
        if (MASKED) { mean_v = mean; var_v = var; }
    }
    const float mean_f = (float)mean;
    const float std_f = __fsqrt_rn(__fadd_rn((float)var, 1e-5f));
    const float mean_vf = (float)mean_v;
    const float std_vf = __fsqrt_rn(__fadd_rn((float)var_v, 1e-5f));
    // ---- advantage normalisation ----
    float a_mean = 0.f, a_den = 1.f;
    if (normalize_advantage) {
        if (!MASKED) {
            const double m = acc[5] / n;
            const double v = fmax((acc[6] - n * m * m) / (n - 1.0), 0.0);   // torch .std(): unbiased
            a_mean = (float)m; a_den = __fadd_rn((float)sqrt(v), 1e-8f);
        } else {
            // torch_ext.py:182-191 get_mean_var_with_masks: clamped denominators
            const double sm_ = fmax(n, 1.0);
            const double m = acc[5] / sm_;
            const double min_sqr = acc[6] / sm_ - m * m;
            const double v = fmax(min_sqr * sm_ / fmax(sm_ - 1.0, 1.0), 0.0);
            a_mean = (float)m; a_den = __fadd_rn((float)sqrt(v), 1e-8f);
        }
    }
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < B; i += stride) {
        const float v = values[i], r = returns[i];
        const float a = __fsub_rn(r, v);   // advantages = returns - values (a2c_common.py:1598), V == 1
        old_values_n[i] = normalize_value ? norm_clamp(v, mean_vf, std_vf) : v;
        returns_n[i] = normalize_value ? norm_clamp(r, mean_f, std_f) : r;
        advs_n[i] = normalize_advantage ? __fdiv_rn(__fsub_rn(a, a_mean), a_den) : a;
    }
    // stats write-back happens only AFTER every block has read the old state: all blocks read it at the
    // top of the kernel, so block 0 may not overwrite it before the others start.  Use a separate
    // finishing kernel instead (prepare_commit_kernel) -- see host code.
}

// single-thread commit of the value-normaliser state (same arithmetic as above)
__global__ void prepare_commit_kernel(const double* __restrict__ partials, int n_partials,
                                      double* vms_mean, double* vms_var, int64_t* vms_count) {
    __shared__ double sm[32 * 7];
    double acc[7] = {0, 0, 0, 0, 0, 0, 0};
    for (int p = threadIdx.x; p < n_partials; p += blockDim.x) {
#pragma unroll
        for (int i = 0; i < 7; ++i) acc[i] += partials[(int64_t)p * 8 + i];
    }
    block_sum_d<7>(acc, sm);
    if (threadIdx.x == 0) {
        const double n = acc[0];
        if (n > 0.0) {
            double mean = vms_mean[0], var = vms_var[0], cnt = (double)vms_count[0];
            const double mv = acc[1] / n, vv = fmax(acc[2] / n - mv * mv, 0.0);
            chan_merge(mean, var, cnt, mv, vv, n);
            const double mr = acc[3] / n, vr = fmax(acc[4] / n - mr * mr, 0.0);
            chan_merge(mean, var, cnt, mr, vr, n);
            vms_mean[0] = mean; vms_var[0] = var;
            vms_count[0] = vms_count[0] + 2 * (int64_t)llround(n);
        }
    }
}

// ---- EMA advantage normaliser (SURVEY 8a row a11): GeneralizedMovingStats 'mean_std' (moving_mean_std.py:84-150), created with
//      decay = adv_rms_momentum (a2c_common.py:473-475), applied in prepare_dataset (:1622-1632).  The batch moments come from the
//      same partial sums as the plain normalisation (slot 0 = valid rows, 5 = sum adv, 6 = sum adv^2); the state (fp32 mean and
//      mean of squares, int32 step) moves by the same decay whatever the number of valid rows; no valid row = no update.
//      Every block derives the new state from the OLD state + partials (identical arithmetic), a one-block commit kernel stores it.
__device__ __forceinline__ bool adv_ema_next(const double* __restrict__ partials, int n_partials, double* sm, const float* __restrict__ state,
                                             float decay, int training, float& mean, float& sqrs) {
    double acc[3] = {0, 0, 0};
    for (int p = threadIdx.x; p < n_partials; p += blockDim.x) {
        acc[0] += partials[(int64_t)p * 8 + 0]; acc[1] += partials[(int64_t)p * 8 + 5]; acc[2] += partials[(int64_t)p * 8 + 6];
    }
    block_sum_d<3>(acc, sm);
    mean = state[0]; sqrs = state[1];
    const bool upd = training && acc[0] > 0.0;
    if (upd) {
        const float xm = (float)(acc[1] / acc[0]), xs = (float)(acc[2] / acc[0]);
        const float mf = __fsub_rn(1.0f, decay);
        mean = __fadd_rn(__fmul_rn(mean, decay), __fmul_rn(mf, xm));      // mean.mul_(m).add_((1 - m) * x_mean)
        sqrs = __fadd_rn(__fmul_rn(sqrs, decay), __fmul_rn(mf, xs));
    }
    return upd;
}

__global__ void __launch_bounds__(256) adv_ema_normalize_kernel(float* __restrict__ advs, int B, const double* __restrict__ partials,
                                                               int n_partials, const float* __restrict__ state, float decay, int training) {
    __shared__ double sm[32 * 3];
    float mean, sqrs;
    adv_ema_next(partials, n_partials, sm, state, decay, training, mean, sqrs);
    const float var = __fsub_rn(sqrs, __fmul_rn(mean, mean));
    const float stdv = __fsqrt_rn(fmaxf(var, 1e-10f));                    // clamp_min(var, 1 / max^2), max = 1e5, eps = 0
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < B; i += stride)
        advs[i] = fminf(fmaxf(__fdiv_rn(__fsub_rn(advs[i], mean), stdv), -5.0f), 5.0f);
}

__global__ void __launch_bounds__(256) adv_ema_commit_kernel(const double* __restrict__ partials, int n_partials, float* state, int* step,
                                                            float decay, int training) {
    __shared__ double sm[32 * 3];
    float mean, sqrs;
    const bool upd = adv_ema_next(partials, n_partials, sm, state, decay, training, mean, sqrs);
    if (threadIdx.x == 0 && upd) { state[0] = mean; state[1] = sqrs; step[0] = step[0] + 1; }
}

// ---- obs moments: grid = (blocks_per_chunk, n_chunks), 256 threads ---------------------------------
// scratch layout: [n_blocks][2*D] doubles (shifted sum, shifted sum of squares)
__global__ void __launch_bounds__(256) moments_partial_kernel(
    const float* __restrict__ x, int D, int rows_per_chunk, int64_t chunk_stride,
    const double* __restrict__ run_mean, double* __restrict__ scratch, int* counter,
    double* mean, double* var, int64_t* count, float* mean_f32, float* std_f32, float eps, int n_rows_total) {
    extern __shared__ double smd[];   // [G][2][CW]
    const int CW = D <= 32 ? 32 : (D <= 64 ? 64 : (D <= 128 ? 128 : 256));
    const int G = 256 / CW;
    const int c = threadIdx.x % CW, g = threadIdx.x / CW;
    const int bpc = gridDim.x;
    const int rows_per_block = (rows_per_chunk + bpc - 1) / bpc;
    const int r0 = blockIdx.x * rows_per_block;
    const int r1 = min(r0 + rows_per_block, rows_per_chunk);
    const float* base = x + ((int64_t)blockIdx.y * chunk_stride) * D;
    const int blk = blockIdx.y * gridDim.x + blockIdx.x;
    const int n_blocks = gridDim.x * gridDim.y;
    for (int c0 = 0; c0 < D; c0 += CW) {
        const int col = c0 + c;
        double s = 0.0, q = 0.0;
        if (col < D) {
            const float shift = (float)run_mean[col];
            int r = r0 + g;
            // 4 independent loads in flight per thread
            for (; r + 3 * G < r1; r += 4 * G) {
                const float v0 = __ldg(base + (int64_t)r * D + col), v1 = __ldg(base + (int64_t)(r + G) * D + col);
                const float v2 = __ldg(base + (int64_t)(r + 2 * G) * D + col), v3 = __ldg(base + (int64_t)(r + 3 * G) * D + col);
                const double d0 = (double)(v0 - shift), d1 = (double)(v1 - shift), d2 = (double)(v2 - shift), d3 = (double)(v3 - shift);
                s += (d0 + d1) + (d2 + d3);
                q += (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
            }
            for (; r < r1; r += G) {
                const double d0 = (double)(__ldg(base + (int64_t)r * D + col) - shift);
                s += d0; q += d0 * d0;
            }
        }
        smd[(g * 2 + 0) * CW + c] = s;
        smd[(g * 2 + 1) * CW + c] = q;
        __syncthreads();
        if (g == 0 && col < D) {
            double ss = 0.0, qq = 0.0;
            for (int gg = 0; gg < G; ++gg) { ss += smd[(gg * 2 + 0) * CW + c]; qq += smd[(gg * 2 + 1) * CW + c]; }
            scratch[(int64_t)blk * 2 * D + col] = ss;
            scratch[(int64_t)blk * 2 * D + D + col] = qq;
        }
        __syncthreads();
    }
    // ---- last block finalises (fixed order => deterministic) ----
    __shared__ int is_last;
    __threadfence();
    if (threadIdx.x == 0) {
        const int prev = atomicAdd(counter, 1);
        is_last = (prev == n_blocks - 1);
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    const double n = (double)n_rows_total;
    const double cnt0 = (double)count[0];
    for (int col = threadIdx.x; col < D; col += blockDim.x) {
        double ss = 0.0, qq = 0.0;
        for (int b = 0; b < n_blocks; ++b) {
            ss += __ldcg(scratch + (int64_t)b * 2 * D + col);
            qq += __ldcg(scratch + (int64_t)b * 2 * D + D + col);
        }
        const double shift = (double)(float)run_mean[col];
        const double ms = ss / n;
        const double bm = shift + ms;
        const double bv = fmax(qq / n - ms * ms, 0.0);
        double m = mean[col], v = var[col], cf = cnt0;
        chan_merge(m, v, cf, bm, bv, n);
        mean[col] = m; var[col] = v;
        mean_f32[col] = (float)m;
        std_f32[col] = __fsqrt_rn(__fadd_rn((float)v, eps));
    }
    __syncthreads();
    if (threadIdx.x == 0) { count[0] = count[0] + (int64_t)n_rows_total; *counter = 0; }
}

// ---- obs moments, vectorised edition (D % 4 == 0): float4 loads, thread <-> fixed 4 columns ----------------------
// block = RP row-lanes x C4 column-quads (C4 = D/4, RP = 256 / C4 rounded down); grid = (blocks_per_chunk, n_chunks).
// scratch layout identical to moments_partial_kernel: [n_blocks][2*D] doubles (shifted sum, shifted sum of squares).
__global__ void __launch_bounds__(256) moments_partial_v4_kernel(
    const float* __restrict__ x, int D, int rows_per_chunk, int64_t chunk_stride,
    const double* __restrict__ run_mean, double* __restrict__ scratch, int* counter,
    double* mean, double* var, int64_t* count, float* mean_f32, float* std_f32, float eps, int n_rows_total,
    int mb_rows, double* __restrict__ mbmom, float* __restrict__ mb_shift) {
    // per-minibatch mode (mbmom != nullptr): blockIdx.z = minibatch index; this launch only produces the shifted batch
    // sums of every minibatch (obs do not change across mini-epochs, so this runs ONCE per epoch); the Chan merge into the
    // running state happens per minibatch in obs_stats_merge_kernel.
    extern __shared__ double smd[];   // [RP][2*D]
    x += (int64_t)blockIdx.z * mb_rows * D;
    scratch += (int64_t)blockIdx.z * gridDim.x * gridDim.y * 2 * D;
    counter += blockIdx.z;
    const int C4 = D >> 2;
    const int RP = blockDim.x / C4;
    const int tid = threadIdx.x;
    const int rr = tid / C4, c4 = tid - rr * C4;
    const bool active = rr < RP;
    const int bpc = gridDim.x;
    const int rows_per_block = (rows_per_chunk + bpc - 1) / bpc;
    const int r0 = blockIdx.x * rows_per_block, r1 = min(r0 + rows_per_block, rows_per_chunk);
    const float4* base = reinterpret_cast<const float4*>(x + ((int64_t)blockIdx.y * chunk_stride) * D);
    const int blk = blockIdx.y * gridDim.x + blockIdx.x;
    const int n_blocks = gridDim.x * gridDim.y;
    double s[4] = {0, 0, 0, 0}, q[4] = {0, 0, 0, 0};
    if (active) {
        float sh[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) sh[j] = (float)run_mean[c4 * 4 + j];
        int r = r0 + rr;
        for (; r + 3 * RP < r1; r += 4 * RP) {
            float4 v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) v[u] = __ldg(base + (int64_t)(r + u * RP) * C4 + c4);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const double d0 = (double)(v[u].x - sh[0]), d1 = (double)(v[u].y - sh[1]), d2 = (double)(v[u].z - sh[2]), d3 = (double)(v[u].w - sh[3]);
                s[0] += d0; s[1] += d1; s[2] += d2; s[3] += d3;
                q[0] += d0 * d0; q[1] += d1 * d1; q[2] += d2 * d2; q[3] += d3 * d3;
            }
        }
        for (; r < r1; r += RP) {
            const float4 v = __ldg(base + (int64_t)r * C4 + c4);
            const double d0 = (double)(v.x - sh[0]), d1 = (double)(v.y - sh[1]), d2 = (double)(v.z - sh[2]), d3 = (double)(v.w - sh[3]);
            s[0] += d0; s[1] += d1; s[2] += d2; s[3] += d3;
            q[0] += d0 * d0; q[1] += d1 * d1; q[2] += d2 * d2; q[3] += d3 * d3;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) { smd[(size_t)rr * 2 * D + c4 * 4 + j] = s[j]; smd[(size_t)rr * 2 * D + D + c4 * 4 + j] = q[j]; }
    }
    __syncthreads();
    for (int j = tid; j < 2 * D; j += blockDim.x) {
        double a = 0.0;
        for (int g = 0; g < RP; ++g) a += smd[(size_t)g * 2 * D + j];
        scratch[(int64_t)blk * 2 * D + j] = a;
    }
    __shared__ int is_last;
    __threadfence();
    __syncthreads();
    if (tid == 0) is_last = (atomicAdd(counter, 1) == n_blocks - 1);
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    // final reduction over blocks: 2*D columns x NS slices of blocks, fixed order
    const int NS = max(1, (int)blockDim.x / (2 * D));
    __syncthreads();
    for (int idx = tid; idx < NS * 2 * D; idx += blockDim.x) {
        const int j = idx % (2 * D), sl = idx / (2 * D);
        double a = 0.0;
        for (int b = sl; b < n_blocks; b += NS) a += __ldcg(scratch + (int64_t)b * 2 * D + j);
        smd[(size_t)sl * 2 * D + j] = a;
    }
    __syncthreads();
    if (mbmom) {
        for (int j = tid; j < 2 * D; j += blockDim.x) {
            double a = 0.0;
            for (int g = 0; g < NS; ++g) a += smd[(size_t)g * 2 * D + j];
            mbmom[(int64_t)blockIdx.z * 2 * D + j] = a;
        }
        if (blockIdx.z == 0)
            for (int col = tid; col < D; col += blockDim.x) mb_shift[col] = (float)run_mean[col];
        __syncthreads();
        if (tid == 0) *counter = 0;
        return;
    }
    const double n = (double)n_rows_total;
    const double cnt0 = (double)count[0];
    for (int col = tid; col < D; col += blockDim.x) {
        double ss = 0.0, qq = 0.0;
        for (int g = 0; g < NS; ++g) { ss += smd[(size_t)g * 2 * D + col]; qq += smd[(size_t)g * 2 * D + D + col]; }
        const double shift = (double)(float)run_mean[col];
        const double ms = ss / n;
        const double bm = shift + ms;
        const double bv = fmax(qq / n - ms * ms, 0.0);
        double m = mean[col], v = var[col], cf = cnt0;
        chan_merge(m, v, cf, bm, bv, n);
        mean[col] = m; var[col] = v;
        mean_f32[col] = (float)m;
        std_f32[col] = __fsqrt_rn(__fadd_rn((float)v, eps));
    }
    __syncthreads();
    if (tid == 0) { count[0] = count[0] + (int64_t)n_rows_total; *counter = 0; }
}

// moments of an already materialised batch (compat path of prepare_dataset when a caller edited batch_dict)
__global__ void __launch_bounds__(256) batch_moments_kernel(const float* __restrict__ values, const float* __restrict__ returns,
                                                           const float* __restrict__ mask, double* __restrict__ partials, int B) {
    __shared__ double sm[32 * 7];
    double acc[7] = {0, 0, 0, 0, 0, 0, 0};
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < B; i += stride) {
        const float v = values[i], r = returns[i];
        const double w = mask ? (mask[i] != 0.f ? 1.0 : 0.0) : 1.0;
        const double dv = v, dr = r, da = __fsub_rn(r, v);
        acc[0] += w; acc[1] += w * dv; acc[2] += w * dv * dv; acc[3] += w * dr; acc[4] += w * dr * dr;
        acc[5] += w * da; acc[6] += w * da * da;
    }
    block_sum_d<7>(acc, sm);
    if (threadIdx.x == 0) {
        double* p = partials + (int64_t)blockIdx.x * 8;
#pragma unroll
        for (int i = 0; i < 7; ++i) p[i] = acc[i];
        p[7] = 0.0;
    }
}

// per-minibatch Chan merge of precomputed (shifted) batch sums into the running obs statistics
__global__ void obs_stats_merge_kernel(const double* __restrict__ mbmom, const float* __restrict__ mb_shift, int D, int n_rows,
                                       double* mean, double* var, int64_t* count, float* mean_f32, float* std_f32, float eps) {
    const double n = (double)n_rows;
    const double cnt0 = (double)count[0];
    for (int col = threadIdx.x; col < D; col += blockDim.x) {
        const double ms = mbmom[col] / n;
        const double bm = (double)mb_shift[col] + ms;
        const double bv = fmax(mbmom[D + col] / n - ms * ms, 0.0);
        double m = mean[col], v = var[col], cf = cnt0;
        chan_merge(m, v, cf, bm, bv, n);
        mean[col] = m; var[col] = v;
        mean_f32[col] = (float)m;
        std_f32[col] = __fsqrt_rn(__fadd_rn((float)v, eps));
    }
    __syncthreads();
    if (threadIdx.x == 0) count[0] = count[0] + (int64_t)n_rows;
}

__global__ void refresh_f32_kernel(const double* mean, const double* var, float* mean_f32, float* std_f32, float eps, int D) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < D) { mean_f32[c] = (float)mean[c]; std_f32[c] = __fsqrt_rn(__fadd_rn((float)var[c], eps)); }
}

__global__ void __launch_bounds__(256) normalize_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                        const double* __restrict__ mean, const double* __restrict__ var,
                                                        float eps, int64_t total, int D, int denorm) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const int c = (int)(i % D);
        const float m = (float)mean[c];
        const float s = __fsqrt_rn(__fadd_rn((float)var[c], eps));
        const float v = x[i];
        if (denorm) {
            const float cl = fminf(fmaxf(v, -5.0f), 5.0f);
            y[i] = __fadd_rn(__fmul_rn(s, cl), m);
        } else {
            y[i] = norm_clamp(v, m, s);
        }
    }
}

// ---- explained variance of every minibatch (torch_ext.py:204-215, PpoDiagnostics.mini_batch, diagnostics.py:55-62) ----------------
// one 1024-thread block per minibatch, two passes over its rows (sums, then squared deviations from the means) in fp64; masked rows are skipped,
// so whatever they hold contributes nothing.  ev[] = {n, ss_y, ss_dy}: unmasked y = returns (population variances); masked y = the
// VALUES (the reference's get_mean_var_with_masks(y_pred, ...)) with its clamp(min=1) guards and Bessel factor.  var_y = 0 gives
// -inf / NaN, like the reference.
__host__ __device__ inline float expvar_finalize(double n, double ss_y, double ss_dy, int masked) {
    double var_y, var_dy;
    if (masked) {
        const double s = n > 1.0 ? n : 1.0;
        const double bessel = s / (s - 1.0 > 1.0 ? s - 1.0 : 1.0);
        var_y = ss_y / s * bessel;
        var_dy = ss_dy / s * bessel;
    } else {
        var_y = ss_y / n;
        var_dy = ss_dy / n;
    }
    return (float)(1.0 - var_dy / var_y);
}

template <bool MASKED>
__global__ void __launch_bounds__(1024) explained_variance_kernel(const float* __restrict__ values, const float* __restrict__ returns,
                                                                 const float* __restrict__ mask, int rows_per_chunk, int n_chunks,
                                                                 int64_t chunk_stride, int64_t mb_offset, float* __restrict__ out,
                                                                 int64_t out_stride, int n_rep, int64_t rep_stride) {
    __shared__ double sm[32 * 3];
    const int64_t base = (int64_t)blockIdx.x * mb_offset;
    // pass 1: count, sum y, sum (returns - values); rows walked chunk by chunk, coalesced within a chunk
    double acc[3] = {0, 0, 0};
    for (int c = 0; c < n_chunks; ++c) {
        const int64_t rc = base + c * chunk_stride;
#pragma unroll 2
        for (int e = threadIdx.x; e < rows_per_chunk; e += blockDim.x) {
            if (MASKED && mask[rc + e] == 0.f) continue;
            const float v = values[rc + e], ret = returns[rc + e];
            acc[0] += 1.0; acc[1] += (double)(MASKED ? v : ret); acc[2] += (double)__fsub_rn(ret, v);
        }
    }
    block_sum_d<3>(acc, sm);
    const double n = acc[0];
    const double my = n > 0.0 ? acc[1] / n : 0.0, md = n > 0.0 ? acc[2] / n : 0.0;
    // pass 2: squared deviations (the minibatch's rows are L2-resident after pass 1)
    double sq[2] = {0, 0};
    for (int c = 0; c < n_chunks; ++c) {
        const int64_t rc = base + c * chunk_stride;
#pragma unroll 2
        for (int e = threadIdx.x; e < rows_per_chunk; e += blockDim.x) {
            if (MASKED && mask[rc + e] == 0.f) continue;
            const float v = values[rc + e], ret = returns[rc + e];
            const double y = (double)(MASKED ? v : ret) - my, d = (double)__fsub_rn(ret, v) - md;
            sq[0] += y * y; sq[1] += d * d;
        }
    }
    block_sum_d<2>(sq, sm);
    if (threadIdx.x == 0) {
        const float ev = expvar_finalize(n, sq[0], sq[1], MASKED);
        for (int k = 0; k < n_rep; ++k) out[(int64_t)blockIdx.x * out_stride + k * rep_stride] = ev;
    }
}

// ---- obs moments of uint8 frames (x * 1/255, a2c_common.py:972-983): one CTA owns 32 columns over every row -------------------
// block = 32 columns x 8 row lanes; the lanes' shifted sums meet in shared memory in a fixed order, so the merged statistics are
// deterministic without cross-CTA partials (an image row has tens of thousands of columns: per-CTA partials would cost
// n_blocks * 2 * D doubles).  The count moves in moments_u8_count_kernel, after every CTA has read the old one.
__global__ void __launch_bounds__(256) moments_u8_kernel(
    const uint8_t* __restrict__ x, int D, int rows_per_chunk, int n_chunks, int64_t chunk_stride,
    double* mean, double* var, const int64_t* count, float* mean_f32, float* std_f32, float eps) {
    __shared__ double sm[8][2][32];
    const int c = threadIdx.x & 31, g = threadIdx.x >> 5;
    const int col = blockIdx.x * 32 + c;
    double s = 0.0, q = 0.0;
    const float shift = col < D ? (float)mean[col] : 0.f;
    if (col < D) {
        for (int ch = 0; ch < n_chunks; ++ch) {
            const uint8_t* base = x + (int64_t)ch * chunk_stride * D + col;
            for (int r = g; r < rows_per_chunk; r += 8) {
                const double d = (double)__fsub_rn(__fdiv_rn((float)__ldg(base + (int64_t)r * D), 255.0f), shift);
                s += d; q += d * d;
            }
        }
    }
    sm[g][0][c] = s;
    sm[g][1][c] = q;
    __syncthreads();
    if (g != 0 || col >= D) return;
    double ss = 0.0, qq = 0.0;
    for (int gg = 0; gg < 8; ++gg) { ss += sm[gg][0][c]; qq += sm[gg][1][c]; }
    const double n = (double)rows_per_chunk * n_chunks;
    const double ms = ss / n;
    const double bm = (double)shift + ms;
    const double bv = fmax(qq / n - ms * ms, 0.0);
    double m = mean[col], v = var[col], cf = (double)count[0];
    chan_merge(m, v, cf, bm, bv, n);
    mean[col] = m; var[col] = v;
    mean_f32[col] = (float)m;
    std_f32[col] = __fsqrt_rn(__fadd_rn((float)v, eps));
}

__global__ void moments_u8_count_kernel(int64_t* count, int64_t n) { count[0] += n; }

}  // namespace

#ifdef B200RL_TEST_HOOKS   // test-only host entry point: compiled into tests/libb200rl_testhooks.so (csrc/build.py), not into the product library
// the explained-variance finalisation (expvar_finalize) over host arrays of (n, ss_y, ss_dy) triples
B200RL_EXPORT int b200rl_hosttest_expvar_finalize(const double* sums, int count, int masked, float* out) {
    for (int i = 0; i < count; ++i) out[i] = expvar_finalize(sums[3 * i], sums[3 * i + 1], sums[3 * i + 2], masked);
    return B200RL_OK;
}
#endif  // B200RL_TEST_HOOKS

B200RL_EXPORT int b200rl_explained_variance_f32(const float* values, const float* returns, const float* mask, int rows_per_chunk,
                                                int n_chunks, int64_t chunk_stride, int n_mb, int64_t mb_offset, float* out,
                                                int64_t out_stride, int n_rep, int64_t rep_stride, void* stream) {
    if (!values || !returns || !out || rows_per_chunk <= 0 || n_chunks <= 0 || n_mb <= 0 || n_rep <= 0) return B200RL_EINVAL;
    cudaStream_t s = as_stream(stream);
    if (mask)
        explained_variance_kernel<true><<<n_mb, 1024, 0, s>>>(values, returns, mask, rows_per_chunk, n_chunks, chunk_stride, mb_offset, out,
                                                             out_stride, n_rep, rep_stride);
    else
        explained_variance_kernel<false><<<n_mb, 1024, 0, s>>>(values, returns, mask, rows_per_chunk, n_chunks, chunk_stride, mb_offset, out,
                                                              out_stride, n_rep, rep_stride);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_prepare_batch_f32(const float* values, const float* returns, const float* mask,
                                           const double* partials, int n_partials,
                                           double* vms_mean, double* vms_var, int64_t* vms_count,
                                           float* old_values_n, float* returns_n, float* advs_n,
                                           int B, int normalize_value, int normalize_advantage, int freeze_stats,
                                           void* stream) {
    if (!values || !returns || !partials || !old_values_n || !returns_n || !advs_n || B <= 0 || n_partials <= 0)
        return B200RL_EINVAL;
    if (normalize_value && (!vms_mean || !vms_var || !vms_count)) return B200RL_EINVAL;
    cudaStream_t s = as_stream(stream);
    const int threads = 256;
    int blocks = (B + threads * 4 - 1) / (threads * 4);
    if (blocks > 132 * 4) blocks = 132 * 4;
    if (blocks < 1) blocks = 1;
    if (!normalize_value) {
        // kernel still dereferences vms_* pointers: require them (agent always allocates them)
        if (!vms_mean || !vms_var || !vms_count) return B200RL_EINVAL;
    }
    if (mask)
        prepare_batch_kernel<true><<<blocks, threads, 0, s>>>(values, returns, mask, partials, n_partials, vms_mean, vms_var,
                                                              vms_count, old_values_n, returns_n, advs_n, B, normalize_value,
                                                              normalize_advantage, freeze_stats);
    else
        prepare_batch_kernel<false><<<blocks, threads, 0, s>>>(values, returns, mask, partials, n_partials, vms_mean, vms_var,
                                                               vms_count, old_values_n, returns_n, advs_n, B, normalize_value,
                                                               normalize_advantage, freeze_stats);
    B200RL_LAUNCH_CHECK();
    if (normalize_value && !freeze_stats) {
        prepare_commit_kernel<<<1, 256, 0, s>>>(partials, n_partials, vms_mean, vms_var, vms_count);
        B200RL_LAUNCH_CHECK();
    }
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_adv_ema_normalize_f32(float* advs, int B, const double* partials, int n_partials, float* ema_state,
                                               int* ema_step, float decay, int training, void* stream) {
    if (!advs || !partials || !ema_state || !ema_step || B <= 0 || n_partials <= 0 || !(decay >= 0.0f && decay <= 1.0f)) return B200RL_EINVAL;
    cudaStream_t s = as_stream(stream);
    int blocks = (B + 256 * 8 - 1) / (256 * 8);
    if (blocks > 132 * 4) blocks = 132 * 4;
    adv_ema_normalize_kernel<<<blocks, 256, 0, s>>>(advs, B, partials, n_partials, ema_state, decay, training);
    B200RL_LAUNCH_CHECK();
    if (training) {
        adv_ema_commit_kernel<<<1, 256, 0, s>>>(partials, n_partials, ema_state, ema_step, decay, training);
        B200RL_LAUNCH_CHECK();
    }
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_batch_moments_f64(const float* values, const float* returns, const float* mask, double* partials,
                                           int max_partials, int B, int* n_blocks_out_host, void* stream) {
    if (!values || !returns || !partials || B <= 0 || max_partials <= 0) return B200RL_EINVAL;
    int blocks = (B + 256 * 8 - 1) / (256 * 8);
    if (blocks > max_partials) blocks = max_partials;
    if (blocks > 132 * 4) blocks = 132 * 4;
    if (n_blocks_out_host) *n_blocks_out_host = blocks;
    batch_moments_kernel<<<blocks, 256, 0, as_stream(stream)>>>(values, returns, mask, partials, B);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_moments_update_f64(const float* x, int D, int rows_per_chunk, int n_chunks,
                                            int64_t chunk_stride, double* mean, double* var, int64_t* count,
                                            float* mean_f32, float* std_f32, float eps,
                                            double* scratch, int scratch_blocks, int* counter, void* stream) {
    if (!x || !mean || !var || !count || !mean_f32 || !std_f32 || !scratch || !counter) return B200RL_EINVAL;
    if (D <= 0 || rows_per_chunk <= 0 || n_chunks <= 0) return B200RL_EINVAL;
    if ((D & 3) == 0 && D <= 512 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 && ((chunk_stride * D) & 3) == 0) {
        const int C4 = D / 4;
        const int threads = C4 >= 256 ? 256 : (256 / C4) * C4;
        const int RP = threads / C4;
        if (RP >= 1 && threads >= 2 * D / 4) {
            int bpc2 = 132 / n_chunks;                                // <= 1 CTA per SM in total (single wave)
            const int max_bpc2 = (rows_per_chunk + 4 * RP - 1) / (4 * RP);
            if (bpc2 > max_bpc2) bpc2 = max_bpc2;
            if (bpc2 < 1) bpc2 = 1;
            while (bpc2 * n_chunks > scratch_blocks && bpc2 > 1) --bpc2;
            if (bpc2 * n_chunks > scratch_blocks) return B200RL_EINVAL;
            const int NS = threads / (2 * D) > 1 ? threads / (2 * D) : 1;
            const size_t smem2 = sizeof(double) * 2 * D * (size_t)(RP > NS ? RP : NS);
            if (smem2 <= 48 * 1024) {
                dim3 grid2(bpc2, n_chunks);
                moments_partial_v4_kernel<<<grid2, threads, smem2, as_stream(stream)>>>(x, D, rows_per_chunk, chunk_stride, mean, scratch,
                                                                                     counter, mean, var, count, mean_f32, std_f32, eps,
                                                                                     rows_per_chunk * n_chunks, 0, nullptr, nullptr);
                B200RL_LAUNCH_CHECK();
                return B200RL_OK;
            }
        }
    }
    int bpc = (132 * 4 + n_chunks - 1) / n_chunks;            // ~4 CTAs per SM in total
    const int max_bpc = (rows_per_chunk + 31) / 32;           // >= 32 rows per block
    if (bpc > max_bpc) bpc = max_bpc;
    if (bpc < 1) bpc = 1;
    while (bpc * n_chunks > scratch_blocks && bpc > 1) --bpc;
    if (bpc * n_chunks > scratch_blocks) return B200RL_EINVAL;
    const int CW = D <= 32 ? 32 : (D <= 64 ? 64 : (D <= 128 ? 128 : 256));
    const int G = 256 / CW;
    const size_t smem = (size_t)G * 2 * CW * sizeof(double);
    dim3 grid(bpc, n_chunks);
    moments_partial_kernel<<<grid, 256, smem, as_stream(stream)>>>(x, D, rows_per_chunk, chunk_stride, mean, scratch, counter,
                                                                   mean, var, count, mean_f32, std_f32, eps,
                                                                   rows_per_chunk * n_chunks);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_moments_update_u8_f64(const uint8_t* x, int D, int rows_per_chunk, int n_chunks, int64_t chunk_stride,
                                               double* mean, double* var, int64_t* count, float* mean_f32, float* std_f32, float eps,
                                               void* stream) {
    if (!x || !mean || !var || !count || !mean_f32 || !std_f32 || D <= 0 || rows_per_chunk <= 0 || n_chunks <= 0) return B200RL_EINVAL;
    if (n_chunks > 1 && chunk_stride < rows_per_chunk) return B200RL_EINVAL;
    cudaStream_t s = as_stream(stream);
    moments_u8_kernel<<<(D + 31) / 32, 256, 0, s>>>(x, D, rows_per_chunk, n_chunks, chunk_stride, mean, var, count, mean_f32, std_f32, eps);
    B200RL_LAUNCH_CHECK();
    moments_u8_count_kernel<<<1, 1, 0, s>>>(count, (int64_t)rows_per_chunk * n_chunks);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_obs_mb_moments_f64(const float* x, int D, int H, int N, int envs_per_mb, const double* run_mean,
                                            double* mbmom, float* mb_shift, double* scratch, int scratch_blocks, int* counters,
                                            void* stream) {
    if (!x || !run_mean || !mbmom || !mb_shift || !scratch || !counters || D <= 0 || H <= 0 || N <= 0 || envs_per_mb <= 0 ||
        N % envs_per_mb != 0)
        return B200RL_EINVAL;
    if ((D & 3) != 0 || D > 512 || (reinterpret_cast<uintptr_t>(x) & 15) != 0) return B200RL_EUNSUPPORTED;
    const int n_mb = N / envs_per_mb;
    const int C4 = D / 4;
    const int threads = C4 >= 256 ? 256 : (256 / C4) * C4;
    const int RP = threads / C4;
    int bpc = (132 * 2) / (H * n_mb);
    const int max_bpc = (envs_per_mb + 4 * RP - 1) / (4 * RP);
    if (bpc > max_bpc) bpc = max_bpc;
    if (bpc < 1) bpc = 1;
    while ((int64_t)bpc * H * n_mb > scratch_blocks && bpc > 1) --bpc;
    if ((int64_t)bpc * H * n_mb > scratch_blocks) return B200RL_EINVAL;
    const int NS = threads / (2 * D) > 1 ? threads / (2 * D) : 1;
    const size_t smem = sizeof(double) * 2 * D * (size_t)(RP > NS ? RP : NS);
    if (smem > 48 * 1024) return B200RL_EUNSUPPORTED;
    dim3 grid(bpc, H, n_mb);
    moments_partial_v4_kernel<<<grid, threads, smem, as_stream(stream)>>>(x, D, envs_per_mb, (int64_t)N, run_mean, scratch, counters, nullptr,
                                                                         nullptr, nullptr, nullptr, nullptr, 0.f, envs_per_mb * H,
                                                                         envs_per_mb, mbmom, mb_shift);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_obs_stats_merge_f64(const double* mbmom_i, const float* mb_shift, int D, int n_rows, double* mean, double* var,
                                             int64_t* count, float* mean_f32, float* std_f32, float eps, void* stream) {
    if (!mbmom_i || !mb_shift || !mean || !var || !count || !mean_f32 || !std_f32 || D <= 0 || n_rows <= 0) return B200RL_EINVAL;
    obs_stats_merge_kernel<<<1, 128, 0, as_stream(stream)>>>(mbmom_i, mb_shift, D, n_rows, mean, var, count, mean_f32, std_f32, eps);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_refresh_norm_f32(const double* mean, const double* var, float* mean_f32, float* std_f32,
                                          float eps, int D, void* stream) {
    if (!mean || !var || !mean_f32 || !std_f32 || D <= 0) return B200RL_EINVAL;
    refresh_f32_kernel<<<(D + 127) / 128, 128, 0, as_stream(stream)>>>(mean, var, mean_f32, std_f32, eps, D);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_normalize_f32(const float* x, float* y, const double* mean, const double* var, float eps,
                                       int64_t rows, int D, int denorm, void* stream) {
    if (!x || !y || !mean || !var || rows < 0 || D <= 0) return B200RL_EINVAL;
    if (rows == 0) return B200RL_OK;
    const int64_t total = rows * D;
    int64_t blocks = (total + 256 * 4 - 1) / (256 * 4);
    if (blocks > 132 * 8) blocks = 132 * 8;
    normalize_kernel<<<(unsigned)blocks, 256, 0, as_stream(stream)>>>(x, y, mean, var, eps, total, D, denorm);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}
