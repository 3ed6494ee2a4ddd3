// fp32 (CUDA-core) 2-D convolutions of the image trunk: network_builder.py:161-181 (_build_cnn2d, plain conv2d) and its autograd.
// Implicit GEMM: no im2col is materialised; each tile loader computes the input pixel of its (row, k) pair.
//   fwd  : Y[m, co, p]  = act( b[co] + sum_k X[m](ci, oh*s+kh-pad, ow*s+kw-pad) . W[co, k] )       k = (ci, kh, kw), p = (oh, ow)
//   dgrad: dX[m, ci, q] = act'(A_prev[m, ci, q]) * sum_{co, kh, kw} dY[m, co, (ih+pad-kh)/s, (iw+pad-kw)/s] . W[co, ci, kh, kw]
//          (a gather over the output pixels that read input pixel q: deterministic, no atomics)
//   wgrad: dWp[s][co, k] = sum_{rows of split s} dY[row, co] . X_col[row, k] ; dbp[s][co] = colsum   (row = (m, oh, ow))
// Activations and gradients are dense NCHW rows ([M, C, H, W], PyTorch's flatten order); the first layer reads the observation arena
// in its chunked row order, uint8 (scaled by 1/255, a2c_common.py:972-983) or fp32, NHWC (permute_input, the default) or NCHW, with the
// optional running normaliser of the flat observation (models.py:54) applied per element of the env's own layout, before zero padding.
// Tiling is the fp32 MLP kernels' (mlp_simt.cu): 128x64 block tile, 8x4 per thread, BK = 16, operands staged in shared memory.
#include "common.cuh"

namespace {

constexpr int BM = 128, BN = 64, BK = 16, NT = 256;

struct Geo {
    int C, H, W, Cout, KH, KW, s, pad, Ho, Wo;
};

template <typename T>
__device__ __forceinline__ float to_f32(T v);
template <>
__device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <>
__device__ __forceinline__ float to_f32<uint8_t>(uint8_t v) { return __fdiv_rn((float)v, 255.0f); }   // obs.float() / 255.0

// element (ci, ih, iw) of one input row, zero outside the image
template <typename T, bool NHWC>
__device__ __forceinline__ float load_in(const T* __restrict__ row, int ci, int ih, int iw, const Geo& g,
                                         const float* __restrict__ nm, const float* __restrict__ ns) {
    if (ih < 0 || ih >= g.H || iw < 0 || iw >= g.W) return 0.f;
    const int e = NHWC ? (ih * g.W + iw) * g.C + ci : (ci * g.H + ih) * g.W + iw;
    float v = to_f32<T>(__ldg(row + e));
    if (nm) {
        v = __fdiv_rn(__fsub_rn(v, __ldg(nm + e)), __ldg(ns + e));
        v = fminf(fmaxf(v, -5.0f), 5.0f);
    }
    return v;
}

// ---------------- forward: rows = (m, oh, ow), cols = co, reduction k = (ci, kh, kw) ----------------
template <typename T, bool NHWC>
__global__ void __launch_bounds__(NT) conv2d_fwd_kernel(
    const T* __restrict__ X, int rows_per_chunk, int64_t chunk_stride, int64_t x_ld,
    const float* __restrict__ nm, const float* __restrict__ ns,
    const float* __restrict__ Wt, const float* __restrict__ bias, float* __restrict__ Y, int M, Geo g, int act) {
    __shared__ float As[BK][BM + 4];
    __shared__ float Bs[BK][BN + 4];
    const int tid = threadIdx.x;
    const int HWo = g.Ho * g.Wo, KHW = g.KH * g.KW, K = g.C * KHW;
    const int64_t P = (int64_t)M * HWo;
    const int64_t p0 = (int64_t)blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;
    const int ty = tid / 16, tx = tid % 16;
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    // A loader: one output pixel per thread (consecutive threads, consecutive pixels), 8 consecutive k
    const int a_row = tid % BM, a_k = (tid / BM) * 8;
    const int b_row = tid >> 2, b_k = (tid & 3) * 4;
    const int64_t gp = p0 + a_row;
    const bool pv = gp < P;
    int ih0 = 0, iw0 = 0;
    const T* row = X;
    if (pv) {
        const int m = (int)(gp / HWo), pix = (int)(gp - (int64_t)m * HWo);
        const int oh = pix / g.Wo, ow = pix - oh * g.Wo;
        ih0 = oh * g.s - g.pad; iw0 = ow * g.s - g.pad;
        row = X + chunk_row(m, rows_per_chunk, chunk_stride) * x_ld;
    }
    for (int k0 = 0; k0 < K; k0 += BK) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int k = k0 + a_k + i;
            float v = 0.f;
            if (pv && k < K) {
                const int ci = k / KHW, r = k - ci * KHW, kh = r / g.KW, kw = r - kh * g.KW;
                v = load_in<T, NHWC>(row, ci, ih0 + kh, iw0 + kw, g, nm, ns);
            }
            As[a_k + i][a_row] = v;
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int k = k0 + b_k + i, n = n0 + b_row;
            Bs[b_k + i][b_row] = (n < g.Cout && k < K) ? __ldg(Wt + (int64_t)n * K + k) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float a[8], b[4];
            *(float4*)&a[0] = *(const float4*)&As[k][ty * 8];
            *(float4*)&a[4] = *(const float4*)&As[k][ty * 8 + 4];
            *(float4*)&b[0] = *(const float4*)&Bs[k][tx * 4];
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int64_t p = p0 + ty * 8 + i;
        if (p >= P) continue;
        const int64_t m = p / HWo;
        const int pix = (int)(p - m * HWo);
        float* y = Y + m * g.Cout * HWo + pix;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n < g.Cout) y[(int64_t)n * HWo] = act_fwd(acc[i][j] + (bias ? __ldg(bias + n) : 0.f), act);
        }
    }
}

// ---------------- dgrad: rows = input pixels (m, ih, iw), cols = ci, reduction r = (co, kh, kw) ----------------
__global__ void __launch_bounds__(NT) conv2d_dgrad_kernel(
    const float* __restrict__ dY, const float* __restrict__ Wt, const float* __restrict__ A_prev, float* __restrict__ dX,
    int M, Geo g, int act_prev) {
    __shared__ float As[BK][BM + 4];   // gathered dY tile [r][row]
    __shared__ float Bs[BK][BN + 4];   // W tile [r][ci]
    const int tid = threadIdx.x;
    const int HW = g.H * g.W, HWo = g.Ho * g.Wo, KHW = g.KH * g.KW, R = g.Cout * KHW;
    const int64_t P = (int64_t)M * HW;
    const int64_t p0 = (int64_t)blockIdx.x * BM;
    const int c0 = blockIdx.y * BN;
    const int ty = tid / 16, tx = tid % 16;
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    const int a_row = tid % BM, a_r = (tid / BM) * 8;
    const int b_r = tid >> 4, b_c = (tid & 15) * 4;
    const int64_t gp = p0 + a_row;
    const bool pv = gp < P;
    int ihp = 0, iwp = 0;
    const float* dy = dY;
    if (pv) {
        const int m = (int)(gp / HW), q = (int)(gp - (int64_t)m * HW);
        const int ih = q / g.W;
        ihp = ih + g.pad; iwp = q - ih * g.W + g.pad;
        dy = dY + (int64_t)m * g.Cout * HWo;
    }
    for (int r0 = 0; r0 < R; r0 += BK) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int r = r0 + a_r + i;
            float v = 0.f;
            if (pv && r < R) {
                const int co = r / KHW, rr = r - co * KHW, kh = rr / g.KW, kw = rr - kh * g.KW;
                const int th = ihp - kh, tw = iwp - kw;
                if (th >= 0 && tw >= 0) {
                    const int oh = th / g.s, ow = tw / g.s;
                    if (oh * g.s == th && ow * g.s == tw && oh < g.Ho && ow < g.Wo) v = __ldg(dy + (int64_t)co * HWo + oh * g.Wo + ow);
                }
            }
            As[a_r + i][a_row] = v;
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int r = r0 + b_r, ci = c0 + b_c + i;
            float w = 0.f;
            if (r < R && ci < g.C) {
                const int co = r / KHW, rr = r - co * KHW;
                w = __ldg(Wt + ((int64_t)co * g.C + ci) * KHW + rr);
            }
            Bs[b_r][b_c + i] = w;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float a[8], b[4];
            *(float4*)&a[0] = *(const float4*)&As[k][ty * 8];
            *(float4*)&a[4] = *(const float4*)&As[k][ty * 8 + 4];
            *(float4*)&b[0] = *(const float4*)&Bs[k][tx * 4];
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int64_t p = p0 + ty * 8 + i;
        if (p >= P) continue;
        const int64_t m = p / HW;
        const int q = (int)(p - m * HW);
        const int64_t base = m * g.C * HW + q;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int ci = c0 + tx * 4 + j;
            if (ci < g.C) {
                const int64_t o = base + (int64_t)ci * HW;
                const float d = A_prev ? act_bwd_from_out(__ldg(A_prev + o), act_prev) : 1.f;
                dX[o] = acc[i][j] * d;
            }
        }
    }
}

// ---------------- wgrad: 64 (co) x 64 (k) block tile, 4x4 per thread, rows of split s in slabs of 16 ----------------
template <typename T, bool NHWC>
__global__ void __launch_bounds__(NT) conv2d_wgrad_kernel(
    const float* __restrict__ dY, const T* __restrict__ X, int rows_per_chunk, int64_t chunk_stride, int64_t x_ld,
    const float* __restrict__ nm, const float* __restrict__ ns, float* __restrict__ dWp, float* __restrict__ dbp,
    int M, Geo g, int64_t rows_per_split, int64_t split_stride) {
    __shared__ float As[BK][64 + 4];   // dY slab [row][co]
    __shared__ float Bs[BK][64 + 4];   // X_col slab [row][k]
    const int tid = threadIdx.x;
    const int HWo = g.Ho * g.Wo, KHW = g.KH * g.KW, K = g.C * KHW;
    const int n0 = blockIdx.x * 64, k0 = blockIdx.y * 64, s = blockIdx.z;
    const int ty = tid / 16, tx = tid % 16;
    const int64_t P = (int64_t)M * HWo;
    const int64_t pbeg = (int64_t)s * rows_per_split, pend = min(pbeg + rows_per_split, P);
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    float bsum = 0.f;
    const int l_m = tid >> 4, l_c = (tid & 15) * 4;
    // the k columns this thread stages never change: decompose them once
    int kci[4], kkh[4], kkw[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int k = k0 + l_c + i;
        kci[i] = k / KHW;
        const int r = k - kci[i] * KHW;
        kkh[i] = r / g.KW; kkw[i] = r - kkh[i] * g.KW;
    }
    for (int64_t pp = pbeg; pp < pend; pp += BK) {
        const int64_t p = pp + l_m;
        const bool mv = p < pend;
        int m = 0, pix = 0, ih0 = 0, iw0 = 0;
        if (mv) {
            m = (int)(p / HWo); pix = (int)(p - (int64_t)m * HWo);
            const int oh = pix / g.Wo, ow = pix - oh * g.Wo;
            ih0 = oh * g.s - g.pad; iw0 = ow * g.s - g.pad;
        }
        const float* dy = dY + (int64_t)m * g.Cout * HWo + pix;
        const T* row = X + (mv ? chunk_row(m, rows_per_chunk, chunk_stride) * x_ld : 0);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int n = n0 + l_c + i, k = k0 + l_c + i;
            As[l_m][l_c + i] = (mv && n < g.Cout) ? __ldg(dy + (int64_t)n * HWo) : 0.f;
            Bs[l_m][l_c + i] = (mv && k < K) ? load_in<T, NHWC>(row, kci[i], ih0 + kkh[i], iw0 + kkw[i], g, nm, ns) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < BK; ++r) {
            float a[4], b[4];
            *(float4*)&a[0] = *(const float4*)&As[r][ty * 4];
            *(float4*)&b[0] = *(const float4*)&Bs[r][tx * 4];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (blockIdx.y == 0 && tid < 64) {
#pragma unroll
            for (int r = 0; r < BK; ++r) bsum += As[r][tid];
        }
        __syncthreads();
    }
    float* out = dWp + (int64_t)s * split_stride;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int n = n0 + ty * 4 + i;
        if (n >= g.Cout) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k = k0 + tx * 4 + j;
            if (k < K) out[(int64_t)n * K + k] = acc[i][j];
        }
    }
    if (dbp && blockIdx.y == 0 && tid < 64 && n0 + tid < g.Cout) dbp[(int64_t)s * split_stride + n0 + tid] = bsum;
}

// geometry check shared by the entry points: B200RL_OK and the output size, or B200RL_EINVAL
int make_geo(Geo& g, int C, int H, int W, int Cout, int KH, int KW, int stride, int pad) {
    if (C <= 0 || H <= 0 || W <= 0 || Cout <= 0 || KH <= 0 || KW <= 0 || stride <= 0 || pad < 0) return B200RL_EINVAL;
    if (H + 2 * pad < KH || W + 2 * pad < KW) return B200RL_EINVAL;
    g = Geo{C, H, W, Cout, KH, KW, stride, pad, (H + 2 * pad - KH) / stride + 1, (W + 2 * pad - KW) / stride + 1};
    // every index the kernels form stays in int32 per row and in int64 across rows
    if ((int64_t)C * H * W >= (1ll << 31) || (int64_t)Cout * g.Ho * g.Wo >= (1ll << 31) || (int64_t)C * KH * KW >= (1ll << 31))
        return B200RL_EINVAL;
    return B200RL_OK;
}

}  // namespace

B200RL_EXPORT int b200rl_conv2d_fwd_f32(const void* X, int x_u8, int x_nhwc, int rows_per_chunk, int64_t chunk_stride, int64_t x_ld,
                                        const float* norm_mean, const float* norm_std, const float* W, const float* b, float* Y,
                                        int M, int C, int H, int Wd, int Cout, int KH, int KW, int stride, int pad, int act,
                                        void* stream) {
    Geo g;
    if (!X || !W || !Y || M <= 0 || rows_per_chunk <= 0 || make_geo(g, C, H, Wd, Cout, KH, KW, stride, pad) != B200RL_OK)
        return B200RL_EINVAL;
    if ((norm_mean == nullptr) != (norm_std == nullptr) || x_ld < (int64_t)C * H * Wd) return B200RL_EINVAL;
    const int64_t P = (int64_t)M * g.Ho * g.Wo;
    if ((P + BM - 1) / BM >= (1ll << 31)) return B200RL_EINVAL;
    dim3 grid((unsigned)((P + BM - 1) / BM), (Cout + BN - 1) / BN);
    cudaStream_t s = as_stream(stream);
    if (x_u8) {
        const uint8_t* x = static_cast<const uint8_t*>(X);
        if (x_nhwc) conv2d_fwd_kernel<uint8_t, true><<<grid, NT, 0, s>>>(x, rows_per_chunk, chunk_stride, x_ld, norm_mean, norm_std, W, b, Y, M, g, act);
        else conv2d_fwd_kernel<uint8_t, false><<<grid, NT, 0, s>>>(x, rows_per_chunk, chunk_stride, x_ld, norm_mean, norm_std, W, b, Y, M, g, act);
    } else {
        const float* x = static_cast<const float*>(X);
        if (x_nhwc) conv2d_fwd_kernel<float, true><<<grid, NT, 0, s>>>(x, rows_per_chunk, chunk_stride, x_ld, norm_mean, norm_std, W, b, Y, M, g, act);
        else conv2d_fwd_kernel<float, false><<<grid, NT, 0, s>>>(x, rows_per_chunk, chunk_stride, x_ld, norm_mean, norm_std, W, b, Y, M, g, act);
    }
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_conv2d_bwd_data_f32(const float* dY, const float* W, const float* A_prev, float* dX, int M, int C, int H, int Wd,
                                             int Cout, int KH, int KW, int stride, int pad, int act_prev, void* stream) {
    Geo g;
    if (!dY || !W || !dX || M <= 0 || make_geo(g, C, H, Wd, Cout, KH, KW, stride, pad) != B200RL_OK) return B200RL_EINVAL;
    const int64_t P = (int64_t)M * H * Wd;
    if ((P + BM - 1) / BM >= (1ll << 31)) return B200RL_EINVAL;
    dim3 grid((unsigned)((P + BM - 1) / BM), (C + BN - 1) / BN);
    conv2d_dgrad_kernel<<<grid, NT, 0, as_stream(stream)>>>(dY, W, A_prev, dX, M, g, act_prev);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_conv2d_bwd_weight_f32(const float* dY, const void* X, int x_u8, int x_nhwc, int rows_per_chunk,
                                               int64_t chunk_stride, int64_t x_ld, const float* norm_mean, const float* norm_std,
                                               float* dW_part, float* db_part, int64_t split_stride, int M, int C, int H, int Wd,
                                               int Cout, int KH, int KW, int stride, int pad, int n_splits, void* stream) {
    Geo g;
    if (!dY || !X || !dW_part || M <= 0 || rows_per_chunk <= 0 || n_splits <= 0 || n_splits > 65535 ||
        make_geo(g, C, H, Wd, Cout, KH, KW, stride, pad) != B200RL_OK)
        return B200RL_EINVAL;
    if ((norm_mean == nullptr) != (norm_std == nullptr) || x_ld < (int64_t)C * H * Wd) return B200RL_EINVAL;
    const int K = C * KH * KW;
    if (n_splits > 1 && split_stride < (int64_t)Cout * K) return B200RL_EINVAL;
    const int64_t P = (int64_t)M * g.Ho * g.Wo;
    int64_t rps = (P + n_splits - 1) / n_splits;
    rps = ((rps + BK - 1) / BK) * BK;          // splits past the last row write zeros, which the reduction expects
    dim3 grid((Cout + 63) / 64, (K + 63) / 64, n_splits);
    cudaStream_t s = as_stream(stream);
    if (x_u8) {
        const uint8_t* x = static_cast<const uint8_t*>(X);
        if (x_nhwc) conv2d_wgrad_kernel<uint8_t, true><<<grid, NT, 0, s>>>(dY, x, rows_per_chunk, chunk_stride, x_ld, norm_mean, norm_std, dW_part, db_part, M, g, rps, split_stride);
        else conv2d_wgrad_kernel<uint8_t, false><<<grid, NT, 0, s>>>(dY, x, rows_per_chunk, chunk_stride, x_ld, norm_mean, norm_std, dW_part, db_part, M, g, rps, split_stride);
    } else {
        const float* x = static_cast<const float*>(X);
        if (x_nhwc) conv2d_wgrad_kernel<float, true><<<grid, NT, 0, s>>>(dY, x, rows_per_chunk, chunk_stride, x_ld, norm_mean, norm_std, dW_part, db_part, M, g, rps, split_stride);
        else conv2d_wgrad_kernel<float, false><<<grid, NT, 0, s>>>(dY, x, rows_per_chunk, chunk_stride, x_ld, norm_mean, norm_std, dW_part, db_part, M, g, rps, split_stride);
    }
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}
