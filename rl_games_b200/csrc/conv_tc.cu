// bf16 tensor-core (wgmma) 2-D convolutions of the image trunk: the `mixed_precision: True` path of conv.cu's three operations, with
// the same semantics, the same fp32 NCHW activation / gradient buffers and the same split-partial weight-gradient format.  Precision
// contract = gemm_tc.cu's (the reference's bf16 autocast of nn.Conv2d): operands rounded to bf16 while they are staged into shared
// memory, fp32 accumulation in registers, fp32 bias / activation / outputs.
//   fwd  : rows = output pixels (m, oh, ow), cols = Cout, reduction k = (ci, kh, kw); A = im2col(norm(X)), B = W[co, k]
//   dgrad: rows = input pixels (m, ih, iw),  cols = C,    reduction r = (co, kh, kw); A = dY at the output pixel each tap reads (zero
//          where the stride does not hit), B = W[co, ci, kh, kw]; times act'(A_prev) in the epilogue (deterministic, no atomics)
//   wgrad: rows = k = (ci, kh, kw),          cols = Cout, reduction = the output pixels of row split s; A = im2col(norm(X))^T,
//          B = dY^T; the tile is written transposed into dW_s[co, k], db_s[co] = row sums of the staged (bf16) dY tile
// The first layer reads the observation arena like conv2d_fwd: chunked rows, uint8 / 255 or fp32, NHWC or NCHW, the optional per-element
// normaliser (±5 clamp) before zero padding.  Weights are read from the bf16 twin of the parameter arena (b200rl_cast_bf16), same layout.
//
// Tiling and data movement follow gemm_tc.cu: one CTA = one [128 x BN] output tile (BN = 32, 64 or 128 from the column count;
// warpgroup g accumulates rows [64 g, 64 g + 64) in registers), reduction in 64-element slabs through a two-stage ring of K-major
// INTERLEAVE operand tiles (tc_common.cuh), one m64nBNk16 wgmma chain per slab.  Only the loaders differ: each thread gathers its
// operand chunks (8 consecutive reduction elements of one tile row, im2col indices stepped, not divided) into registers as bf16.  The
// gather of slab s + 1 is issued right after the wgmma chain of slab s is committed, so it runs while the tensor cores work; each
// warpgroup waits for its previous chain before the stage barrier, so a stage is rewritten only after every MMA that read it is done.
// Epilogue: the accumulators go to a [128 x (BN + 1)] fp32 tile in the (then idle) ring; lane = output row, so consecutive lanes write
// consecutive pixels of one NCHW plane (fwd, dgrad) or consecutive k of one dW row (wgrad).
#include "common.cuh"
#include "tc_common.cuh"

namespace {

using namespace tc;

constexpr int GT = 256;              // threads per CTA: two warpgroups
constexpr int SLAB = 64;             // reduction elements per ring stage
constexpr int BM = 128;              // output rows per CTA
constexpr int BNMAX = 128;           // output columns per CTA (64 fp32 accumulators per thread)
constexpr uint32_t RS = (SLAB / 8) * 128u;                                 // K-major tile: bytes per group of 8 rows
constexpr uint32_t A_BYTES = BM * SLAB * 2, B_BYTES = BNMAX * SLAB * 2, STAGE_BYTES = A_BYTES + B_BYTES;
constexpr uint32_t ACC_BYTES = BM * (BNMAX + 1) * 4;                        // fp32 accumulator tile of the epilogue (reuses the ring)
constexpr uint32_t SMEM_BYTES = 2 * STAGE_BYTES > ACC_BYTES ? 2 * STAGE_BYTES : ACC_BYTES;

enum { MODE_FWD = 0, MODE_DGRAD = 1, MODE_WGRAD = 2 };

struct Geo {
    int C, H, W, Cout, KH, KW, s, pad, Ho, Wo;
};

struct ConvArgs {
    const void* X; int rows_per_chunk; int64_t chunk_stride; int64_t x_ld; const float* nm; const float* ns;   // input rows (fwd, wgrad)
    const float* dY;                                                     // output gradient, NCHW (dgrad, wgrad)
    const __nv_bfloat16* Wb; int w_vec;                                  // bf16 weights [Cout, C, KH, KW]; w_vec: rows 16-byte aligned
    const float* bias; float* Y; int act;                               // fwd
    const float* A_prev; float* dX; int act_prev;                       // dgrad
    float* dW; float* db; int64_t split_stride; int64_t rows_per_split; // wgrad
    int M; Geo g;
    int64_t Mo; int No; int64_t R;                                      // output rows, output cols, reduction length
};

template <typename T>
__device__ __forceinline__ float to_f32(T v);
template <>
__device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <>
__device__ __forceinline__ float to_f32<uint8_t>(uint8_t v) { return __fdiv_rn((float)v, 255.0f); }   // obs.float() / 255.0

// element (ci, ih, iw) of one input row, zero outside the image (conv.cu's reading of the arena)
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

// i = (a * nb + b) * nc + c, stepped by one: the im2col indices of consecutive reduction elements without a division each
struct Idx3 { int a, b, c; };
__device__ __forceinline__ Idx3 idx3(int64_t i, int nb, int nc) {
    const int64_t ab = i / nc, a = ab / nb;
    return Idx3{(int)a, (int)(ab - a * nb), (int)(i - ab * nc)};
}
__device__ __forceinline__ void step3(Idx3& x, int nb, int nc) {
    if (++x.c == nc) { x.c = 0; if (++x.b == nb) { x.b = 0; ++x.a; } }
}

// what a tile row needs for its gathers, decomposed once per CTA: a base pointer and up to three indices
struct RowInfo { const void* p; int u, v, w; bool ok; };

// item i of a K-major [rows x 64] tile = chunk (r, cg): r = (i & 7) | ((i >> 6) << 3), cg = (i >> 3) & 7 (gemm_tc.cu's order: a warp
// stores 4 conflict-free 128-byte core matrices)
__device__ __forceinline__ void item_rc(int i, int& r, int& cg) {
    cg = (i >> 3) & 7;
    r = (i & 7) | ((i >> 6) << 3);
}

template <int MODE, typename T>
__device__ __forceinline__ RowInfo row_a(const ConvArgs& p, int64_t gr) {
    const Geo& g = p.g;
    RowInfo ri{nullptr, 0, 0, 0, gr < p.Mo};
    if (!ri.ok) return ri;
    if constexpr (MODE == MODE_FWD) {                 // output pixel (m, oh, ow): its input row and the top-left tap
        const int HWo = g.Ho * g.Wo;
        const int m = (int)(gr / HWo), pix = (int)(gr - (int64_t)m * HWo), oh = pix / g.Wo, ow = pix - oh * g.Wo;
        ri.p = static_cast<const T*>(p.X) + chunk_row(m, p.rows_per_chunk, p.chunk_stride) * p.x_ld;
        ri.u = oh * g.s - g.pad; ri.v = ow * g.s - g.pad;
    } else if constexpr (MODE == MODE_DGRAD) {        // input pixel (m, ih, iw): its sample's dY and its padded position
        const int HW = g.H * g.W;
        const int m = (int)(gr / HW), q = (int)(gr - (int64_t)m * HW), ih = q / g.W;
        ri.p = p.dY + (int64_t)m * g.Cout * g.Ho * g.Wo;
        ri.u = ih + g.pad; ri.v = q - ih * g.W + g.pad;
    } else {                                          // reduction column k = (ci, kh, kw)
        const Idx3 x = idx3(gr, g.KH, g.KW);
        ri.u = x.a; ri.v = x.b - g.pad; ri.w = x.c - g.pad;
    }
    return ri;
}

template <int MODE>
__device__ __forceinline__ RowInfo row_b(const ConvArgs& p, int gn) {
    const Geo& g = p.g;
    RowInfo ri{nullptr, gn, 0, 0, gn < p.No};
    if (!ri.ok) return ri;
    if constexpr (MODE == MODE_FWD) ri.p = p.Wb + (int64_t)gn * g.C * g.KH * g.KW;         // filter co
    else if constexpr (MODE == MODE_WGRAD) ri.p = p.dY + (int64_t)gn * g.Ho * g.Wo;       // dY plane co
    return ri;                                                                             // dgrad: input channel ci = u
}

// A chunk: reduction elements [r0, r0 + 8) of one tile row, rounded to bf16
template <int MODE, typename T, bool NHWC>
__device__ __forceinline__ uint4 gather_a(const RowInfo& ri, int64_t r0, int64_t r_end, const ConvArgs& p) {
    const Geo& g = p.g;
    float f[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = 0.f;
    if (!ri.ok || r0 >= r_end) return pack8_bf16(f);
    if constexpr (MODE == MODE_FWD) {
        Idx3 x = idx3(r0, g.KH, g.KW);                // (ci, kh, kw)
        const T* row = static_cast<const T*>(ri.p);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (r0 + j < r_end) f[j] = load_in<T, NHWC>(row, x.a, ri.u + x.b, ri.v + x.c, g, p.nm, p.ns);
            step3(x, g.KH, g.KW);
        }
    } else if constexpr (MODE == MODE_DGRAD) {
        Idx3 x = idx3(r0, g.KH, g.KW);                // (co, kh, kw)
        const float* dy = static_cast<const float*>(ri.p);
        const int HWo = g.Ho * g.Wo;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int th = ri.u - x.b, tw = ri.v - x.c;
            if (r0 + j < r_end && th >= 0 && tw >= 0) {
                const int oh = th / g.s, ow = tw / g.s;
                if (oh * g.s == th && ow * g.s == tw && oh < g.Ho && ow < g.Wo) f[j] = __ldg(dy + (int64_t)x.a * HWo + oh * g.Wo + ow);
            }
            step3(x, g.KH, g.KW);
        }
    } else {
        Idx3 x = idx3(r0, g.Ho, g.Wo);                // output pixel (m, oh, ow)
        const T* X = static_cast<const T*>(p.X);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (r0 + j < r_end) {
                const T* row = X + chunk_row(x.a, p.rows_per_chunk, p.chunk_stride) * p.x_ld;
                f[j] = load_in<T, NHWC>(row, ri.u, x.b * g.s + ri.v, x.c * g.s + ri.w, g, p.nm, p.ns);
            }
            step3(x, g.Ho, g.Wo);
        }
    }
    return pack8_bf16(f);
}

// B chunk: reduction elements [r0, r0 + 8) of one tile row (weights stay bf16; dY is rounded)
template <int MODE>
__device__ __forceinline__ uint4 gather_b(const RowInfo& ri, int64_t r0, int64_t r_end, const ConvArgs& p) {
    const Geo& g = p.g;
    if constexpr (MODE == MODE_FWD) {
        const __nv_bfloat16* w = static_cast<const __nv_bfloat16*>(ri.p) + r0;
        if (ri.ok && p.w_vec && r0 + 8 <= r_end) return __ldg(reinterpret_cast<const uint4*>(w));
    }
    float f[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = 0.f;
    if (!ri.ok || r0 >= r_end) return pack8_bf16(f);
    if constexpr (MODE == MODE_FWD) {
        const __nv_bfloat16* w = static_cast<const __nv_bfloat16*>(ri.p) + r0;
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (r0 + j < r_end) f[j] = __bfloat162float(w[j]);
    } else if constexpr (MODE == MODE_DGRAD) {
        Idx3 x = idx3(r0, g.KH, g.KW);                // (co, kh, kw) of filter co, input channel ci = u
        const int KHW = g.KH * g.KW;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (r0 + j < r_end) f[j] = __bfloat162float(p.Wb[((int64_t)x.a * g.C + ri.u) * KHW + x.b * g.KW + x.c]);
            step3(x, g.KH, g.KW);
        }
    } else {
        Idx3 x = idx3(r0, g.Ho, g.Wo);                // output pixel (m, oh, ow) of dY plane co
        const float* dy = static_cast<const float*>(ri.p);
        const int64_t sample = (int64_t)g.Cout * g.Ho * g.Wo;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (r0 + j < r_end) f[j] = __ldg(dy + x.a * sample + x.b * g.Wo + x.c);
            step3(x, g.Ho, g.Wo);
        }
    }
    return pack8_bf16(f);
}

template <int MODE, typename T, bool NHWC, int BN>
__global__ void __launch_bounds__(GT, 1) conv_tc_kernel(const ConvArgs p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    constexpr int IA = BM * 8 / GT, IB = BN * 8 / GT;          // chunks per thread of the A / B tile
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
    const int64_t m0 = (int64_t)blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;
    // reduction range: the whole K (fwd / dgrad) or this split's output pixels (wgrad)
    int64_t r_begin = 0, r_end = p.R;
    if (MODE == MODE_WGRAD) { r_begin = min((int64_t)blockIdx.z * p.rows_per_split, p.R); r_end = min(r_begin + p.rows_per_split, p.R); }
    const int n_slabs = (int)((r_end - r_begin + SLAB - 1) / SLAB);
    RowInfo ra[IA], rb[IB];
#pragma unroll
    for (int it = 0; it < IA; ++it) { int r, cg; item_rc(tid + it * GT, r, cg); ra[it] = row_a<MODE, T>(p, m0 + r); }
#pragma unroll
    for (int it = 0; it < IB; ++it) { int r, cg; item_rc(tid + it * GT, r, cg); rb[it] = row_b<MODE>(p, n0 + r); }
    uint4 va[IA], vb[IB];
    auto gather = [&](int sl) {
        const int64_t rr = r_begin + (int64_t)sl * SLAB;
#pragma unroll
        for (int it = 0; it < IA; ++it) { int r, cg; item_rc(tid + it * GT, r, cg); va[it] = gather_a<MODE, T, NHWC>(ra[it], rr + cg * 8, r_end, p); }
#pragma unroll
        for (int it = 0; it < IB; ++it) { int r, cg; item_rc(tid + it * GT, r, cg); vb[it] = gather_b<MODE>(rb[it], rr + cg * 8, r_end, p); }
    };
    if (n_slabs > 0) gather(0);
    float acc[BN / 2];       // this warpgroup's [64 x BN] accumulator tile (wgmma fragment layout, tc_common.cuh)
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
    float bsum = 0.f;        // wgrad: bias gradient of output column n0 + tid (threads < BN of the CTAs with blockIdx.x == 0)
    for (int sl = 0; sl < n_slabs; ++sl) {
        uint8_t* sA = smem + (sl & 1) * STAGE_BYTES;
        uint8_t* sB = sA + A_BYTES;
        // stage sl & 1 was last read by the MMAs of slab sl - 2: every warpgroup waited for them before the previous barrier
#pragma unroll
        for (int it = 0; it < IA; ++it) { int r, cg; item_rc(tid + it * GT, r, cg); *reinterpret_cast<uint4*>(sA + tile_off(r, cg, 128u, RS)) = va[it]; }
#pragma unroll
        for (int it = 0; it < IB; ++it) { int r, cg; item_rc(tid + it * GT, r, cg); *reinterpret_cast<uint4*>(sB + tile_off(r, cg, 128u, RS)) = vb[it]; }
        fence_async_smem();
        wgmma_wait<0>();    // this warpgroup's MMAs of slab sl - 1 are done (they read the other stage)
        __syncthreads();
        {
            // this warpgroup's 64 rows of A start 8 row groups further; folded into the 32-bit address (see gemm_tc.cu)
            const uint32_t a_base = smem_u32(sA) + (uint32_t)wg * 8u * RS, b_base = smem_u32(sB);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < SLAB / 16; ++k)
                wgmma_m64<BN, 0, 0>(acc, make_smem_desc(a_base + k * 256u, 128u, RS), make_smem_desc(b_base + k * 256u, 128u, RS));
            wgmma_commit();
        }
        if (MODE == MODE_WGRAD && p.db && blockIdx.x == 0 && tid < BN) {
            // row sum of the (bf16) dY tile just staged: row n = tid, 64 reduction elements
            const uint8_t* row = sB + (uint32_t)(tid & 7) * 16u + (uint32_t)(tid >> 3) * RS;
            float s = 0.f;
#pragma unroll 8
            for (int r = 0; r < SLAB; ++r) s += __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(row + (uint32_t)(r >> 3) * 128u + (uint32_t)(r & 7) * 2u));
            bsum += s;
        }
        if (sl + 1 < n_slabs) gather(sl + 1);      // in flight while the tensor cores run the chain just committed
    }
    wgmma_wait<0>();
    __syncthreads();          // every MMA has read its operands and the bias sums are done: the stages become the accumulator tile
    constexpr int LS = BN + 1;                   // row stride of the fp32 accumulator tile (odd: conflict-free reads with lane = row)
    float* sAcc = reinterpret_cast<float*>(smem);
    static_assert(BM * LS * 4 <= SMEM_BYTES, "accumulator tile fits the shared memory");
    {
        const int r = 64 * wg + 16 * (warp & 3) + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            sAcc[r * LS + 8 * j + c] = acc[4 * j];
            sAcc[r * LS + 8 * j + c + 1] = acc[4 * j + 1];
            sAcc[(r + 8) * LS + 8 * j + c] = acc[4 * j + 2];
            sAcc[(r + 8) * LS + 8 * j + c + 1] = acc[4 * j + 3];
        }
    }
    __syncthreads();
    // ---- epilogue: warp w owns rows [32 (w & 3), +32) (lane = row) and columns [(w >> 2) BN / 2, +BN / 2) ----
    const Geo& g = p.g;
    const int rl = 32 * (warp & 3) + lane, c_begin = (warp >> 2) * (BN / 2);
    const int64_t row = m0 + rl;
    if (row < p.Mo) {
        const float* acc_row = sAcc + rl * LS;
        if (MODE == MODE_FWD) {
            const int64_t HWo = (int64_t)g.Ho * g.Wo, m = row / HWo;
            float* out = p.Y + m * g.Cout * HWo + (row - m * HWo);
            for (int c = c_begin; c < c_begin + BN / 2; ++c) {
                const int n = n0 + c;
                if (n < p.No) out[n * HWo] = act_fwd(acc_row[c] + (p.bias ? __ldg(p.bias + n) : 0.f), p.act);
            }
        } else if (MODE == MODE_DGRAD) {
            const int64_t HW = (int64_t)g.H * g.W, m = row / HW, base = m * g.C * HW + (row - m * HW);
            for (int c = c_begin; c < c_begin + BN / 2; ++c) {
                const int n = n0 + c;
                if (n < p.No) {
                    const int64_t o = base + n * HW;
                    p.dX[o] = p.A_prev ? acc_row[c] * act_bwd_from_out(__ldg(p.A_prev + o), p.act_prev) : acc_row[c];
                }
            }
        } else {
            float* out = p.dW + (int64_t)blockIdx.z * p.split_stride + row;
            for (int c = c_begin; c < c_begin + BN / 2; ++c) {
                const int n = n0 + c;
                if (n < p.No) out[(int64_t)n * p.Mo] = acc_row[c];
            }
        }
    }
    if (MODE == MODE_WGRAD && p.db && blockIdx.x == 0 && tid < BN && n0 + tid < p.No)
        p.db[(int64_t)blockIdx.z * p.split_stride + n0 + tid] = bsum;
}

// geometry check shared by the entry points (conv.cu's): B200RL_OK and the output size, or B200RL_EINVAL
int make_geo(Geo& g, int C, int H, int W, int Cout, int KH, int KW, int stride, int pad) {
    if (C <= 0 || H <= 0 || W <= 0 || Cout <= 0 || KH <= 0 || KW <= 0 || stride <= 0 || pad < 0) return B200RL_EINVAL;
    if (H + 2 * pad < KH || W + 2 * pad < KW) return B200RL_EINVAL;
    g = Geo{C, H, W, Cout, KH, KW, stride, pad, (H + 2 * pad - KH) / stride + 1, (W + 2 * pad - KW) / stride + 1};
    if ((int64_t)C * H * W >= (1ll << 31) || (int64_t)Cout * g.Ho * g.Wo >= (1ll << 31) || (int64_t)C * KH * KW >= (1ll << 31))
        return B200RL_EINVAL;
    return B200RL_OK;
}

template <int MODE, typename T, bool NHWC, int BN>
int launch_t(const ConvArgs& a, dim3 grid, void* stream) {
    static bool raised = false;
    if (!raised) {
        cudaError_t e = cudaFuncSetAttribute(conv_tc_kernel<MODE, T, NHWC, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES);
        if (e != cudaSuccess) return (int)e;
        raised = true;
    }
    conv_tc_kernel<MODE, T, NHWC, BN><<<grid, GT, SMEM_BYTES, as_stream(stream)>>>(a);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

// output columns per CTA: the narrowest wgmma tile that holds the layer's columns, 128 past 64
template <int MODE, typename T, bool NHWC>
int launch(const ConvArgs& a, int grid_z, void* stream) {
    const int bn = a.No <= 32 ? 32 : a.No <= 64 ? 64 : 128;
    const int64_t gx = (a.Mo + BM - 1) / BM, gy = (a.No + bn - 1) / bn;
    if (gx >= (1ll << 31) || gy > 65535 || grid_z > 65535) return B200RL_EUNSUPPORTED;
    const dim3 grid((unsigned)gx, (unsigned)gy, (unsigned)grid_z);
    if (bn == 32) return launch_t<MODE, T, NHWC, 32>(a, grid, stream);
    if (bn == 64) return launch_t<MODE, T, NHWC, 64>(a, grid, stream);
    return launch_t<MODE, T, NHWC, 128>(a, grid, stream);
}

template <int MODE>
int launch_src(const ConvArgs& a, int x_u8, int x_nhwc, int grid_z, void* stream) {
    if (x_u8) return x_nhwc ? launch<MODE, uint8_t, true>(a, grid_z, stream) : launch<MODE, uint8_t, false>(a, grid_z, stream);
    return x_nhwc ? launch<MODE, float, true>(a, grid_z, stream) : launch<MODE, float, false>(a, grid_z, stream);
}

// a source whose chunk covers all its rows is dense
inline int dense_or(int rows_per_chunk, int rows) { return rows_per_chunk >= rows ? rows : rows_per_chunk; }

}  // namespace

B200RL_EXPORT int b200rl_conv2d_fwd_tc(const void* X, int x_u8, int x_nhwc, int rows_per_chunk, int64_t chunk_stride, int64_t x_ld,
                                       const float* norm_mean, const float* norm_std, const void* W_bf16, const float* b, float* Y,
                                       int M, int C, int H, int Wd, int Cout, int KH, int KW, int stride, int pad, int act, void* stream) {
    ConvArgs a{};
    if (!X || !W_bf16 || !Y || M <= 0 || rows_per_chunk <= 0 || make_geo(a.g, C, H, Wd, Cout, KH, KW, stride, pad) != B200RL_OK)
        return B200RL_EINVAL;
    if ((norm_mean == nullptr) != (norm_std == nullptr) || x_ld < (int64_t)C * H * Wd) return B200RL_EINVAL;
    a.X = X; a.rows_per_chunk = dense_or(rows_per_chunk, M); a.chunk_stride = chunk_stride; a.x_ld = x_ld; a.nm = norm_mean; a.ns = norm_std;
    a.Wb = static_cast<const __nv_bfloat16*>(W_bf16);
    a.w_vec = ((int64_t)C * KH * KW) % 8 == 0 && (reinterpret_cast<uintptr_t>(W_bf16) & 15) == 0;
    a.bias = b; a.Y = Y; a.act = act; a.M = M;
    a.Mo = (int64_t)M * a.g.Ho * a.g.Wo; a.No = Cout; a.R = (int64_t)C * KH * KW;
    return launch_src<MODE_FWD>(a, x_u8, x_nhwc, 1, stream);
}

B200RL_EXPORT int b200rl_conv2d_bwd_data_tc(const float* dY, const void* W_bf16, const float* A_prev, float* dX, int M, int C, int H, int Wd,
                                            int Cout, int KH, int KW, int stride, int pad, int act_prev, void* stream) {
    ConvArgs a{};
    if (!dY || !W_bf16 || !dX || M <= 0 || make_geo(a.g, C, H, Wd, Cout, KH, KW, stride, pad) != B200RL_OK) return B200RL_EINVAL;
    a.dY = dY; a.Wb = static_cast<const __nv_bfloat16*>(W_bf16); a.A_prev = A_prev; a.dX = dX; a.act_prev = act_prev; a.M = M;
    a.Mo = (int64_t)M * H * Wd; a.No = C; a.R = (int64_t)Cout * KH * KW;
    return launch<MODE_DGRAD, float, false>(a, 1, stream);
}

B200RL_EXPORT int b200rl_conv2d_bwd_weight_tc(const float* dY, const void* X, int x_u8, int x_nhwc, int rows_per_chunk,
                                              int64_t chunk_stride, int64_t x_ld, const float* norm_mean, const float* norm_std,
                                              float* dW_part, float* db_part, int64_t split_stride, int M, int C, int H, int Wd,
                                              int Cout, int KH, int KW, int stride, int pad, int n_splits, void* stream) {
    ConvArgs a{};
    if (!dY || !X || !dW_part || M <= 0 || rows_per_chunk <= 0 || n_splits <= 0 ||
        make_geo(a.g, C, H, Wd, Cout, KH, KW, stride, pad) != B200RL_OK)
        return B200RL_EINVAL;
    if ((norm_mean == nullptr) != (norm_std == nullptr) || x_ld < (int64_t)C * H * Wd) return B200RL_EINVAL;
    const int64_t K = (int64_t)C * KH * KW;
    if (n_splits > 1 && split_stride < (int64_t)Cout * K) return B200RL_EINVAL;
    a.X = X; a.rows_per_chunk = dense_or(rows_per_chunk, M); a.chunk_stride = chunk_stride; a.x_ld = x_ld; a.nm = norm_mean; a.ns = norm_std;
    a.dY = dY; a.dW = dW_part; a.db = db_part; a.split_stride = split_stride; a.M = M;
    a.Mo = K; a.No = Cout; a.R = (int64_t)M * a.g.Ho * a.g.Wo;
    const int64_t rps = (a.R + n_splits - 1) / n_splits;
    a.rows_per_split = ((rps + SLAB - 1) / SLAB) * SLAB;       // trailing splits may be empty: they write zeros, which the reducer expects
    return launch_src<MODE_WGRAD>(a, x_u8, x_nhwc, n_splits, stream);
}
