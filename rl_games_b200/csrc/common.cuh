// Shared device helpers for libb200rl (sm_90a).  No torch types anywhere in csrc/.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/b200rl.h"

#define B200RL_LAUNCH_CHECK()                          \
    do {                                               \
        cudaError_t e__ = cudaGetLastError();          \
        if (e__ != cudaSuccess) return (int)e__;       \
    } while (0)

#define B200RL_EXPORT extern "C" __attribute__((visibility("default")))
static inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// ---- programmatic dependent launch (PDL) ---------------------------------------------------------------------------
// The per-minibatch chain (forward -> backward 1 -> backward 2 -> optimiser) is four dependent launches of persistent kernels
// whose prologues (TMEM allocation, barrier init, smem zero fill, observation prefetch) need nothing from the predecessor.
// Kernels launched through launch_k() carry cudaLaunchAttributeProgrammaticStreamSerialization, so their CTAs may be
// scheduled while the predecessor's last CTAs are still running; every such kernel calls pdl_sync() before it reads or
// writes ANY global memory the predecessor chain touches (the only pre-wait global reads anywhere are the forward kernel's
// observation rows, produced by the environment, never by one of these kernels).  pdl_sync() = griddepcontrol.wait (the
// predecessor grid has completed and its writes are visible) followed by griddepcontrol.launch_dependents; because the
// trigger comes AFTER the wait, "my successor is running" implies "my predecessor completed", so completion is transitive
// along the chain.  Without the launch attribute both instructions are no-ops.  Captured by stream capture as programmatic
// dependency edges of the CUDA graph.
__device__ __forceinline__ void pdl_sync() {
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
extern int g_b200rl_pdl;     // api.cu; b200rl_set_pdl()
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = g_b200rl_pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Block-wide sum of NV doubles per thread; result valid in thread 0 (and broadcast via smem to all).
// blockDim.x must be a multiple of 32 and <= 1024.  `sm` must hold 32*NV doubles.
template <int NV>
__device__ __forceinline__ void block_sum_d(double (&v)[NV], double* sm) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
    for (int i = 0; i < NV; ++i) v[i] = warp_sum(v[i]);
    __syncthreads();
    if (lane == 0) {
#pragma unroll
        for (int i = 0; i < NV; ++i) sm[warp * NV + i] = v[i];
    }
    __syncthreads();
    if (warp == 0) {
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            double x = (lane < nw) ? sm[lane * NV + i] : 0.0;
            x = warp_sum(x);
            if (lane == 0) sm[i] = x;
        }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < NV; ++i) v[i] = sm[i];
    __syncthreads();
}

// ---- Philox4x32-10 (Salmon et al.), counter-based so launches are CUDA-graph replayable ----------
// Counter layout: ctr_lo = row (env index), ctr_hi = bit fields that must never overlap, or two draws would share a stream.
//   policy samplers (rollout.cu, mlp_tc.cu, discrete.cu): epoch << 20 | step << 4 | q,  step < 2^16, q < 16:
//     Gaussian heads q = 0..7 (four normals per q, up to 32 actions), categorical heads q = 8 + j (j < CAT_MAXH = 8); the wide
//     categorical sampler's head j uses q = 8 + (j & 7) with (j >> 3) in the high word of ctr_lo, which is 0 for every other
//     policy sampler (rows < 2^31)
//   synthetic env (rollout.cu synth_env_step_kernel, its own keys): epoch << 20 | step << 10 | q, step < 2^10,
//     q < 2^9 (feature group of four), bit 9 set for the done draw
// tests/_philox_ref.py restates this generator and the mappings below bit for bit on the host.
struct Philox4 { uint32_t x, y, z, w; };
__device__ __forceinline__ Philox4 philox4x32_10(uint64_t ctr_lo, uint64_t ctr_hi, uint64_t key) {
    uint32_t c0 = (uint32_t)ctr_lo, c1 = (uint32_t)(ctr_lo >> 32), c2 = (uint32_t)ctr_hi, c3 = (uint32_t)(ctr_hi >> 32);
    uint32_t k0 = (uint32_t)key, k1 = (uint32_t)(key >> 32);
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    return Philox4{c0, c1, c2, c3};
}
__device__ __forceinline__ float u32_to_unit_open(uint32_t u) {   // (0,1]
    return ((float)(u >> 8) + 1.0f) * (1.0f / 16777216.0f);
}
// two standard normals from two 32-bit words (Box-Muller)
__device__ __forceinline__ void box_muller(uint32_t a, uint32_t b, float& n0, float& n1) {
    const float u = u32_to_unit_open(a), v = u32_to_unit_open(b);
    const float r = sqrtf(-2.0f * __logf(u));
    float s, c;
    __sincosf(6.283185307179586f * v, &s, &c);
    n0 = r * c; n1 = r * s;
}

__device__ __forceinline__ float act_fwd(float x, int act) {
    switch (act) {
        case B200RL_ACT_ELU:  return x > 0.f ? x : expm1f(x);
        case B200RL_ACT_RELU: return x > 0.f ? x : 0.f;
        case B200RL_ACT_TANH: return tanhf(x);
        default: return x;
    }
}
// derivative expressed through the activation OUTPUT a
__device__ __forceinline__ float act_bwd_from_out(float a, int act) {
    switch (act) {
        case B200RL_ACT_ELU:  return a > 0.f ? 1.f : a + 1.f;
        case B200RL_ACT_RELU: return a > 0.f ? 1.f : 0.f;
        case B200RL_ACT_TANH: return 1.f - a * a;
        default: return 1.f;
    }
}

// arena chunk mapping: local row m -> element row index
__device__ __forceinline__ int64_t chunk_row(int m, int rows_per_chunk, int64_t chunk_stride) {
    const int c = m / rows_per_chunk;
    return (int64_t)c * chunk_stride + (m - c * rows_per_chunk);
}
