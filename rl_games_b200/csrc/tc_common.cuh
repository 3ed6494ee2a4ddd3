// Hopper (sm_90a) tensor-core building blocks: wgmma on shared-memory operand descriptors, mbarrier, the register-accumulator chain
// of the fused forward and backward kernels (mma_frag) and the per-CTA fp32 accumulator buffer that the remaining fused MLP kernels
// address by (lane, column).  Descriptor bit layouts follow the PTX ISA's wgmma matrix descriptor (the same fields CUTLASS's GmmaDescriptor names).
//
// Shared-memory operand tiles use the canonical INTERLEAVE (no-swizzle) layout: 16-byte chunks of 8 bf16
// that are contiguous along the tile's "column" index, 8 consecutive "rows" stacked at 16 B stride (one 128 B
// core matrix), with two free strides:
//     offset(r, c) = (r % 8) * 16 + (c % 8) * 2 + (c / 8) * CS + (r / 8) * RS            [bytes]
// The SAME bytes serve as a K-major operand (rows = M/N, cols = K: LBO = CS, SBO = RS) and as an MN-major
// operand (cols = M/N, rows = K: SBO = CS, LBO = RS) -- which is what lets one activation / delta tile feed
// the forward/dgrad MMAs (K-major) and the weight-gradient MMAs (MN-major) without any transposed copy.
// In both views SBO is the stride between groups of 8 along M/N, so a sub-tile 8g rows further along M/N starts g * SBO
// bytes later (desc_advance_mn).
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- descriptors -------------------------------------------------------------------------------
// wgmma matrix descriptor: start_address[0,14) (>>4), leading_byte_offset[16,30) (>>4), stride_byte_offset[32,46) (>>4),
// base_offset[49,52) = 0, layout_type[62,64) = 0 (INTERLEAVE, no swizzle)
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    return d;
}
// the same operand view, `groups` x 8 rows further along M/N
__device__ __forceinline__ uint64_t desc_advance_mn(uint64_t d, uint32_t groups) {
    return d + (uint64_t)(groups * (uint32_t)((d >> 32) & 0x3FFF));
}

// generic-proxy smem writes -> visible to the async proxy (wgmma operand reads, TMA)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- mbarrier ----------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}

// ---- L2 cache policies ---------------------------------------------------------------------------------
// A minibatch update moves ~200 MB through the 50 MB L2.  Scratch that a later kernel of the same update reads back (activation and
// delta tiles, split-gradient rows) is stored with evict_last; data read for the last time in the update (observation rows, the
// tiles' last reads, the split-gradient rows in the reducer) is loaded with evict_first, so that it does not push out the former.
// The hints change where lines live, never what a load returns.
__device__ __forceinline__ uint64_t l2_policy_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t l2_policy_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint32_t ld_hint_u32(const void* p, uint64_t pol) {
    uint32_t v;
    asm volatile("ld.global.nc.L2::cache_hint.b32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ void st_hint_u32(void* p, uint32_t v, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.b32 [%0], %1, %2;" ::"l"(p), "r"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_hint_u16(void* p, uint16_t v, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.b16 [%0], %1, %2;" ::"l"(p), "h"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_hint_u128(void* p, uint4 v, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.v4.b32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "l"(pol)
                 : "memory");
}
// cached-at-L2-only loads (__ldcg) with a policy
__device__ __forceinline__ float ldcg_hint(const float* p, uint64_t pol) {
    float v;
    asm volatile("ld.global.cg.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ float4 ldcg_hint(const float4* p, uint64_t pol) {
    float4 v;
    asm volatile("ld.global.cg.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "l"(pol));
    return v;
}

// Lines of [p, p + bytes), both ends 128-byte aligned, whose data no one will read again: dropped from L2 without a write-back to
// HBM.  Run by the 32 lanes of one warp.  A read of a discarded byte before its next write returns an indeterminate value, so the
// caller must be the last reader.  The B200RL_L2_DISCARD_POISON build (a test library, never the product) stores 0xFF bytes there
// instead -- NaN in fp32 and bf16 -- so that a read after the discard fails deterministically instead of by timing.
__device__ __forceinline__ void l2_discard(void* p, size_t bytes) {
    for (size_t o = (size_t)(threadIdx.x & 31) * 128u; o < bytes; o += 32u * 128u) {
#ifdef B200RL_L2_DISCARD_POISON
        uint4* q = reinterpret_cast<uint4*>(static_cast<uint8_t*>(p) + o);
#pragma unroll
        for (int i = 0; i < 8; ++i) q[i] = make_uint4(~0u, ~0u, ~0u, ~0u);
#else
        asm volatile("discard.global.L2 [%0], 128;" ::"l"(static_cast<uint8_t*>(p) + o) : "memory");
#endif
    }
}

// ---- wgmma: D[64 x n] += A[64 x 16] . B[16 x n], bf16 operands from shared memory, fp32 accumulators in the registers of one
//      warpgroup (thread t: rows 16 (t/32) + (t%32)/4 and +8, columns 8j + 2 (t%4) + {0, 1} -> d[4j .. 4j+3]).
//      TA / TB = 1 select the MN-major view of the operand.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n8(float (&d)[4], uint64_t a, uint64_t b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 {%0,%1,%2,%3}, %4, %5, p, 1, 1, %6, %7;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "l"(a), "l"(b), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n16(float (&d)[8], uint64_t a, uint64_t b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %10, %11;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a), "l"(b), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n32(float (&d)[16], uint64_t a, uint64_t b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %18, %19;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64(float (&d)[32], uint64_t a, uint64_t b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %34, %35;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t a, uint64_t b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, %66, %67;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "n"(TA), "n"(TB));
}
template <int NS, int TA, int TB>
__device__ __forceinline__ void wgmma_m64(float (&d)[NS / 2], uint64_t a, uint64_t b) {
    if constexpr (NS == 8) wgmma_m64n8<TA, TB>(d, a, b);
    else if constexpr (NS == 16) wgmma_m64n16<TA, TB>(d, a, b);
    else if constexpr (NS == 32) wgmma_m64n32<TA, TB>(d, a, b);
    else if constexpr (NS == 64) wgmma_m64n64<TA, TB>(d, a, b);
    else { static_assert(NS == 128, "wgmma tile width"); wgmma_m64n128<TA, TB>(d, a, b); }
}

// ---- register-accumulator MMA -----------------------------------------------------------------------------------
// One operand of a wgmma chain, as seen by the calling warpgroup: 32-bit shared address of its sub-tile at k = 0 (any offset along
// M/N already folded in: 64-bit descriptor arithmetic between chained wgmmas makes ptxas serialise them), byte step per k step of
// 16 reduction elements, and the two descriptor strides.
struct MmaOperand { uint32_t addr, kstep, lbo, sbo; };
// d[64 x NS] += sum over k < NK of A_k[64 x 16] . B_k[16 x NS] on a fragment the calling warpgroup owns.  Issues and commits the chain
// and returns: no wait, no global memory, no barrier.  d must not be touched before a wgmma_wait<> that covers this group.
template <int NS, int TA, int TB, int NK>
__device__ __forceinline__ void mma_frag(float (&d)[NS / 2], const MmaOperand a, const MmaOperand b) {
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < NK; ++k)
        wgmma_m64<NS, TA, TB>(d, make_smem_desc(a.addr + k * a.kstep, a.lbo, a.sbo), make_smem_desc(b.addr + k * b.kstep, b.lbo, b.sbo));
    wgmma_commit();
}
// fragment -> tile coordinates: d[4j], d[4j+1] sit at row frag_row(), columns 8j + frag_col() + {0, 1}; d[4j+2], d[4j+3] 8 rows below.
// The 32 lanes of a warp cover 8 rows x 4 column pairs per j = one 128-byte core matrix of an INTERLEAVE tile.
__device__ __forceinline__ int frag_row() { return 16 * ((threadIdx.x >> 5) & 3) + ((threadIdx.x & 31) >> 2); }
__device__ __forceinline__ int frag_col() { return 2 * (threadIdx.x & 3); }

// ---- per-CTA accumulator buffer ------------------------------------------------------------------------------
// The fused kernels keep 128-row fp32 accumulators addressed as (lane, column) with taddr = (lane << 16) | column: layer outputs
// that the epilogue reads back row by row, and weight gradients that stay resident across every tile a persistent CTA processes.
// Hopper has no tensor memory, so the columns live in a [TMEM_COLS][128] fp32 region of global memory per CTA (256 KB, L2-resident):
// mma128() runs the MMAs on the warpgroups' registers and writes the result there, tmem_ld* reads one lane per thread.
// A translation unit that uses it defines TC_ACC_POOL_CTAS (the largest grid of its kernels) before including this header.
// Kernels that share a pool must run in stream order (each one touches the pool only after griddepcontrol.wait): the pool is
// indexed by blockIdx.x, so two streams running kernels of the same translation unit at once would overwrite each other's
// accumulators.  Cost: every mma128() round-trips its accumulators through L2 and ends with a CTA barrier (DESIGN.md §4).
constexpr int TMEM_COLS = 512, TMEM_LANES = 128;
#ifdef TC_ACC_POOL_CTAS
static __device__ float g_acc_pool[(size_t)TC_ACC_POOL_CTAS * TMEM_COLS * TMEM_LANES];
__device__ __forceinline__ float* acc_cta() { return g_acc_pool + (size_t)blockIdx.x * TMEM_COLS * TMEM_LANES; }

// columns [0, ncols) of this CTA's accumulator buffer: the base address is 0
__device__ __forceinline__ void tmem_alloc(uint32_t* smem_dst, uint32_t ncols) {
    (void)ncols;
    if ((threadIdx.x & 31) == 0) *smem_dst = 0u;
}

// lanes (taddr >> 16) + 0..31 (one per thread of the warp), N consecutive columns from (taddr & 0xFFFF)
template <int N>
__device__ __forceinline__ void tmem_ldn(uint32_t taddr, float (&v)[N]) {
    const float* src = acc_cta() + (size_t)(taddr & 0xFFFFu) * TMEM_LANES + (taddr >> 16) + (threadIdx.x & 31);
#pragma unroll
    for (int i = 0; i < N; ++i) v[i] = __ldcg(src + (size_t)i * TMEM_LANES);
}
__device__ __forceinline__ void tmem_ld16(uint32_t taddr, float (&v)[16]) { tmem_ldn<16>(taddr, v); }
__device__ __forceinline__ void tmem_ld32(uint32_t taddr, float (&v)[32]) { tmem_ldn<32>(taddr, v); }

// D[128 x N] at accumulator columns [dcol, dcol + N)  (+)=  sum over k < nk of A_k[128 x 16] . B_k[16 x N], where descs(k, a, b)
// yields the descriptors of step k exactly as for a 128-row MMA.  Called by EVERY thread of the CTA (NWG warpgroups); the 2 x N/NS
// [64 x NS] sub-tiles are spread over the warpgroups, each accumulates in registers (from the buffer when acc, else from 0) and
// stores its sub-tile back.  Ends with __syncthreads(): the result is visible to every thread.
template <int N, int TA, int TB, int NWG, class Descs>
__device__ __forceinline__ void mma128(uint32_t dcol, int nk, bool acc, Descs descs) {
    constexpr int NS0 = 2 * N / NWG;
    constexpr int NS1 = NS0 >= 64 ? 64 : (NS0 <= 8 ? 8 : NS0);
    constexpr int NS = NS1 < N ? NS1 : N;
    static_assert(N % NS == 0 && (NS & (NS - 1)) == 0, "accumulator sub-tile width");
    constexpr int UNITS = 2 * (N / NS);
    const int wg = threadIdx.x >> 7, w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
    float* buf = acc_cta();
    for (int u = wg; u < UNITS; u += NWG) {
        const int mh = u & 1, ns = u >> 1;
        float* base = buf + (size_t)(dcol + ns * NS + 2 * (l & 3)) * TMEM_LANES + 64 * mh + 16 * w + (l >> 2);
        float d[NS / 2];
#pragma unroll
        for (int j = 0; j < NS / 8; ++j) {
            float* b0 = base + (size_t)(8 * j) * TMEM_LANES;
            d[4 * j + 0] = acc ? __ldcg(b0) : 0.f;
            d[4 * j + 1] = acc ? __ldcg(b0 + TMEM_LANES) : 0.f;
            d[4 * j + 2] = acc ? __ldcg(b0 + 8) : 0.f;
            d[4 * j + 3] = acc ? __ldcg(b0 + TMEM_LANES + 8) : 0.f;
        }
        wgmma_fence();
        for (int k = 0; k < nk; ++k) {
            uint64_t a, b;
            descs(k, a, b);
            wgmma_m64<NS, TA, TB>(d, desc_advance_mn(a, 8u * mh), desc_advance_mn(b, (uint32_t)(ns * NS / 8)));
        }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int j = 0; j < NS / 8; ++j) {
            float* b0 = base + (size_t)(8 * j) * TMEM_LANES;
            __stcg(b0, d[4 * j + 0]);
            __stcg(b0 + TMEM_LANES, d[4 * j + 1]);
            __stcg(b0 + 8, d[4 * j + 2]);
            __stcg(b0 + TMEM_LANES + 8, d[4 * j + 3]);
        }
    }
    __syncthreads();
}
#endif  // TC_ACC_POOL_CTAS

// pack 8 floats -> 8 bf16 (16 bytes)
__host__ __device__ __forceinline__ uint4 pack8_bf16(const float* f) {
    __nv_bfloat162 a = __floats2bfloat162_rn(f[0], f[1]), b = __floats2bfloat162_rn(f[2], f[3]);
    __nv_bfloat162 c = __floats2bfloat162_rn(f[4], f[5]), d = __floats2bfloat162_rn(f[6], f[7]);
    uint4 u;
    u.x = *reinterpret_cast<uint32_t*>(&a); u.y = *reinterpret_cast<uint32_t*>(&b);
    u.z = *reinterpret_cast<uint32_t*>(&c); u.w = *reinterpret_cast<uint32_t*>(&d);
    return u;
}

// byte offset of the 16-byte chunk holding (row r, columns 8*cg .. 8*cg+7) in an INTERLEAVE tile
__host__ __device__ __forceinline__ uint32_t tile_off(int r, int cg, uint32_t CS, uint32_t RS) {
    return (uint32_t)(r & 7) * 16u + (uint32_t)cg * CS + (uint32_t)(r >> 3) * RS;
}

}  // namespace tc
