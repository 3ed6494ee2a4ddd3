// Optimiser step: (1/world) scaling + global-norm clip + Adam + on-device adaptive-KL LR schedule.
// Replaces a2c_common.py:493-514 (trancate_gradients_and_step), torch.optim.Adam(eps=1e-8,
// weight_decay, fused=True) (a2c_continuous.py:44-48) and schedulers.py:19-33 + a2c_common.py:1557-1563
// (kl.item() host sync per minibatch).  One launch: every CTA recomputes the global grad norm from the
// (L2-resident) flat gradient buffer in the same order, so no inter-CTA reduction or atomics are needed
// and the result is deterministic; the last CTA to finish advances (step, lr).
#include "common.cuh"
#include "loss_math.cuh"
#include "tc_common.cuh"
#include <cuda_bf16.h>
#include <string.h>

namespace {

struct OptCfgDev {
    double beta1, beta2, eps, weight_decay, grad_norm, kl_threshold, min_lr, max_lr, lr_multiplier, grad_scale;
    int truncate_grads, adaptive_lr;
};

// Adaptive-KL scheduler step (schedulers.py:19-33; python floats == fp64), run by one thread after the optimiser step.
//   adaptive_lr == 1: schedule_type 'per_minibatch' -- one scheduler step per optimiser step on this minibatch's KL.
//   adaptive_lr == 2 / 3: schedule_type 'standard' (a2c_common.py:1565-1571) -- one scheduler step per MINI-EPOCH on the mean of its
//     minibatches' KLs (torch_ext.mean_list): 2 = add this KL to the running sum / count in state_d[4] / state_d[5];
//     3 = last minibatch of the mini-epoch: add, step the scheduler on the mean, reset the accumulators.
__host__ __device__ __forceinline__ double lr_schedule_step(double lr, double kl, const OptCfgDev& c, double* state_d) {
    if (c.adaptive_lr >= 2) {
        const double s = state_d[4] + kl, cnt = state_d[5] + 1.0;
        const bool apply = c.adaptive_lr == 3;
        state_d[4] = apply ? 0.0 : s;
        state_d[5] = apply ? 0.0 : cnt;
        if (!apply) return lr;
        kl = s / cnt;
    }
    if (kl > 2.0 * c.kl_threshold) return fmax(lr / c.lr_multiplier, c.min_lr);
    if (kl < 0.5 * c.kl_threshold) return fmin(lr * c.lr_multiplier, c.max_lr);
    return lr;
}

// optional tail work of the optimiser kernels' last CTA: training-mode update of the obs normaliser for the NEXT minibatch
// (Chan merge of its precomputed batch sums, running_mean_std.py:55-67) -- saves one tiny launch per minibatch
struct ObsMergeDev {
    const double* mbmom; const float* shift; int D; int n_rows;
    double* mean; double* var; long long* count; float* mean_f32; float* std_f32; float eps;
};
__device__ __forceinline__ void obs_merge_tail(const ObsMergeDev& o) {
    // called by ALL threads of the last CTA (blockDim >= 1)
    if (!o.mbmom) return;
    const double n = (double)o.n_rows;
    const double cnt0 = (double)o.count[0];
    for (int col = threadIdx.x; col < o.D; col += blockDim.x) {
        const double ms = o.mbmom[col] / n;
        const double bm = (double)o.shift[col] + ms;
        const double bv = fmax(o.mbmom[o.D + col] / n - ms * ms, 0.0);
        const double tot = cnt0 + n, delta = bm - o.mean[col];
        const double new_mean = o.mean[col] + delta * n / tot;
        const double M2 = o.var[col] * cnt0 + bv * n + delta * delta * cnt0 * n / tot;
        const double v = M2 / tot;
        o.mean[col] = new_mean; o.var[col] = v;
        o.mean_f32[col] = (float)new_mean;
        o.std_f32[col] = __fsqrt_rn(__fadd_rn((float)v, o.eps));
    }
    __syncthreads();
    if (threadIdx.x == 0) o.count[0] = o.count[0] + (long long)o.n_rows;
}

struct PackTabDev { int n_seg; int off[4]; int R[4]; int C[4]; unsigned CS[4]; unsigned dst[4]; };

// one element of the fused Adam update (torch.optim.Adam fused semantics) + refresh of the packed bf16 weight copy
__device__ __forceinline__ void adam_update_one(int i, float g, int truncate, float coef, float* __restrict__ params,
                                                float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq, float b1, float b2,
                                                float step_size, float bc2_sqrt, float eps, float wd, unsigned char* __restrict__ wpack,
                                                const PackTabDev& tab) {
    if (truncate) g *= coef;
    float p = params[i];
    if (wd != 0.f) g = fmaf(wd, p, g);
    float m = exp_avg[i], v = exp_avg_sq[i];
    m = m + (g - m) * (1.0f - b1);                 // lerp (torch fused adam)
    v = b2 * v + (1.0f - b2) * g * g;
    const float denom = sqrtf(v) / bc2_sqrt + eps;
    p -= step_size * m / denom;
    params[i] = p; exp_avg[i] = m; exp_avg_sq[i] = v;
    if (wpack) {
        // refresh the bf16 operand copy the tensor-core kernels consume (INTERLEAVE weight tile: CS = (Rpad/8)*128, RS = 128)
#pragma unroll
        for (int sgi = 0; sgi < 4; ++sgi) {
            if (sgi < tab.n_seg) {
                const int loc = i - tab.off[sgi];
                if (loc >= 0 && loc < tab.R[sgi] * tab.C[sgi]) {
                    const int r = loc / tab.C[sgi], cc = loc - r * tab.C[sgi];
                    const unsigned o = tab.dst[sgi] + (unsigned)(r & 7) * 16u + (unsigned)(cc >> 3) * tab.CS[sgi] + (unsigned)(r >> 3) * 128u +
                                       (unsigned)(cc & 7) * 2u;
                    *reinterpret_cast<__nv_bfloat16*>(wpack + o) = __float2bfloat16_rn(p);
                }
            }
        }
    }
}

__global__ void __launch_bounds__(1024) adam_step_kernel(float* __restrict__ params, const float* __restrict__ grads,
                                                        float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq, int n,
                                                        double* state_d, const float* __restrict__ kl_dev, OptCfgDev c,
                                                        float* __restrict__ stats_out, int* counter, unsigned char* __restrict__ wpack,
                                                        PackTabDev tab, ObsMergeDev om) {
    __shared__ double sm[32];
    __shared__ int is_last;
    pdl_sync();
    const double lr = state_d[0];
    const double step = state_d[1] + 1.0;
    // running products beta^step live in the device state (state_d[2], state_d[3]); 0 means "not started" == 1.0
    const double p1 = (state_d[2] > 0.0 ? state_d[2] : 1.0) * c.beta1;
    const double p2 = (state_d[3] > 0.0 ? state_d[3] : 1.0) * c.beta2;
    const float gs = (float)c.grad_scale;
    // ---- global norm (identical in every CTA: same order, fp32 per-thread partials, fp64 block reduction) ----
    double acc[1] = {0.0};
    if (c.truncate_grads || stats_out) {
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        const int n4 = ((reinterpret_cast<uintptr_t>(grads) & 15) == 0) ? (n >> 2) : 0;
        const float4* g4 = reinterpret_cast<const float4*>(grads);
        for (int i = threadIdx.x; i < n4; i += blockDim.x) {
            const float4 g = __ldg(g4 + i);
            a0 = fmaf(g.x * gs, g.x * gs, a0); a1 = fmaf(g.y * gs, g.y * gs, a1);
            a2 = fmaf(g.z * gs, g.z * gs, a2); a3 = fmaf(g.w * gs, g.w * gs, a3);
        }
        for (int i = n4 * 4 + threadIdx.x; i < n; i += blockDim.x) {
            const float g = __ldg(grads + i) * gs;
            a0 = fmaf(g, g, a0);
        }
        acc[0] = ((double)a0 + (double)a1) + ((double)a2 + (double)a3);
        block_sum_d<1>(acc, sm);
    }
    const float total_norm = (float)sqrt(acc[0]);
    float coef = 1.0f;
    if (c.truncate_grads) coef = fminf((float)c.grad_norm / (total_norm + 1e-6f), 1.0f);
    const float b1 = (float)c.beta1, b2 = (float)c.beta2;
    const double bc1 = 1.0 - p1, bc2 = 1.0 - p2;
    const float step_size = (float)(lr / bc1);
    const float bc2_sqrt = (float)sqrt(bc2);
    const float eps = (float)c.eps, wd = (float)c.weight_decay;
    const int per = (n + gridDim.x - 1) / gridDim.x;
    const int i0 = blockIdx.x * per, i1 = min(i0 + per, n);
    for (int i = i0 + threadIdx.x; i < i1; i += blockDim.x)
        adam_update_one(i, __ldg(grads + i) * gs, c.truncate_grads, coef, params, exp_avg, exp_avg_sq, b1, b2, step_size, bc2_sqrt, eps, wd,
                        wpack, tab);
    // ---- last CTA advances step / lr (all CTAs have read them by now) ----
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const int prev = atomicAdd(counter, 1);
        is_last = (prev == (int)gridDim.x - 1);
    }
    __syncthreads();
    if (is_last && threadIdx.x == 0) {
        double new_lr = lr;
        if (c.adaptive_lr && kl_dev) {
            const double kl = (double)(__ldg(kl_dev) * gs);   // summed over ranks by the all-reduce -> mean (a2c_common.py:1559-1561)
            new_lr = lr_schedule_step(lr, kl, c, state_d);
        }
        state_d[0] = new_lr;
        state_d[1] = step;
        state_d[2] = p1;
        state_d[3] = p2;
        if (stats_out) { stats_out[B200RL_STAT_LR] = (float)lr; stats_out[B200RL_STAT_GNORM] = total_norm; }
        *counter = 0;
    }
    if (is_last) obs_merge_tail(om);
}

// =====================================================================================================================
// Fused gradient all-reduce + clip + Adam over NVLink peer memory (one launch per minibatch, replaces
// cat -> dist.all_reduce -> /world -> scatter -> clip_grad_norm_ -> optimizer.step of a2c_common.py:493-514 and the
// KL all-reduce of :1559-1561).  Every rank's gradient arena (+KL slot) lives in a CUDA-IPC mapped buffer; each rank
//   0. signals "my gradients for step s are ready" into every peer's flag array (st.release.sys) and waits for all peers,
//   1. sums ALL peers' buffers slice by slice with plain peer loads (fixed rank order => every rank computes bit-identical
//      reduced gradients), stores the sum locally and records per-CTA sum-of-squares partials,
//   2. grid barrier (all CTAs are co-resident: grid <= #SMs, one CTA per SM),
//   3. clip + Adam + packed-bf16 refresh from the local reduced copy; the last CTA advances (lr, step, seq).
// Gradient buffers are double-buffered by minibatch parity, so the single cross-rank barrier per step also protects the
// buffer written two steps later (a rank can only reach step s+1 after every rank entered step s+... see DESIGN.md).
struct PeerPtrs { const float* grads[8]; unsigned long long* flags[8]; };

__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ld_acquire_gpu_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
// Grid barrier on a monotonic 64-bit arrival counter (never reset, never wraps: 2^64 arrivals).  All CTAs are co-resident (grid <= #SMs).
__device__ __forceinline__ void grid_barrier_arrive_wait(unsigned long long* grid_bar) {
    const unsigned long long arrived = atomicAdd(grid_bar, 1ull);
    const unsigned long long target = (arrived / gridDim.x + 1ull) * gridDim.x;
    while (ld_acquire_gpu_u64(grid_bar) < target) { }
}

__global__ void __launch_bounds__(1024) allreduce_adam_kernel(PeerPtrs peers, int world, int rank, unsigned long long* my_flags,
                                                             unsigned long long* seq_ptr, float* __restrict__ red, double* __restrict__ nrm_part,
                                                             unsigned long long* grid_bar, float* __restrict__ params, float* __restrict__ exp_avg,
                                                             float* __restrict__ exp_avg_sq, int n, double* state_d, OptCfgDev c,
                                                             float* __restrict__ stats_out, int* counter, unsigned char* __restrict__ wpack,
                                                             PackTabDev tab, ObsMergeDev om) {
    __shared__ double sm[32];
    __shared__ int is_last;
    pdl_sync();
    const unsigned long long seq = *seq_ptr + 1ull;
    // ---- 0. cross-rank barrier: my gradients (written by the previous kernel in this stream) are complete ----
    if (blockIdx.x == 0 && threadIdx.x < world) st_release_sys(peers.flags[threadIdx.x] + rank, seq);
    if (threadIdx.x < world) {
        while (ld_acquire_sys(my_flags + threadIdx.x) < seq) { }
    }
    __syncthreads();
    const double lr = state_d[0];
    const double step = state_d[1] + 1.0;
    const double p1 = (state_d[2] > 0.0 ? state_d[2] : 1.0) * c.beta1;
    const double p2 = (state_d[3] > 0.0 ? state_d[3] : 1.0) * c.beta2;
    const float gs = (float)c.grad_scale;
    // ---- 1. reduce my slice across ranks (n gradient entries + the KL slot at index n) ----
    const int ntot = n + 1;
    const int per = (ntot + gridDim.x - 1) / gridDim.x;
    const int i0 = blockIdx.x * per, i1 = min(i0 + per, ntot);
    float a0 = 0.f;
    for (int i = i0 + threadIdx.x; i < i1; i += blockDim.x) {
        float sacc = 0.f;
        for (int pr = 0; pr < world; ++pr) sacc += __ldcv(peers.grads[pr] + i);     // volatile: peer data, never from a stale L1 line
        red[i] = sacc;
        if (i < n) { const float g = sacc * gs; a0 = fmaf(g, g, a0); }
    }
    double acc[1] = {(double)a0};
    block_sum_d<1>(acc, sm);
    if (threadIdx.x == 0) nrm_part[blockIdx.x] = acc[0];
    // ---- 2. grid barrier (monotonic counter) ----
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        grid_barrier_arrive_wait(grid_bar);
    }
    __syncthreads();
    // ---- 3. clip + Adam on my slice ----
    double nsqv[1] = {threadIdx.x < gridDim.x ? __ldcg(nrm_part + threadIdx.x) : 0.0};     // gridDim.x <= 128 <= blockDim.x
    block_sum_d<1>(nsqv, sm);
    const float total_norm = (float)sqrt(nsqv[0]);
    float coef = 1.0f;
    if (c.truncate_grads) coef = fminf((float)c.grad_norm / (total_norm + 1e-6f), 1.0f);
    const float b1 = (float)c.beta1, b2 = (float)c.beta2;
    const double bc1 = 1.0 - p1, bc2 = 1.0 - p2;
    const float step_size = (float)(lr / bc1);
    const float bc2_sqrt = (float)sqrt(bc2);
    const float eps = (float)c.eps, wd = (float)c.weight_decay;
    for (int i = i0 + threadIdx.x; i < min(i1, n); i += blockDim.x)
        adam_update_one(i, __ldcg(red + i) * gs, c.truncate_grads, coef, params, exp_avg, exp_avg_sq, b1, b2, step_size, bc2_sqrt, eps, wd,
                        wpack, tab);
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) is_last = (atomicAdd(counter, 1) == (int)gridDim.x - 1);
    __syncthreads();
    if (is_last && threadIdx.x == 0) {
        double new_lr = lr;
        if (c.adaptive_lr) {
            const double kl = (double)(__ldcg(red + n) * gs);
            new_lr = lr_schedule_step(lr, kl, c, state_d);
        }
        state_d[0] = new_lr; state_d[1] = step; state_d[2] = p1; state_d[3] = p2;
        if (stats_out) { stats_out[B200RL_STAT_LR] = (float)lr; stats_out[B200RL_STAT_GNORM] = total_norm; stats_out[B200RL_STAT_KL] = __ldcg(red + n) * gs; }
        *seq_ptr = seq;
        *counter = 0;
    }
    if (is_last) obs_merge_tail(om);
}

// Opt-in stage timing of reduce_adam_kernel (tools/tc_stage_timing.py --build compiles a variant with -DB200RL_TC_TIMING): thread 0 of
// CTA 0 stamps clock64() at the phase boundaries.  Never compiled into the product library.
#ifdef B200RL_TC_TIMING
__device__ long long g_ra_stamp[32];
#define RA_STAMP(i) do { if (blockIdx.x == 0 && threadIdx.x == 0) g_ra_stamp[i] = clock64(); } while (0)
extern "C" B200RL_EXPORT int b200rl_debug_ra_stamps(long long* host_out) {
    return (int)cudaMemcpyFromSymbol(host_out, g_ra_stamp, sizeof(long long) * 32);
}
#else
#define RA_STAMP(i) do {} while (0)
#endif

// =====================================================================================================================
// Single-GPU fused tail of a minibatch: split-gradient reduction + loss finalisation + clip + Adam (+ packed-weight refresh,
// LR schedule, next-minibatch obs merge) in ONE launch -- replaces reduce_finalize_kernel + adam_step_kernel when there is
// no cross-rank exchange in between.  The reduced gradient never makes a second trip: each CTA sums ITS slice of the flat
// gradient over all splits (fixed order => deterministic), publishes its sum-of-squares partial, crosses one grid barrier
// (grid <= #SMs, one CTA per SM, all co-resident) and updates the same slice.
//
// MULTI = true is the multi-GPU edition: `grads` is this rank's CUDA-IPC mapped exchange buffer (n gradient entries + the KL
// slot at index n).  After a CTA has reduced ITS slice over the splits it publishes "slice b of step seq is ready" to the same
// CTA index on every peer (st.release.sys into per-CTA flags) and waits for the peers' slice b, then sums the slice over all
// ranks in fixed rank order straight from peer memory (bit-identical on every rank).  No rank-wide barrier and no second
// kernel: split reduction, all-reduce, clip and Adam are one launch, and the exchange of slice b overlaps with the split
// reduction of the other slices.  Buffers alternate by update parity: a CTA only reaches step s+1's wait after every peer's
// CTA b finished reading step s, so writing the same parity again at step s+2 cannot overtake a reader.
constexpr int PEER_FLAG_STRIDE = 160;     // u64 flags per source rank (>= max grid of this kernel)
struct PeerStage {
    PeerPtrs peers;                       // grads[r]: rank r's exchange buffer (this parity); flags[r]: rank r's per-CTA flag array
    int world, rank;
    unsigned long long* my_flags;         // [world][PEER_FLAG_STRIDE]
    unsigned long long* seq_ptr;
    float* red;                           // [n + 1] all-reduced gradient + KL (local)
};

template <bool MULTI>
__global__ void __launch_bounds__(1024) reduce_adam_kernel(const float* __restrict__ part, int n_splits, int64_t split_stride,
                                                          const double* __restrict__ lpart, int n_lpart, int lstride, int A,
                                                          const float* __restrict__ entropy_coef_dev, float* __restrict__ stats,
                                                          float* __restrict__ kl_out, float* __restrict__ grads, float* __restrict__ params,
                                                          float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq, int n, double* state_d,
                                                          OptCfgDev c, int* counter, double* __restrict__ nrm_part, unsigned long long* grid_bar,
                                                          unsigned char* __restrict__ wpack, PackTabDev tab, ObsMergeDev om, int kg_log2, int per, int vec4, PeerStage ps) {
    __shared__ double sm[32];
    __shared__ double smf[256];
    __shared__ float4 sred4[1024];
    double* smf32 = reinterpret_cast<double*>(sred4);       // 1024 doubles = 8 KB of the 16 KB reduction scratch (used before it)
    __shared__ int is_last;
    const int tid = threadIdx.x;
    RA_STAMP(0);      // kernel start
    pdl_sync();
    const double lr = state_d[0];
    const double step = state_d[1] + 1.0;
    const double p1 = (state_d[2] > 0.0 ? state_d[2] : 1.0) * c.beta1;
    const double p2 = (state_d[3] > 0.0 ? state_d[3] : 1.0) * c.beta2;
    const float gs = (float)c.grad_scale;
    const int i0 = min(blockIdx.x * per, n), i1 = min(i0 + per, n);      // per: slice length (a multiple of 4 when vec4)
    float a0 = 0.f;
    unsigned long long seq = 0ull;
    if (MULTI) seq = *ps.seq_ptr + 1ull;       // advanced by the last CTA at the very end, after every CTA has read it
    // ---- 1a. one CTA: loss partials -> stats, KL slot, d_logstd (= gradient entries [0, A)).  Single GPU: the last CTA (its
    //      slice is the shortest); multi GPU: CTA 0, the owner of the slice that contains [0, A) and publisher of the KL slot ----
    if (blockIdx.x == (MULTI ? 0u : gridDim.x - 1)) {
        // all 1024 threads: slot = tid % 32, 32 row groups -> at most ceil(n_lpart / 32) dependent loads per thread (it was 37 with 4
        // groups: this CTA is the one every other CTA waits for at the grid barrier); fixed summation order => deterministic
        const int slots = LOSS_NSC + A;              // <= 24
        {
            const int slot = tid & 31, grp = tid >> 5;
            double s = 0.0;
            if (slot < slots)
                for (int p = grp; p < n_lpart; p += 32) s += lpart[(int64_t)p * lstride + slot];
            smf32[tid] = s;
        }
        __syncthreads();
        if (tid < 256) {      // 8 partial sums per slot
            const int slot = tid & 31, g8 = tid >> 5;
            smf[tid] = (smf32[(4 * g8) * 32 + slot] + smf32[(4 * g8 + 1) * 32 + slot]) + (smf32[(4 * g8 + 2) * 32 + slot] + smf32[(4 * g8 + 3) * 32 + slot]);
        }
        __syncthreads();
        if (tid < slots)
            smf[tid] = ((smf[tid] + smf[32 + tid]) + (smf[64 + tid] + smf[96 + tid])) + ((smf[128 + tid] + smf[160 + tid]) + (smf[192 + tid] + smf[224 + tid]));
        __syncthreads();
        if (tid == 0) {
            stats[B200RL_STAT_ALOSS] = (float)smf[0];
            stats[B200RL_STAT_CLOSS] = (float)smf[1];
            stats[B200RL_STAT_ENTROPY] = (float)smf[2];
            stats[B200RL_STAT_BLOSS] = (float)smf[3];
            stats[B200RL_STAT_KL] = (float)smf[4];
            if (kl_out) *kl_out = (float)smf[4];
            stats[B200RL_STAT_SUMMASK] = (float)smf[5];
            stats[B200RL_STAT_CLIPFRAC] = (float)(smf[6] / fmax(smf[5], 1.0));
        }
        if (tid < A) {
            const double ec = (double)__ldg(entropy_coef_dev);
            const float g = (float)(smf[LOSS_NSC + tid] - ec * smf[7]);
            grads[tid] = g;
            a0 = (g * gs) * (g * gs);
        }
    }
    RA_STAMP(1);      // loss finalisation done (CTA 0 does none in the single-GPU edition: it is the last CTA's job)
    // ---- 1b. my slice of the flat gradient: sum over the splits, KG k-groups per element ----
    const uint64_t pol = tc::l2_policy_first();       // the split rows are read once, here
    if (vec4) {
        // 16-byte edition (split rows and slice bounds are 4-float aligned): 4x the bytes in flight per thread -- the pass is
        // latency-bound (~232 KB of L2-resident partials per CTA).  Entries < A or >= n inside a group are loaded but ignored.
        const int KG = 1 << kg_log2, EPB = 1024 >> kg_log2;          // EPB float4 groups per pass
        const int el = tid & (EPB - 1), kg = tid >> (10 - kg_log2);
        for (int base = i0; base < i1; base += 4 * EPB) {
            const int i = base + 4 * el;
            const bool on = i < i1;
            float4 s0 = make_float4(0.f, 0.f, 0.f, 0.f), s1 = s0, s2 = s0, s3 = s0;
            if (on) {
                const float* src = part + i;
                int k = kg;
                for (; k + 3 * KG < n_splits; k += 4 * KG) {
                    const float4 v0 = tc::ldcg_hint(reinterpret_cast<const float4*>(src + (int64_t)k * split_stride), pol);
                    const float4 v1 = tc::ldcg_hint(reinterpret_cast<const float4*>(src + (int64_t)(k + KG) * split_stride), pol);
                    const float4 v2 = tc::ldcg_hint(reinterpret_cast<const float4*>(src + (int64_t)(k + 2 * KG) * split_stride), pol);
                    const float4 v3 = tc::ldcg_hint(reinterpret_cast<const float4*>(src + (int64_t)(k + 3 * KG) * split_stride), pol);
                    s0.x += v0.x; s0.y += v0.y; s0.z += v0.z; s0.w += v0.w;
                    s1.x += v1.x; s1.y += v1.y; s1.z += v1.z; s1.w += v1.w;
                    s2.x += v2.x; s2.y += v2.y; s2.z += v2.z; s2.w += v2.w;
                    s3.x += v3.x; s3.y += v3.y; s3.z += v3.z; s3.w += v3.w;
                }
                for (; k < n_splits; k += KG) {
                    const float4 v0 = tc::ldcg_hint(reinterpret_cast<const float4*>(src + (int64_t)k * split_stride), pol);
                    s0.x += v0.x; s0.y += v0.y; s0.z += v0.z; s0.w += v0.w;
                }
            }
            sred4[tid] = make_float4((s0.x + s1.x) + (s2.x + s3.x), (s0.y + s1.y) + (s2.y + s3.y), (s0.z + s1.z) + (s2.z + s3.z),
                                     (s0.w + s1.w) + (s2.w + s3.w));
            __syncthreads();
            if (on && kg == 0) {
                float4 g = sred4[el];
                for (int j = 1; j < KG; ++j) { const float4 t = sred4[j * EPB + el]; g.x += t.x; g.y += t.y; g.z += t.z; g.w += t.w; }
                const float gv[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
                for (int cc = 0; cc < 4; ++cc) {
                    if (i + cc >= A && i + cc < i1) {
                        grads[i + cc] = gv[cc];
                        a0 = fmaf(gv[cc] * gs, gv[cc] * gs, a0);
                    }
                }
            }
            __syncthreads();
        }
    } else {
        float* sred = reinterpret_cast<float*>(sred4);
        const int KG = 1 << kg_log2, EPB = 1024 >> kg_log2;
        const int el = tid & (EPB - 1), kg = tid >> (10 - kg_log2);
        for (int base = i0; base < i1; base += EPB) {
            const int i = base + el;
            const bool on = i < i1 && i >= A;
            float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
            if (on) {
                const float* src = part + i;
                int k = kg;
                for (; k + 3 * KG < n_splits; k += 4 * KG) {
                    s0 += tc::ldcg_hint(src + (int64_t)k * split_stride, pol);
                    s1 += tc::ldcg_hint(src + (int64_t)(k + KG) * split_stride, pol);
                    s2 += tc::ldcg_hint(src + (int64_t)(k + 2 * KG) * split_stride, pol);
                    s3 += tc::ldcg_hint(src + (int64_t)(k + 3 * KG) * split_stride, pol);
                }
                for (; k < n_splits; k += KG) s0 += tc::ldcg_hint(src + (int64_t)k * split_stride, pol);
            }
            sred[tid] = (s0 + s1) + (s2 + s3);
            __syncthreads();
            if (on && kg == 0) {
                float g = sred[el];
                for (int j = 1; j < KG; ++j) g += sred[j * EPB + el];
                grads[i] = g;
                a0 = fmaf(g * gs, g * gs, a0);
            }
            __syncthreads();
        }
    }
    // ---- 1b'. this CTA was the only reader of its slice of every split row, and every load of it has returned (the sums are in
    //      shared memory, behind the pass's barrier): drop those lines from L2 instead of writing them back.  Only the 128-byte lines
    //      that lie wholly inside the slice, so that a neighbouring CTA's slice never loses a line it has yet to read.  The next
    //      writer is the backward kernel's flush.  Multi-GPU: `part` is this rank's own; the exchange buffers are left alone.
    if (i1 > i0) {
        const int warp = tid >> 5;
        for (int k = warp; k < n_splits; k += 32) {
            const uintptr_t a = reinterpret_cast<uintptr_t>(part + (int64_t)k * split_stride + i0),
                            b = reinterpret_cast<uintptr_t>(part + (int64_t)k * split_stride + i1);
            const uintptr_t lo = (a + 127) & ~(uintptr_t)127, hi = b & ~(uintptr_t)127;
            if (hi > lo) tc::l2_discard(reinterpret_cast<void*>(lo), hi - lo);
        }
    }
    if (MULTI) {
        // ---- 1c. exchange: publish my slice, wait for the same slice of every peer, sum over ranks from peer memory ----
        __threadfence_system();
        __syncthreads();
        if (tid < ps.world) st_release_sys(ps.peers.flags[tid] + (size_t)ps.rank * PEER_FLAG_STRIDE + blockIdx.x, seq);
        if (tid < ps.world) {
            while (ld_acquire_sys(ps.my_flags + (size_t)tid * PEER_FLAG_STRIDE + blockIdx.x) < seq) { }
        }
        __syncthreads();
        a0 = 0.f;                               // the norm is the norm of the all-reduced gradient
        for (int i = i0 + tid; i < i1; i += blockDim.x) {
            float sacc = 0.f;
            for (int pr = 0; pr < ps.world; ++pr) sacc += __ldcv(ps.peers.grads[pr] + i);     // volatile: peer data, never a stale L1 line
            ps.red[i] = sacc;
            a0 = fmaf(sacc * gs, sacc * gs, a0);
        }
        if (blockIdx.x == 0 && tid == 0) {
            float sacc = 0.f;
            for (int pr = 0; pr < ps.world; ++pr) sacc += __ldcv(ps.peers.grads[pr] + n);     // KL slot
            ps.red[n] = sacc;
        }
    }
    RA_STAMP(2);      // split reduction (and peer exchange) done
    const float* gsrc = MULTI ? ps.red : grads;
    double acc[1] = {(double)a0};
    block_sum_d<1>(acc, sm);
    if (tid == 0) nrm_part[blockIdx.x] = acc[0];
    // ---- 2. grid barrier (monotonic counter) ----
    __threadfence();
    __syncthreads();
    if (tid == 0) {
        grid_barrier_arrive_wait(grid_bar);
    }
    __syncthreads();
    RA_STAMP(3);      // grid barrier passed
    // ---- 3. clip + Adam on my slice ----
    double nsqv[1] = {tid < gridDim.x ? __ldcg(nrm_part + tid) : 0.0};     // gridDim.x <= 132 <= blockDim.x
    block_sum_d<1>(nsqv, sm);
    const float total_norm = (float)sqrt(nsqv[0]);
    float coef = 1.0f;
    if (c.truncate_grads) coef = fminf((float)c.grad_norm / (total_norm + 1e-6f), 1.0f);
    const float b1 = (float)c.beta1, b2 = (float)c.beta2;
    const double bc1 = 1.0 - p1, bc2 = 1.0 - p2;
    const float step_size = (float)(lr / bc1);
    const float bc2_sqrt = (float)sqrt(bc2);
    const float eps = (float)c.eps, wd = (float)c.weight_decay;
    for (int i = i0 + tid; i < i1; i += blockDim.x)
        adam_update_one(i, __ldcg(gsrc + i) * gs, c.truncate_grads, coef, params, exp_avg, exp_avg_sq, b1, b2, step_size, bc2_sqrt, eps, wd,
                        wpack, tab);
    RA_STAMP(4);      // Adam on my slice done
    __threadfence();
    __syncthreads();
    if (tid == 0) is_last = (atomicAdd(counter, 1) == (int)gridDim.x - 1);
    __syncthreads();
    if (is_last && tid == 0) {
        double new_lr = lr;
        const float* klp = MULTI ? ps.red + n : kl_out;      // summed over ranks by the exchange -> mean via grad_scale (a2c_common.py:1559-1561)
        if (c.adaptive_lr && klp) {
            const double kl = (double)(__ldcg(klp) * gs);
            new_lr = lr_schedule_step(lr, kl, c, state_d);
        }
        state_d[0] = new_lr; state_d[1] = step; state_d[2] = p1; state_d[3] = p2;
        stats[B200RL_STAT_LR] = (float)lr; stats[B200RL_STAT_GNORM] = total_norm;
        if (MULTI) { stats[B200RL_STAT_KL] = __ldcg(ps.red + n) * gs; *ps.seq_ptr = seq; }
        *counter = 0;
    }
    if (is_last) obs_merge_tail(om);
    RA_STAMP(5);      // kernel end (CTA 0; the last CTA also runs the obs-merge tail)
}

}  // namespace

static ObsMergeDev make_obs_merge(const b200rl_obs_merge* h) {
    ObsMergeDev o{};
    if (h && h->mbmom) {
        o.mbmom = h->mbmom; o.shift = h->shift; o.D = h->D; o.n_rows = h->n_rows; o.mean = h->mean; o.var = h->var;
        o.count = (long long*)h->count; o.mean_f32 = h->mean_f32; o.std_f32 = h->std_f32; o.eps = h->eps;
    }
    return o;
}

static int make_pack_tab(const b200rl_pack_table* tab_host, PackTabDev& tab) {
    if (!tab_host) return B200RL_OK;
    if (tab_host->n_seg < 0 || tab_host->n_seg > 4) return B200RL_EINVAL;
    tab.n_seg = tab_host->n_seg;
    for (int i = 0; i < tab.n_seg; ++i) {
        tab.off[i] = tab_host->flat_off[i]; tab.R[i] = tab_host->rows[i]; tab.C[i] = tab_host->cols[i];
        tab.CS[i] = tab_host->cs_bytes[i]; tab.dst[i] = tab_host->dst_off[i];
    }
    return B200RL_OK;
}
static OptCfgDev make_opt_cfg(const b200rl_opt_cfg* h) {
    OptCfgDev c;
    c.beta1 = h->beta1; c.beta2 = h->beta2; c.eps = h->eps; c.weight_decay = h->weight_decay;
    c.grad_norm = h->grad_norm; c.kl_threshold = h->kl_threshold; c.min_lr = h->min_lr;
    c.max_lr = h->max_lr; c.lr_multiplier = h->lr_multiplier; c.grad_scale = h->grad_scale;
    c.truncate_grads = h->truncate_grads; c.adaptive_lr = h->adaptive_lr;
    return c;
}

static int reduce_adam_launch(const float* part, int n_splits, int64_t split_stride, const double* loss_partials, int n_loss_partials, int A,
                              const float* entropy_coef_dev, float* stats, float* kl_out, float* grads, float* params, float* exp_avg,
                              float* exp_avg_sq, int n, double* state_d, const b200rl_opt_cfg* cfg_host, int* counter, double* nrm_part,
                              int nrm_part_len, void* grid_bar, void* wpack, const b200rl_pack_table* tab_host,
                              const b200rl_obs_merge* merge_next_host, const PeerStage* ps, void* stream) {
    if (!part || !loss_partials || !entropy_coef_dev || !stats || !grads || !params || !exp_avg || !exp_avg_sq || !state_d || !cfg_host ||
        !counter || !nrm_part || !grid_bar)
        return B200RL_EINVAL;
    if (n <= 0 || n_splits <= 0 || n_loss_partials <= 0 || A <= 0 || A + 1 > 16 || A >= n) return B200RL_EINVAL;
    if ((wpack != nullptr) != (tab_host != nullptr)) return B200RL_EINVAL;
    PackTabDev tab{};
    if (make_pack_tab(tab_host, tab) != B200RL_OK) return B200RL_EINVAL;
    int blocks = (n + 255) / 256;         // a slice of >= 256 entries per CTA; all CTAs must be co-resident (grid barrier)
    if (blocks > 132) blocks = 132;
    if (blocks > nrm_part_len || blocks > PEER_FLAG_STRIDE) return B200RL_EINVAL;
    int per = (n + blocks - 1) / blocks;
    // 16-byte loads when every split row and every slice start is 4-float aligned
    const int vec4 = (split_stride % 4 == 0) && split_stride >= (int64_t)(n + 3) / 4 * 4 && ((reinterpret_cast<uintptr_t>(part) & 15) == 0);
    if (vec4) per = (per + 3) / 4 * 4;
    const int units = vec4 ? per / 4 : per;      // elements (or float4 groups) of one slice
    int kg_log2 = 0;                      // k-groups per unit: as many as fit in one 1024-thread pass over the slice
    while (kg_log2 < 3 && (1024 >> (kg_log2 + 1)) >= units) ++kg_log2;
    cudaError_t le;
    if (ps)
        le = launch_k(reduce_adam_kernel<true>, dim3(blocks), dim3(1024), 0, as_stream(stream), part, n_splits, split_stride, loss_partials,
                      n_loss_partials, b200rl_loss_partial_stride(), A, entropy_coef_dev, stats, kl_out, grads, params, exp_avg, exp_avg_sq, n,
                      state_d, make_opt_cfg(cfg_host), counter, nrm_part, (unsigned long long*)grid_bar, (unsigned char*)wpack, tab,
                      make_obs_merge(merge_next_host), kg_log2, per, vec4, *ps);
    else
        le = launch_k(reduce_adam_kernel<false>, dim3(blocks), dim3(1024), 0, as_stream(stream), part, n_splits, split_stride, loss_partials,
                      n_loss_partials, b200rl_loss_partial_stride(), A, entropy_coef_dev, stats, kl_out, grads, params, exp_avg, exp_avg_sq, n,
                      state_d, make_opt_cfg(cfg_host), counter, nrm_part, (unsigned long long*)grid_bar, (unsigned char*)wpack, tab,
                      make_obs_merge(merge_next_host), kg_log2, per, vec4, PeerStage{});
    if (le != cudaSuccess) return (int)le;
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_reduce_adam_f32(const float* part, int n_splits, int64_t split_stride, const double* loss_partials,
                                         int n_loss_partials, int A, const float* entropy_coef_dev, float* stats, float* kl_out,
                                         float* grads, float* params, float* exp_avg, float* exp_avg_sq, int n, double* state_d,
                                         const b200rl_opt_cfg* cfg_host, int* counter, double* nrm_part, int nrm_part_len, void* grid_bar,
                                         void* wpack, const b200rl_pack_table* tab_host, const b200rl_obs_merge* merge_next_host,
                                         void* stream) {
    return reduce_adam_launch(part, n_splits, split_stride, loss_partials, n_loss_partials, A, entropy_coef_dev, stats, kl_out, grads, params,
                              exp_avg, exp_avg_sq, n, state_d, cfg_host, counter, nrm_part, nrm_part_len, grid_bar, wpack, tab_host,
                              merge_next_host, nullptr, stream);
}

B200RL_EXPORT int b200rl_reduce_allreduce_adam_f32(const float* part, int n_splits, int64_t split_stride, const double* loss_partials,
                                                   int n_loss_partials, int A, const float* entropy_coef_dev, float* stats,
                                                   const void* const* peer_grads_host, void* const* peer_cta_flags_host, int world, int rank,
                                                   void* my_cta_flags, void* seq_ptr, float* red, float* params, float* exp_avg,
                                                   float* exp_avg_sq, int n, double* state_d, const b200rl_opt_cfg* cfg_host, int* counter,
                                                   double* nrm_part, int nrm_part_len, void* grid_bar, void* wpack,
                                                   const b200rl_pack_table* tab_host, const b200rl_obs_merge* merge_next_host, void* stream) {
    if (!peer_grads_host || !peer_cta_flags_host || world < 1 || world > 8 || rank < 0 || rank >= world || !my_cta_flags || !seq_ptr || !red)
        return B200RL_EINVAL;
    PeerStage ps{};
    for (int i = 0; i < world; ++i) {
        if (!peer_grads_host[i] || !peer_cta_flags_host[i]) return B200RL_EINVAL;
        ps.peers.grads[i] = (const float*)peer_grads_host[i];
        ps.peers.flags[i] = (unsigned long long*)peer_cta_flags_host[i];
    }
    ps.world = world; ps.rank = rank; ps.my_flags = (unsigned long long*)my_cta_flags; ps.seq_ptr = (unsigned long long*)seq_ptr; ps.red = red;
    float* own = const_cast<float*>(ps.peers.grads[rank]);       // this rank's exchange buffer: [n] gradient entries + the KL slot
    return reduce_adam_launch(part, n_splits, split_stride, loss_partials, n_loss_partials, A, entropy_coef_dev, stats, own + n, own, params,
                              exp_avg, exp_avg_sq, n, state_d, cfg_host, counter, nrm_part, nrm_part_len, grid_bar, wpack, tab_host,
                              merge_next_host, &ps, stream);
}

B200RL_EXPORT int b200rl_adam_step_f32(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int n,
                                       double* state_d, const float* kl_dev, const b200rl_opt_cfg* cfg_host,
                                       float* stats_out, int* counter, void* wpack, const b200rl_pack_table* tab_host,
                                       const b200rl_obs_merge* merge_next_host, void* stream) {
    if (!params || !grads || !exp_avg || !exp_avg_sq || !state_d || !cfg_host || !counter || n <= 0) return B200RL_EINVAL;
    if ((wpack != nullptr) != (tab_host != nullptr)) return B200RL_EINVAL;
    PackTabDev tab{};
    if (tab_host) {
        if (tab_host->n_seg < 0 || tab_host->n_seg > 4) return B200RL_EINVAL;
        tab.n_seg = tab_host->n_seg;
        for (int i = 0; i < tab.n_seg; ++i) {
            tab.off[i] = tab_host->flat_off[i]; tab.R[i] = tab_host->rows[i]; tab.C[i] = tab_host->cols[i];
            tab.CS[i] = tab_host->cs_bytes[i]; tab.dst[i] = tab_host->dst_off[i];
        }
    }
    OptCfgDev c;
    c.beta1 = cfg_host->beta1; c.beta2 = cfg_host->beta2; c.eps = cfg_host->eps; c.weight_decay = cfg_host->weight_decay;
    c.grad_norm = cfg_host->grad_norm; c.kl_threshold = cfg_host->kl_threshold; c.min_lr = cfg_host->min_lr;
    c.max_lr = cfg_host->max_lr; c.lr_multiplier = cfg_host->lr_multiplier; c.grad_scale = cfg_host->grad_scale;
    c.truncate_grads = cfg_host->truncate_grads; c.adaptive_lr = cfg_host->adaptive_lr;
    int blocks = (n + 2047) / 2048;       // two elements per thread in the update; every CTA re-derives the norm from L2
    if (blocks > 132) blocks = 132;
    if (blocks < 1) blocks = 1;
    cudaError_t le = launch_k(adam_step_kernel, dim3(blocks), dim3(1024), 0, as_stream(stream), params, grads, exp_avg, exp_avg_sq, n, state_d, kl_dev, c, stats_out,
                                                            counter, (unsigned char*)wpack, tab, make_obs_merge(merge_next_host));
    if (le != cudaSuccess) return (int)le;
    return B200RL_OK;
}

// One adaptive-KL scheduler step on a given base LR, outside an optimiser launch (state_d[0] = schedule(base_lr, kl * kl_scale)).
// Used once after a checkpoint restore: the reference's first optimiser step then runs on the checkpoint's optimizer LR while its
// scheduler continues from the agent's own last_lr (a2c_common.py:852-866 loads the optimizer state but not last_lr).
__global__ void lr_schedule_apply_kernel(double* state_d, const float* __restrict__ kl_dev, double kl_scale, double base_lr, OptCfgDev c) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        c.adaptive_lr = 1;
        state_d[0] = lr_schedule_step(base_lr, (double)(*kl_dev) * kl_scale, c, state_d);
    }
}

B200RL_EXPORT int b200rl_lr_schedule_apply(double* state_d, const float* kl_dev, double kl_scale, double base_lr,
                                           const b200rl_opt_cfg* cfg_host, void* stream) {
    if (!state_d || !kl_dev || !cfg_host) return B200RL_EINVAL;
    lr_schedule_apply_kernel<<<1, 32, 0, as_stream(stream)>>>(state_d, kl_dev, kl_scale, base_lr, make_opt_cfg(cfg_host));
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

// ---- CUDA-IPC plumbing for the peer-mapped gradient buffers (multi-GPU, one process per GPU) ----------------------
B200RL_EXPORT int b200rl_ipc_alloc(int64_t bytes, void** dev_ptr_out_host, void* handle64_out_host) {
    if (bytes <= 0 || !dev_ptr_out_host || !handle64_out_host) return B200RL_EINVAL;
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, (size_t)bytes);
    if (e != cudaSuccess) return (int)e;
    e = cudaMemset(p, 0, (size_t)bytes);
    if (e != cudaSuccess) return (int)e;
    cudaIpcMemHandle_t h;
    e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) return (int)e;
    static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
    memcpy(handle64_out_host, &h, 64);
    *dev_ptr_out_host = p;
    return B200RL_OK;
}
B200RL_EXPORT int b200rl_ipc_open(const void* handle64_host, void** dev_ptr_out_host) {
    if (!handle64_host || !dev_ptr_out_host) return B200RL_EINVAL;
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64_host, 64);
    void* p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) return (int)e;
    *dev_ptr_out_host = p;
    return B200RL_OK;
}
B200RL_EXPORT int b200rl_ipc_close(void* p) { return p ? (int)cudaIpcCloseMemHandle(p) : B200RL_EINVAL; }
B200RL_EXPORT int b200rl_ipc_free(void* p) { return p ? (int)cudaFree(p) : B200RL_EINVAL; }

B200RL_EXPORT int b200rl_allreduce_adam_f32(const void* const* peer_grads_host, void* const* peer_flags_host, int world, int rank,
                                            void* my_flags, void* seq_ptr, float* red, double* nrm_part, int nrm_part_len, void* grid_bar,
                                            float* params, float* exp_avg, float* exp_avg_sq, int n, double* state_d,
                                            const b200rl_opt_cfg* cfg_host, float* stats_out, int* counter, void* wpack,
                                            const b200rl_pack_table* tab_host, const b200rl_obs_merge* merge_next_host, void* stream) {
    if (!peer_grads_host || !peer_flags_host || world < 1 || world > 8 || rank < 0 || rank >= world || !my_flags || !seq_ptr || !red ||
        !nrm_part || !grid_bar || !params || !exp_avg || !exp_avg_sq || !state_d || !cfg_host || !counter || n <= 0)
        return B200RL_EINVAL;
    if ((wpack != nullptr) != (tab_host != nullptr)) return B200RL_EINVAL;
    PeerPtrs pp{};
    for (int i = 0; i < world; ++i) {
        if (!peer_grads_host[i] || !peer_flags_host[i]) return B200RL_EINVAL;
        pp.grads[i] = (const float*)peer_grads_host[i];
        pp.flags[i] = (unsigned long long*)peer_flags_host[i];
    }
    PackTabDev tab{};
    if (tab_host) {
        if (tab_host->n_seg < 0 || tab_host->n_seg > 4) return B200RL_EINVAL;
        tab.n_seg = tab_host->n_seg;
        for (int i = 0; i < tab.n_seg; ++i) {
            tab.off[i] = tab_host->flat_off[i]; tab.R[i] = tab_host->rows[i]; tab.C[i] = tab_host->cols[i];
            tab.CS[i] = tab_host->cs_bytes[i]; tab.dst[i] = tab_host->dst_off[i];
        }
    }
    OptCfgDev c;
    c.beta1 = cfg_host->beta1; c.beta2 = cfg_host->beta2; c.eps = cfg_host->eps; c.weight_decay = cfg_host->weight_decay;
    c.grad_norm = cfg_host->grad_norm; c.kl_threshold = cfg_host->kl_threshold; c.min_lr = cfg_host->min_lr;
    c.max_lr = cfg_host->max_lr; c.lr_multiplier = cfg_host->lr_multiplier; c.grad_scale = cfg_host->grad_scale;
    c.truncate_grads = cfg_host->truncate_grads; c.adaptive_lr = cfg_host->adaptive_lr;
    int blocks = (n + 1 + 2047) / 2048;
    if (blocks > 128) blocks = 128;       // all CTAs must be co-resident for the in-kernel grid barrier (132 SMs, 1 CTA/SM)
    if (blocks < 1) blocks = 1;
    if (blocks > nrm_part_len) return B200RL_EINVAL;
    cudaError_t le = launch_k(allreduce_adam_kernel, dim3(blocks), dim3(1024), 0, as_stream(stream), pp, world, rank, (unsigned long long*)my_flags, (unsigned long long*)seq_ptr,
                                                                 red, nrm_part, (unsigned long long*)grid_bar, params, exp_avg, exp_avg_sq, n, state_d, c,
                                                                 stats_out, counter, (unsigned char*)wpack, tab, make_obs_merge(merge_next_host));
    if (le != cudaSuccess) return (int)le;
    return B200RL_OK;
}

#ifdef B200RL_TEST_HOOKS   // test-only host entry points: compiled into tests/libb200rl_testhooks.so (csrc/build.py), not into the product library
// host test entry point: the scheduler step of the optimiser kernels (lr_schedule_step, __host__ __device__) on HOST memory;
// cfg->adaptive_lr selects the mode (1 per minibatch, 2 accumulate, 3 accumulate + step on the mean + reset).  Not in include/b200rl.h.
B200RL_EXPORT double b200rl_hosttest_lr_schedule_step(double lr, double kl, const b200rl_opt_cfg* cfg_host, double* state_d) {
    return lr_schedule_step(lr, kl, make_opt_cfg(cfg_host), state_d);
}
#endif  // B200RL_TEST_HOOKS
