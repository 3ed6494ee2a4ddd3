// Value-only loss head of the central value network (asymmetric critic) -- SURVEY.md 8f rank 1 (algos_torch/central_value.py:276-301
// calc_loss / calc_gradients: loss = masked mean of common_losses.critic_loss).
//
// The per-row arithmetic is __host__ __device__ and is also exercised on the CPU (tests/test_critic_rows_cpu.py); GPU parity:
// tests/test_cv_gpu.py.
#include "common.cuh"

namespace {

// critic_loss of one row (common_losses.py:7-38) and d(loss)/d(value); returns the loss
__host__ __device__ inline float value_loss_row(float val, float old_v, float ret, float e_clip, int clip_value, float& dc) {
    if (clip_value) {
        const float delta = val - old_v;
        const float vpc = old_v + fminf(fmaxf(delta, -e_clip), e_clip);
        const float e1 = val - ret, e2 = vpc - ret;
        const float l1 = e1 * e1, l2 = e2 * e2;
        const float g1 = 2.0f * e1, g2 = (delta >= -e_clip && delta <= e_clip) ? 2.0f * e2 : 0.0f;
        dc = (l1 > l2) ? g1 : ((l1 < l2) ? g2 : 0.5f * (g1 + g2));
        return fmaxf(l1, l2);
    }
    const float e1 = ret - val;
    dc = -2.0f * e1;
    return e1 * e1;
}

struct ValueLossArgs {
    const float* values; int value_ld; const float* old_values_n; const float* returns_n; const float* mask; int rows_per_chunk;
    int64_t chunk_stride; int M; float e_clip; int clip_value; const float* inv_count_dev; float* d_value; int dv_ld;
};

// everything one kernel thread does except the block reduction (__host__ __device__: the arena addressing runs on the CPU too,
// b200rl_hosttest_value_loss_arena).  acc: sum w*c_loss, sum mask, sum w
__host__ __device__ inline void value_loss_thread(const ValueLossArgs& a, int m, double (&acc)[3]) {
    const int c = m / a.rows_per_chunk;
    const int64_t ar = (int64_t)c * a.chunk_stride + (m - c * a.rows_per_chunk);
    const float mk = a.mask ? a.mask[ar] : 1.0f;
    const float w = mk * (a.inv_count_dev ? a.inv_count_dev[0] : (1.0f / (float)a.M));
    float dc;
    const float l = value_loss_row(a.values[(int64_t)m * a.value_ld], a.old_values_n[ar], a.returns_n[ar], a.e_clip, a.clip_value, dc);
    a.d_value[(int64_t)m * a.dv_ld] = w * dc;
    acc[0] = (double)w * l; acc[1] = mk; acc[2] = w;
}

// partial row (8 doubles per block): sum w*c_loss, sum mask, sum w, 0...
__global__ void __launch_bounds__(256) value_loss_kernel(const ValueLossArgs a, double* __restrict__ partials) {
    __shared__ double sm[32 * 3];
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    double acc[3] = {0, 0, 0};
    if (m < a.M) value_loss_thread(a, m, acc);
    block_sum_d<3>(acc, sm);
    if (threadIdx.x == 0) {
        double* p = partials + (int64_t)blockIdx.x * 8;
        p[0] = acc[0]; p[1] = acc[1]; p[2] = acc[2];
#pragma unroll
        for (int i = 3; i < 8; ++i) p[i] = 0.0;
    }
}

// Multi-agent envs (agents = G > 1), central_value.py:224-226: the critic's value of env e (one state row per env), de-normalised with
// the value normaliser when it is on (running_mean_std.py:104-106, as normalize_kernel's denorm), written to the G agent rows e*G .. e*G+G-1
// of the actor's values[t] / last_values.  One thread per agent row.
__global__ void __launch_bounds__(256) cv_value_broadcast_kernel(const float* __restrict__ val, const double* __restrict__ vms_mean,
                                                                 const double* __restrict__ vms_var, int normalize_value,
                                                                 float* __restrict__ out, int N, int G) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= N * G) return;
    float v = val[r / G];
    if (normalize_value) {
        const float m = (float)vms_mean[0], s = __fsqrt_rn(__fadd_rn((float)vms_var[0], 1e-5f));
        v = __fadd_rn(__fmul_rn(s, fminf(fmaxf(v, -5.0f), 5.0f)), m);
    }
    out[r] = v;
}

// central_value.py:235-244 update_multiagent_tensors: the actor's [H, N*G] old values and returns viewed as (N, G, H), transposed to
// (G, N, H) and cut to the first N*H rows = agent 0 of every env; here as the critic's [H, N] arena: dst[t][e] = src[t][e*G].  (The
// reference cuts its dones without the transpose; a feed-forward critic never reads them.)
__global__ void __launch_bounds__(256) cv_gather_agent0_kernel(const float* __restrict__ src_a, const float* __restrict__ src_b,
                                                               float* __restrict__ dst_a, float* __restrict__ dst_b, int H, int N, int G) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)H * N) return;
    const int64_t t = i / N, e = i - t * N;
    const int64_t s = t * N * G + e * G;
    dst_a[i] = src_a[s];
    dst_b[i] = src_b[s];
}

}  // namespace

B200RL_EXPORT int b200rl_value_loss_f32(const float* values, int value_ld, const float* old_values_n, const float* returns_n,
                                        const float* mask, int rows_per_chunk, int64_t chunk_stride, int M, float e_clip, int clip_value,
                                        const float* inv_count_dev, float* d_value, int dv_ld, double* partials, int max_partials,
                                        int* n_blocks_out_host, void* stream) {
    if (!values || !old_values_n || !returns_n || !d_value || !partials || M <= 0 || value_ld <= 0 || dv_ld <= 0 || rows_per_chunk <= 0)
        return B200RL_EINVAL;
    const int blocks = (M + 255) / 256;
    if (n_blocks_out_host) *n_blocks_out_host = blocks;
    if (blocks > max_partials) return B200RL_EINVAL;
    const ValueLossArgs a{values, value_ld, old_values_n, returns_n, mask, rows_per_chunk, chunk_stride, M, e_clip, clip_value, inv_count_dev,
                          d_value, dv_ld};
    value_loss_kernel<<<blocks, 256, 0, as_stream(stream)>>>(a, partials);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_cv_value_broadcast_f32(const float* val, const double* vms_mean, const double* vms_var, int normalize_value,
                                                float* out, int N, int agents, void* stream) {
    if (!val || !out || N <= 0 || agents <= 0) return B200RL_EINVAL;
    if (normalize_value && (!vms_mean || !vms_var)) return B200RL_EINVAL;
    const int64_t rows = (int64_t)N * agents;
    if (rows > INT32_MAX) return B200RL_EINVAL;
    cv_value_broadcast_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, as_stream(stream)>>>(val, vms_mean, vms_var, normalize_value, out, N,
                                                                                           agents);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_cv_gather_agent0_f32(const float* src_a, const float* src_b, float* dst_a, float* dst_b, int H, int N, int agents,
                                              void* stream) {
    if (!src_a || !src_b || !dst_a || !dst_b || H <= 0 || N <= 0 || agents <= 0) return B200RL_EINVAL;
    const int64_t total = (int64_t)H * N;
    cv_gather_agent0_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(src_a, src_b, dst_a, dst_b, H, N, agents);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

#ifdef B200RL_TEST_HOOKS   // test-only host entry points: compiled into tests/libb200rl_testhooks.so (csrc/build.py), not into the product library
// host test entry point (CPU, host arrays): the same row function; not declared in include/b200rl.h, never called by the product
B200RL_EXPORT int b200rl_hosttest_value_loss_rows(const float* values, const float* old_values_n, const float* returns_n, const float* w,
                                                 int M, float e_clip, int clip_value, float* d_value, double* loss_sum) {
    double s = 0.0;
    for (int m = 0; m < M; ++m) {
        float dc;
        const float l = value_loss_row(values[m], old_values_n[m], returns_n[m], e_clip, clip_value, dc);
        d_value[m] = w[m] * dc;
        s += (double)w[m] * l;
    }
    *loss_sum = s;
    return B200RL_OK;
}

// the kernel's per-thread body over HOST arrays laid out like the device arena (arguments of the C-ABI entry point, no stream)
B200RL_EXPORT int b200rl_hosttest_value_loss_arena(const float* values, int value_ld, const float* old_values_n, const float* returns_n,
                                                  const float* mask, int rows_per_chunk, int64_t chunk_stride, int M, float e_clip, int clip_value,
                                                  const float* inv_count, float* d_value, int dv_ld, double* partial8) {
    const ValueLossArgs a{values, value_ld, old_values_n, returns_n, mask, rows_per_chunk, chunk_stride, M, e_clip, clip_value, inv_count, d_value,
                          dv_ld};
    double tot[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int m = 0; m < M; ++m) {
        double acc[3] = {0, 0, 0};
        value_loss_thread(a, m, acc);
        for (int i = 0; i < 3; ++i) tot[i] += acc[i];
    }
    for (int i = 0; i < 8; ++i) partial8[i] = tot[i];
    return B200RL_OK;
}
#endif  // B200RL_TEST_HOOKS
