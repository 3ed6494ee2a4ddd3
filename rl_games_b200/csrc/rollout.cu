// Rollout-step kernels (a2c_common.py:985-1069 play_steps, per env step):
//   policy_head_sample -- mu/value heads, sigma = exp(logstd), a = mu + sigma*eps, neglogp, denormalised
//                         value (models.py:329-364, :58-60), written directly into time-step t of the
//                         experience arena (replaces 8 ExperienceBuffer.update_data copies, experience.py:433-456)
//   post_step          -- reward shaping (tr_helpers.py:33-42), timeout bootstrap (a2c_common.py:1021-1023),
//                         episode accounting and AverageMeter updates without dones.nonzero() host syncs
//                         (a2c_common.py:1027-1051, torch_ext.py:326-352)
//   synth_env_step     -- synthetic on-GPU measurement env (not part of the reference; SURVEY.md 8d)
#include "common.cuh"
#include "loss_math.cuh"

namespace {

constexpr int PT = 128;
constexpr int MAXA = 32;
constexpr int MAXA_SD = 16;   // state-dependent sigma: value + up to 15 mu rows, up to 15 raw-sigma rows

// SD = state-dependent sigma: 1 + 2A head rows (value, mu, raw sigma), sigma per row through sigma_param
template <int MA, bool SD>
__device__ __forceinline__ void policy_head_sample_body(
    const float* __restrict__ a_last, int Hl, const float* __restrict__ Wh, const float* __restrict__ bh,
    const float* __restrict__ logstd, const double* __restrict__ vms_mean, const double* __restrict__ vms_var,
    int normalize_value, const float* __restrict__ noise, uint64_t seed, const uint64_t* __restrict__ rng_epoch_dev,
    uint32_t step_index, float* __restrict__ actions, float* __restrict__ mus, float* __restrict__ sigmas,
    float* __restrict__ neglogp, float* __restrict__ values, float* __restrict__ env_actions, int clip_actions,
    const float* __restrict__ act_low, const float* __restrict__ act_high,
    const uint8_t* __restrict__ dones_cur, uint8_t* __restrict__ dones_out, const float* __restrict__ prev_dones,
    float* __restrict__ valid_out, int N, int A, int values_only, const SigmaCfgDev& scfg) {
    extern __shared__ float smf[];
    const int AH = A + 1;
    const int HR = SD ? 1 + 2 * A : AH;   // head rows
    float* tile = smf;                    // [PT][Hl+1]
    float* sW = tile + PT * (Hl + 1);     // [HR][Hl]
    float* sB = sW + HR * Hl;             // [HR]
    float* sSig = sB + HR;                // sigma[A], logstd[A] (fixed sigma)
    const int tid = threadIdx.x, e0 = blockIdx.x * PT;
    const int rows = min(PT, N - e0);
    for (int i = tid; i < rows * Hl; i += PT) {
        const int r = i / Hl, k = i - r * Hl;
        tile[r * (Hl + 1) + k] = __ldg(a_last + (int64_t)(e0 + r) * Hl + k);
    }
    for (int i = tid; i < HR * Hl; i += PT) sW[i] = __ldg(Wh + i);
    if (tid < HR) sB[tid] = __ldg(bh + tid);
    if (!SD && tid < A) { const float ls = __ldg(logstd + tid); sSig[tid] = expf(ls); sSig[A + tid] = ls; }
    __syncthreads();
    if (tid >= rows) return;
    const int e = e0 + tid;
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
            if (SD && !values_only && j < A) raw[j] = fmaf(a, sW[(AH + j) * Hl + k], raw[j]);
        }
    }
    // value: denorm_value (running_mean_std.py:104-106): sqrt(var+eps)*clamp(v,-5,5)+mean
    float val = head[0];
    if (normalize_value) {
        const float m = (float)vms_mean[0], s = __fsqrt_rn(__fadd_rn((float)vms_var[0], 1e-5f));
        val = __fadd_rn(__fmul_rn(s, fminf(fmaxf(val, -5.0f), 5.0f)), m);
    }
    values[e] = val;
    if (values_only) return;
    // noise
    float eps[MA];
    if (noise) {
#pragma unroll
        for (int j = 0; j < MA; ++j) eps[j] = (j < A) ? __ldg(noise + (int64_t)e * A + j) : 0.f;
    } else {
        const uint64_t ep = rng_epoch_dev ? *rng_epoch_dev : 0ull;
#pragma unroll
        for (int q = 0; q < MA / 4; ++q) {
            if (q * 4 < A) {
                const Philox4 r = philox4x32_10((uint64_t)e, (ep << 20) | ((uint64_t)step_index << 4) | (uint64_t)q, seed);
                box_muller(r.x, r.y, eps[q * 4 + 0], eps[q * 4 + 1]);
                box_muller(r.z, r.w, eps[q * 4 + 2], eps[q * 4 + 3]);
            }
        }
    }
    float sumz2 = 0.f, sumls = 0.f;
#pragma unroll
    for (int j = 0; j < MA; ++j) {
        if (j < A) {
            float sg_sd = 0.f, ls_sd = 0.f, unused;
            if (SD) sigma_param(raw[j], scfg, sg_sd, ls_sd, unused);
            const float mu = head[1 + j], sg = SD ? sg_sd : sSig[j];
            const float act = __fadd_rn(mu, __fmul_rn(sg, eps[j]));
            const float z = (act - mu) / sg;
            sumz2 += z * z;
            sumls += SD ? ls_sd : sSig[A + j];
            actions[(int64_t)e * A + j] = act;
            mus[(int64_t)e * A + j] = mu;
            sigmas[(int64_t)e * A + j] = sg;
            if (env_actions) {
                float ea = act;
                if (clip_actions) {
                    // a2c_common.py:1500-1510 + :144-148
                    const float lo = __ldg(act_low + j), hi = __ldg(act_high + j);
                    ea = fminf(fmaxf(act, -1.0f), 1.0f) * ((hi - lo) * 0.5f) + (hi + lo) * 0.5f;
                }
                env_actions[(int64_t)e * A + j] = ea;
            }
        }
    }
    neglogp[e] = 0.5f * sumz2 + 0.9189385332046727f * (float)A + sumls;
    if (dones_out) dones_out[e] = dones_cur[e];
    if (valid_out) valid_out[e] = prev_dones ? (1.0f - prev_dones[e]) : 1.0f;
}

__global__ void __launch_bounds__(PT) policy_head_sample_kernel(
    const float* __restrict__ a_last, int Hl, const float* __restrict__ Wh, const float* __restrict__ bh,
    const float* __restrict__ logstd, const double* __restrict__ vms_mean, const double* __restrict__ vms_var,
    int normalize_value, const float* __restrict__ noise, uint64_t seed, const uint64_t* __restrict__ rng_epoch_dev,
    uint32_t step_index, float* __restrict__ actions, float* __restrict__ mus, float* __restrict__ sigmas,
    float* __restrict__ neglogp, float* __restrict__ values, float* __restrict__ env_actions, int clip_actions,
    const float* __restrict__ act_low, const float* __restrict__ act_high,
    const uint8_t* __restrict__ dones_cur, uint8_t* __restrict__ dones_out, const float* __restrict__ prev_dones,
    float* __restrict__ valid_out, int N, int A, int values_only) {
    policy_head_sample_body<MAXA, false>(a_last, Hl, Wh, bh, logstd, vms_mean, vms_var, normalize_value, noise, seed, rng_epoch_dev,
                                         step_index, actions, mus, sigmas, neglogp, values, env_actions, clip_actions, act_low, act_high,
                                         dones_cur, dones_out, prev_dones, valid_out, N, A, values_only, SigmaCfgDev{});
}

// state-dependent sigma (A <= 15)
__global__ void __launch_bounds__(PT) policy_head_sample_sd_kernel(
    const float* __restrict__ a_last, int Hl, const float* __restrict__ Wh, const float* __restrict__ bh,
    SigmaCfgDev scfg, const double* __restrict__ vms_mean, const double* __restrict__ vms_var,
    int normalize_value, const float* __restrict__ noise, uint64_t seed, const uint64_t* __restrict__ rng_epoch_dev,
    uint32_t step_index, float* __restrict__ actions, float* __restrict__ mus, float* __restrict__ sigmas,
    float* __restrict__ neglogp, float* __restrict__ values, float* __restrict__ env_actions, int clip_actions,
    const float* __restrict__ act_low, const float* __restrict__ act_high,
    const uint8_t* __restrict__ dones_cur, uint8_t* __restrict__ dones_out, const float* __restrict__ prev_dones,
    float* __restrict__ valid_out, int N, int A, int values_only) {
    policy_head_sample_body<MAXA_SD, true>(a_last, Hl, Wh, bh, nullptr, vms_mean, vms_var, normalize_value, noise, seed, rng_epoch_dev,
                                           step_index, actions, mus, sigmas, neglogp, values, env_actions, clip_actions, act_low, act_high,
                                           dones_cur, dones_out, prev_dones, valid_out, N, A, values_only, scfg);
}

struct ShaperDev {
    float scale_value, shift_value, min_val, max_val, gamma;
    int log_val, value_bootstrap;
};

// scratch: [n_blocks][4] doubles {count, sum_r, sum_sr, sum_len}
template <typename DT>
__global__ void __launch_bounds__(256) post_step_kernel(
    const float* __restrict__ rewards, const DT* __restrict__ dones, const void* __restrict__ time_outs, int time_outs_kind,
    const float* __restrict__ values_t, const float* __restrict__ valid_t, float* __restrict__ rewards_out_t,
    uint8_t* __restrict__ dones_cur, float* __restrict__ prev_dones, float* __restrict__ ep_state, double* meter,
    int games_to_track, double* scratch, int* counter, int N, ShaperDev c) {
    __shared__ double sm[32 * 4];
    __shared__ int is_last;
    pdl_sync();
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    double acc[4] = {0, 0, 0, 0};
    if (e < N) {
        const float r = rewards[e];
        float sh = __fmul_rn(__fadd_rn(r, c.shift_value), c.scale_value);
        sh = fminf(fmaxf(sh, c.min_val), c.max_val);
        if (c.log_val) sh = logf(sh);
        if (c.value_bootstrap && time_outs_kind) {
            const float to = time_outs_kind == 1 ? (float)((const uint8_t*)time_outs)[e] : ((const float*)time_outs)[e];
            sh = __fadd_rn(sh, __fmul_rn(__fmul_rn(c.gamma, values_t[e]), to));
        }
        rewards_out_t[e] = sh;
        const float live = valid_t ? valid_t[e] : 1.0f;
        float cr = ep_state[e] + r * live;
        float cs = ep_state[N + e] + sh * live;
        float cl = ep_state[2 * N + e] + live;
        const float d = (float)dones[e];
        const bool done = d != 0.f;
        if (done) { acc[0] = 1.0; acc[1] = cr; acc[2] = cs; acc[3] = cl; }
        const float nd = 1.0f - d;
        ep_state[e] = cr * nd; ep_state[N + e] = cs * nd; ep_state[2 * N + e] = cl * nd;
        dones_cur[e] = done ? 1 : 0;
        if (prev_dones) prev_dones[e] = d;
    }
    block_sum_d<4>(acc, sm);
    if (threadIdx.x == 0) {
#pragma unroll
        for (int i = 0; i < 4; ++i) scratch[(int64_t)blockIdx.x * 4 + i] = acc[i];
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) is_last = (atomicAdd(counter, 1) == (int)gridDim.x - 1);
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    double t[4] = {0, 0, 0, 0};
    for (int b = threadIdx.x; b < (int)gridDim.x; b += blockDim.x) {
#pragma unroll
        for (int i = 0; i < 4; ++i) t[i] += __ldcg(scratch + (int64_t)b * 4 + i);
    }
    block_sum_d<4>(t, sm);
    if (threadIdx.x == 0) {
        // AverageMeter.update (torch_ext.py:333-342); meter = {mean_r, mean_sr, mean_len, current_size, total_done}
        const double n = t[0];
        if (n > 0.0) {
            const double size = fmin(n, (double)games_to_track);
            const double old_size = fmin((double)games_to_track - size, meter[3]);
            const double size_sum = old_size + size;
            meter[0] = (meter[0] * old_size + (t[1] / n) * size) / size_sum;
            meter[1] = (meter[1] * old_size + (t[2] / n) * size) / size_sum;
            meter[2] = (meter[2] * old_size + (t[3] / n) * size) / size_sum;
            meter[3] = size_sum;
            meter[4] += n;
        }
        *counter = 0;
    }
}

// Multi-agent edition of post_step (a2c_common.py:1039-1051 with num_agents = G > 1): the step's done rows are ranked in index
// order and only ranks 0, G, 2G, ... (all_done_indices[::G]) feed the meters and the selected-index list; current_* are zeroed on
// every done row.  One pass: a CTA takes tiles in ticket order, ranks its rows with warp ballots, and gets the count of done rows
// before its tile by decoupled look-back over the earlier tiles' status words -- the ranks depend on row order only, never on
// scheduling.  A CTA waits only on tiles whose tickets were drawn before its own, so every tile it waits on is already running.
// tile_status: u64 per tile, 0 = not published, else (flag << 62) | count (flag 1 = tile's own count, 2 = count through the tile).
// The last CTA reduces the per-tile meter partials in tile order, writes sel_count and re-arms tile_status and the counters.
constexpr int MA_THREADS = 256, MA_SLABS = 4, MA_TILE = MA_THREADS * MA_SLABS;
static_assert(MA_TILE == B200RL_POST_STEP_MA_TILE, "include/b200rl.h states the tile size");
constexpr unsigned long long MA_AGG = 1ull << 62, MA_INCL = 2ull << 62, MA_VAL = (1ull << 62) - 1;

template <typename DT>
__global__ void __launch_bounds__(MA_THREADS) post_step_ma_kernel(
    const float* __restrict__ rewards, const DT* __restrict__ dones, const void* __restrict__ time_outs, int time_outs_kind,
    const float* __restrict__ values_t, const float* __restrict__ valid_t, float* __restrict__ rewards_out_t,
    uint8_t* __restrict__ dones_cur, float* __restrict__ prev_dones, float* __restrict__ ep_state, double* meter,
    int games_to_track, double* scratch, unsigned long long* tile_status, int* counters, int64_t* __restrict__ sel_idx,
    int* sel_count, int N, int G, ShaperDev c) {
    __shared__ double sm[32 * 4];
    __shared__ int slab_count[MA_SLABS][MA_THREADS / 32];
    __shared__ int s_tile, s_excl, is_last;
    pdl_sync();
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_tile = atomicAdd(counters, 1);
    __syncthreads();
    const int tile = s_tile;
    float cr[MA_SLABS], cs[MA_SLABS], cl[MA_SLABS];
    bool done[MA_SLABS];
    unsigned ball[MA_SLABS];
#pragma unroll
    for (int k = 0; k < MA_SLABS; ++k) {
        const int e = tile * MA_TILE + k * MA_THREADS + tid;
        done[k] = false;
        if (e < N) {
            const float r = rewards[e];
            float sh = __fmul_rn(__fadd_rn(r, c.shift_value), c.scale_value);
            sh = fminf(fmaxf(sh, c.min_val), c.max_val);
            if (c.log_val) sh = logf(sh);
            if (c.value_bootstrap && time_outs_kind) {
                const float to = time_outs_kind == 1 ? (float)((const uint8_t*)time_outs)[e] : ((const float*)time_outs)[e];
                sh = __fadd_rn(sh, __fmul_rn(__fmul_rn(c.gamma, values_t[e]), to));
            }
            rewards_out_t[e] = sh;
            const float live = valid_t ? valid_t[e] : 1.0f;
            cr[k] = ep_state[e] + r * live;
            cs[k] = ep_state[N + e] + sh * live;
            cl[k] = ep_state[2 * N + e] + live;
            const float d = (float)dones[e];
            done[k] = d != 0.f;
            const float nd = 1.0f - d;
            ep_state[e] = cr[k] * nd; ep_state[N + e] = cs[k] * nd; ep_state[2 * N + e] = cl[k] * nd;
            dones_cur[e] = done[k] ? 1 : 0;
            if (prev_dones) prev_dones[e] = d;
        }
        ball[k] = __ballot_sync(0xffffffffu, done[k]);
        if (lane == 0) slab_count[k][warp] = __popc(ball[k]);
    }
    __syncthreads();
    // exclusive prefix over (slab, warp) in row order, in place; warp 0 lane i holds entry i of the 32
    if (warp == 0) {
        const int v = slab_count[lane / (MA_THREADS / 32)][lane % (MA_THREADS / 32)];
        int incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
        }
        slab_count[lane / (MA_THREADS / 32)][lane % (MA_THREADS / 32)] = incl - v;
        const unsigned long long agg = (unsigned long long)__shfl_sync(0xffffffffu, incl, 31);
        if (lane == 0) {
            volatile unsigned long long* st = tile_status;
            unsigned long long excl = 0;
            if (tile == 0) {
                st[0] = MA_INCL | agg;
            } else {
                st[tile] = MA_AGG | agg;
                for (int j = tile - 1; j >= 0; --j) {
                    unsigned long long w;
                    do { w = st[j]; } while (w == 0ull);
                    excl += w & MA_VAL;
                    if ((w & ~MA_VAL) == MA_INCL) break;
                }
                st[tile] = MA_INCL | (excl + agg);
            }
            s_excl = (int)excl;
        }
    }
    __syncthreads();
    const unsigned lt = (1u << lane) - 1u;
    double acc[4] = {0, 0, 0, 0};
#pragma unroll
    for (int k = 0; k < MA_SLABS; ++k) {
        if (!done[k]) continue;
        const int rank = s_excl + slab_count[k][warp] + __popc(ball[k] & lt);
        if (rank % G == 0) {
            sel_idx[rank / G] = (int64_t)(tile * MA_TILE + k * MA_THREADS + tid);
            acc[0] += 1.0; acc[1] += cr[k]; acc[2] += cs[k]; acc[3] += cl[k];
        }
    }
    block_sum_d<4>(acc, sm);
    if (tid == 0) {
#pragma unroll
        for (int i = 0; i < 4; ++i) scratch[(int64_t)tile * 4 + i] = acc[i];
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) is_last = (atomicAdd(counters + 1, 1) == (int)gridDim.x - 1);
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    double t[4] = {0, 0, 0, 0};
    for (int b = tid; b < (int)gridDim.x; b += blockDim.x) {
#pragma unroll
        for (int i = 0; i < 4; ++i) t[i] += __ldcg(scratch + (int64_t)b * 4 + i);
        tile_status[b] = 0ull;
    }
    block_sum_d<4>(t, sm);
    if (tid == 0) {
        const double n = t[0];
        if (n > 0.0) {      // AverageMeter.update over the selected rows (torch_ext.py:333-342)
            const double size = fmin(n, (double)games_to_track);
            const double old_size = fmin((double)games_to_track - size, meter[3]);
            const double size_sum = old_size + size;
            meter[0] = (meter[0] * old_size + (t[1] / n) * size) / size_sum;
            meter[1] = (meter[1] * old_size + (t[2] / n) * size) / size_sum;
            meter[2] = (meter[2] * old_size + (t[3] / n) * size) / size_sum;
            meter[3] = size_sum;
            meter[4] += n;
        }
        *sel_count = (int)n;
        counters[0] = 0;
        counters[1] = 0;
    }
}

// one thread per (env, group of 4 features)
__global__ void __launch_bounds__(256) synth_env_step_kernel(const float* __restrict__ actions, float* __restrict__ obs,
                                                            float* __restrict__ rewards, uint8_t* __restrict__ dones,
                                                            uint8_t* __restrict__ time_outs, int* __restrict__ ep_t, int N, int D,
                                                            int A, int max_len, float p_done, uint64_t seed,
                                                            const uint64_t* __restrict__ rng_epoch_dev, uint32_t step_index) {
    const int groups = (D + 3) / 4;
    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (int64_t)N * groups) return;
    const int e = (int)(gid / groups), q = (int)(gid - (int64_t)e * groups);
    const uint64_t ep = rng_epoch_dev ? *rng_epoch_dev : 0ull;
    const uint64_t hi = (ep << 20) | ((uint64_t)step_index << 10) | (uint64_t)q;
    const Philox4 r = philox4x32_10((uint64_t)e, hi, seed ^ 0x5851F42D4C957F2Dull);
    float n0, n1, n2, n3;
    box_muller(r.x, r.y, n0, n1);
    box_muller(r.z, r.w, n2, n3);
    const int k = q * 4;
    float* o = obs + (int64_t)e * D + k;
    if ((D & 3) == 0) {
        *reinterpret_cast<float4*>(o) = make_float4(n0, n1, n2, n3);
    } else {
        if (k + 0 < D) o[0] = n0;
        if (k + 1 < D) o[1] = n1;
        if (k + 2 < D) o[2] = n2;
        if (k + 3 < D) o[3] = n3;
    }
    if (q == 0) {
        float s = 0.f;
        if (actions)
            for (int j = 0; j < A; ++j) { const float a = __ldg(actions + (int64_t)e * A + j); s = fmaf(a, a, s); }
        rewards[e] = -s;
        const Philox4 r2 = philox4x32_10((uint64_t)e, hi | (1ull << 9), seed ^ 0x9E3779B97F4A7C15ull);
        const int t = ep_t[e] + 1;
        const bool to = t >= max_len;
        const bool term = u32_to_unit_open(r2.x) <= p_done;
        const bool done = to || term;
        dones[e] = done ? 1 : 0;
        time_outs[e] = (to && !term) ? 1 : 0;
        ep_t[e] = done ? 0 : t;
    }
}

__global__ void bump_u64_kernel(uint64_t* p) { *p += 1; }

}  // namespace

B200RL_EXPORT int b200rl_policy_head_sample_f32(const float* a_last, int Hl, const float* W_head, const float* b_head,
                                                const float* logstd, const double* vms_mean, const double* vms_var,
                                                int normalize_value, const float* noise, uint64_t seed,
                                                const uint64_t* rng_epoch_dev, uint32_t step_index,
                                                float* actions, float* mus, float* sigmas, float* neglogp, float* values,
                                                float* env_actions, int clip_actions, const float* act_low, const float* act_high,
                                                const uint8_t* dones_cur, uint8_t* dones_out, const float* prev_dones,
                                                float* valid_out, int N, int A, int values_only, void* stream) {
    if (!a_last || !W_head || !b_head || !logstd || !values || N <= 0 || A <= 0 || A + 1 > MAXA || Hl <= 0) return B200RL_EINVAL;
    if (!values_only && (!actions || !mus || !sigmas || !neglogp)) return B200RL_EINVAL;
    if (normalize_value && (!vms_mean || !vms_var)) return B200RL_EINVAL;
    if (env_actions && clip_actions && (!act_low || !act_high)) return B200RL_EINVAL;
    if (dones_out && !dones_cur) return B200RL_EINVAL;
    const size_t smem = sizeof(float) * ((size_t)PT * (Hl + 1) + (size_t)(A + 1) * Hl + (A + 1) + 2 * A);
    if (smem > 200 * 1024) return B200RL_EUNSUPPORTED;
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(policy_head_sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return (int)e;
    }
    policy_head_sample_kernel<<<(N + PT - 1) / PT, PT, smem, as_stream(stream)>>>(
        a_last, Hl, W_head, b_head, logstd, vms_mean, vms_var, normalize_value, noise, seed, rng_epoch_dev, step_index, actions, mus,
        sigmas, neglogp, values, env_actions, clip_actions, act_low, act_high, dones_cur, dones_out, prev_dones, valid_out, N, A,
        values_only);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_policy_head_sample_sd_f32(const float* a_last, int Hl, const float* W_head, const float* b_head,
                                                   const b200rl_sigma_cfg* sigma_cfg_host, const double* vms_mean, const double* vms_var,
                                                   int normalize_value, const float* noise, uint64_t seed,
                                                   const uint64_t* rng_epoch_dev, uint32_t step_index,
                                                   float* actions, float* mus, float* sigmas, float* neglogp, float* values,
                                                   float* env_actions, int clip_actions, const float* act_low, const float* act_high,
                                                   const uint8_t* dones_cur, uint8_t* dones_out, const float* prev_dones,
                                                   float* valid_out, int N, int A, int values_only, void* stream) {
    if (!a_last || !W_head || !b_head || !sigma_cfg_host || !values || N <= 0 || A <= 0 || A + 1 > MAXA_SD || Hl <= 0) return B200RL_EINVAL;
    if (sigma_cfg_host->parametrization < SIGMA_EXP || sigma_cfg_host->parametrization > SIGMA_LINEAR) return B200RL_EINVAL;
    if (!values_only && (!actions || !mus || !sigmas || !neglogp)) return B200RL_EINVAL;
    if (normalize_value && (!vms_mean || !vms_var)) return B200RL_EINVAL;
    if (env_actions && clip_actions && (!act_low || !act_high)) return B200RL_EINVAL;
    if (dones_out && !dones_cur) return B200RL_EINVAL;
    const int HR = 1 + 2 * A;
    const size_t smem = sizeof(float) * ((size_t)PT * (Hl + 1) + (size_t)HR * Hl + HR + 2 * A);
    if (smem > 200 * 1024) return B200RL_EUNSUPPORTED;
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(policy_head_sample_sd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return (int)e;
    }
    policy_head_sample_sd_kernel<<<(N + PT - 1) / PT, PT, smem, as_stream(stream)>>>(
        a_last, Hl, W_head, b_head, sigma_cfg_dev(*sigma_cfg_host), vms_mean, vms_var, normalize_value, noise, seed, rng_epoch_dev,
        step_index, actions, mus, sigmas, neglogp, values, env_actions, clip_actions, act_low, act_high, dones_cur, dones_out, prev_dones,
        valid_out, N, A, values_only);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_post_step_f32(const float* rewards, const void* dones, int dones_is_u8, const void* time_outs,
                                       int time_outs_kind, const float* values_t, const float* valid_t,
                                       float* rewards_out_t, uint8_t* dones_cur, float* prev_dones_f32,
                                       float* ep_state, double* meter, int games_to_track,
                                       double* scratch, int scratch_blocks, int* counter, int N,
                                       const b200rl_shaper_cfg* cfg_host, void* stream) {
    if (!rewards || !dones || !rewards_out_t || !dones_cur || !ep_state || !meter || !scratch || !counter || !cfg_host || N <= 0)
        return B200RL_EINVAL;
    if (time_outs_kind && (!time_outs || !values_t)) return B200RL_EINVAL;
    const int blocks = (N + 255) / 256;
    if (blocks > scratch_blocks) return B200RL_EINVAL;
    ShaperDev c;
    c.scale_value = cfg_host->scale_value; c.shift_value = cfg_host->shift_value; c.min_val = cfg_host->min_val;
    c.max_val = cfg_host->max_val; c.gamma = cfg_host->gamma; c.log_val = cfg_host->log_val;
    c.value_bootstrap = cfg_host->value_bootstrap;
    cudaStream_t s = as_stream(stream);
    cudaError_t le;
    if (dones_is_u8)
        le = launch_k(post_step_kernel<uint8_t>, dim3(blocks), dim3(256), 0, s, rewards, (const uint8_t*)dones, time_outs, time_outs_kind, values_t,
                      valid_t, rewards_out_t, dones_cur, prev_dones_f32, ep_state, meter, games_to_track, scratch, counter, N, c);
    else
        le = launch_k(post_step_kernel<float>, dim3(blocks), dim3(256), 0, s, rewards, (const float*)dones, time_outs, time_outs_kind, values_t,
                      valid_t, rewards_out_t, dones_cur, prev_dones_f32, ep_state, meter, games_to_track, scratch, counter, N, c);
    if (le != cudaSuccess) return (int)le;
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_post_step_ma_f32(const float* rewards, const void* dones, int dones_is_u8, const void* time_outs,
                                          int time_outs_kind, const float* values_t, const float* valid_t,
                                          float* rewards_out_t, uint8_t* dones_cur, float* prev_dones_f32,
                                          float* ep_state, double* meter, int games_to_track,
                                          double* scratch, uint64_t* tile_status, int scratch_tiles, int* counters,
                                          int64_t* sel_idx, int* sel_count, int N, int agents,
                                          const b200rl_shaper_cfg* cfg_host, void* stream) {
    if (!rewards || !dones || !rewards_out_t || !dones_cur || !ep_state || !meter || !scratch || !tile_status || !counters ||
        !sel_idx || !sel_count || !cfg_host || N <= 0 || agents <= 0)
        return B200RL_EINVAL;
    if (time_outs_kind && (!time_outs || !values_t)) return B200RL_EINVAL;
    const int tiles = (N + MA_TILE - 1) / MA_TILE;
    if (tiles > scratch_tiles) return B200RL_EINVAL;
    ShaperDev c;
    c.scale_value = cfg_host->scale_value; c.shift_value = cfg_host->shift_value; c.min_val = cfg_host->min_val;
    c.max_val = cfg_host->max_val; c.gamma = cfg_host->gamma; c.log_val = cfg_host->log_val;
    c.value_bootstrap = cfg_host->value_bootstrap;
    cudaStream_t s = as_stream(stream);
    unsigned long long* st = reinterpret_cast<unsigned long long*>(tile_status);
    cudaError_t le;
    if (dones_is_u8)
        le = launch_k(post_step_ma_kernel<uint8_t>, dim3(tiles), dim3(MA_THREADS), 0, s, rewards, (const uint8_t*)dones, time_outs,
                      time_outs_kind, values_t, valid_t, rewards_out_t, dones_cur, prev_dones_f32, ep_state, meter, games_to_track,
                      scratch, st, counters, sel_idx, sel_count, N, agents, c);
    else
        le = launch_k(post_step_ma_kernel<float>, dim3(tiles), dim3(MA_THREADS), 0, s, rewards, (const float*)dones, time_outs,
                      time_outs_kind, values_t, valid_t, rewards_out_t, dones_cur, prev_dones_f32, ep_state, meter, games_to_track,
                      scratch, st, counters, sel_idx, sel_count, N, agents, c);
    if (le != cudaSuccess) return (int)le;
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_synth_env_step(const float* actions, float* obs, float* rewards, uint8_t* dones, uint8_t* time_outs,
                                        int* ep_t, int N, int D, int A, int max_len, float p_done,
                                        uint64_t seed, const uint64_t* rng_epoch_dev, uint32_t step_index, void* stream) {
    if (!obs || !rewards || !dones || !time_outs || !ep_t || N <= 0 || D <= 0 || A < 0) return B200RL_EINVAL;
    const int64_t total = (int64_t)N * ((D + 3) / 4);
    synth_env_step_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(
        actions, obs, rewards, dones, time_outs, ep_t, N, D, A, max_len, p_done, seed, rng_epoch_dev, step_index);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_bump_u64(uint64_t* p, void* stream) {
    if (!p) return B200RL_EINVAL;
    bump_u64_kernel<<<1, 1, 0, as_stream(stream)>>>(p);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}
