// LSTM-with-dones cell kernels (fp32): the pointwise half of common/layers/recurrent.py:20-80 (LSTMWithDones ->
// torch.nn.LSTM, gate order i,f,g,o) and of its BPTT, for the rollout (one step) and the seq_length-window training
// forward/backward.  The GEMM halves (x W_ih^T, h W_hh^T and their dgrad/wgrad) run on the linear_* kernels.
// State zeroing at episode boundaries (a2c_common.py:1150-1153 in the rollout, RnnWithDones.forward :26-58 in training) is
// folded in as a multiplication of the carried (h, c) by (1 - done) when they are handed to the next step.
#include "common.cuh"

namespace {

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

// gates: [S, 4*Hd] pre-activations in, activations (i,f,g,o) out.   cin: [S,Hd] (already masked c_{t-1})
// outputs: c_out [S,Hd]; h_out [S,Hd] dense; optional h_scatter: row s -> (s / spc) * scatter_stride + s % spc  (MLP-order buffer)
// optional next-step carries: hin_next = h * (1 - done_next[s]), cin_next = c * (1 - done_next[s]) with done_next rows chunk-mapped.
__global__ void __launch_bounds__(256) lstm_cell_fwd_kernel(float* __restrict__ gates, const float* __restrict__ cin, float* __restrict__ c_out,
                                                           float* __restrict__ h_out, float* __restrict__ h_scatter, int spc,
                                                           int64_t scatter_stride, float* __restrict__ hin_next, float* __restrict__ cin_next,
                                                           const uint8_t* __restrict__ done_next, int d_rpc, int64_t d_stride, int S, int Hd) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (int64_t)S * Hd) return;
    const int s = (int)(idx / Hd), k = (int)(idx - (int64_t)s * Hd);
    float* g = gates + (int64_t)s * 4 * Hd;
    const float i = sigmoidf_(g[k]), f = sigmoidf_(g[Hd + k]), gg = tanhf(g[2 * Hd + k]), o = sigmoidf_(g[3 * Hd + k]);
    g[k] = i; g[Hd + k] = f; g[2 * Hd + k] = gg; g[3 * Hd + k] = o;
    const float c = f * cin[idx] + i * gg;
    const float h = o * tanhf(c);
    c_out[idx] = c;
    h_out[idx] = h;
    if (h_scatter) h_scatter[((int64_t)(s / spc) * scatter_stride + (s % spc)) * Hd + k] = h;
    if (hin_next) {
        float m = 1.0f;
        if (done_next) m = 1.0f - (float)done_next[chunk_row(s, d_rpc, d_stride)];
        hin_next[idx] = h * m;
        cin_next[idx] = c * m;
    }
}

// Backward of one cell step.  dh_in = dH_mlp[row(s)] (chunk scatter order, optional) + dhin_next[s] * m_next ; dc_in = dcin_next * m_next.
// Writes dgates [S,4Hd] (pre-activation gradients) and dcin [S,Hd] (gradient w.r.t. the masked c input of THIS step).
__global__ void __launch_bounds__(256) lstm_cell_bwd_kernel(const float* __restrict__ gates_act, const float* __restrict__ c_t,
                                                           const float* __restrict__ cin, const float* __restrict__ dH, int spc,
                                                           int64_t scatter_stride, const float* __restrict__ dhin_next,
                                                           const float* __restrict__ dcin_next, const uint8_t* __restrict__ done_next, int d_rpc,
                                                           int64_t d_stride, float* __restrict__ dgates, float* __restrict__ dcin, int S, int Hd) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (int64_t)S * Hd) return;
    const int s = (int)(idx / Hd), k = (int)(idx - (int64_t)s * Hd);
    const float* g = gates_act + (int64_t)s * 4 * Hd;
    const float i = g[k], f = g[Hd + k], gg = g[2 * Hd + k], o = g[3 * Hd + k];
    float m = 1.0f;
    if (done_next) m = 1.0f - (float)done_next[chunk_row(s, d_rpc, d_stride)];
    float dh = dH ? dH[((int64_t)(s / spc) * scatter_stride + (s % spc)) * Hd + k] : 0.f;
    float dc = 0.f;
    if (dhin_next) { dh += dhin_next[idx] * m; dc += dcin_next[idx] * m; }
    const float tc = tanhf(c_t[idx]);
    dc += dh * o * (1.0f - tc * tc);
    float* dg = dgates + (int64_t)s * 4 * Hd;
    dg[k] = dc * gg * i * (1.0f - i);
    dg[Hd + k] = dc * cin[idx] * f * (1.0f - f);
    dg[2 * Hd + k] = dc * i * (1.0f - gg * gg);
    dg[3 * Hd + k] = dh * tc * o * (1.0f - o);
    dcin[idx] = dc * f;
}

// out[s][k] = in[row(s)][k] * (1 - done[drow(s)])   (masked initial state of a window / zeroing after an episode end)
__global__ void __launch_bounds__(256) rnn_mask_rows_kernel(const float* __restrict__ in, int in_rpc, int64_t in_stride, float* __restrict__ out,
                                                           const uint8_t* __restrict__ done, int d_rpc, int64_t d_stride, int S, int Hd) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (int64_t)S * Hd) return;
    const int s = (int)(idx / Hd), k = (int)(idx - (int64_t)s * Hd);
    const float m = done ? 1.0f - (float)done[chunk_row(s, d_rpc, d_stride)] : 1.0f;
    out[idx] = in[chunk_row(s, in_rpc, in_stride) * Hd + k] * m;
}

// Train-time reset flags of an RNN policy on a next_step-autoreset env (a2c_common.py:1180-1191): besides the buffer's own dones the
// state reset also fires ENTERING the first real row after a filler reset row (valid == 0), mirroring the rollout-side re-zero.
//   out[t, n] = dones[t, n] | (t > 0 && valid[t - 1, n] == 0)
__host__ __device__ inline uint8_t rnn_train_done(const uint8_t* dones, const float* valid, int64_t i, int N) {
    return (uint8_t)((dones[i] != 0) || (i >= N && valid[i - N] == 0.0f));
}
__global__ void __launch_bounds__(256) rnn_train_dones_kernel(const uint8_t* __restrict__ dones, const float* __restrict__ valid,
                                                              uint8_t* __restrict__ out, int64_t n, int N) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = rnn_train_done(dones, valid, i, N);
}

// ---- LSTM cell + LayerNorm of its output (rnn.layer_norm: True; network_builder.py:279-280, :485-486) ----------------------------
// y = LayerNorm(h) = (h - mean) * rstd * gamma + beta over the Hd units of a row (biased variance, eps 1e-5); the carried states stay the
// raw (h, c).  One warp per row; every pass strides the row by 32, so any Hd works and nothing is held per element in registers.
constexpr int LN_ROWS_PER_CTA = 8;
constexpr float LN_EPS = 1e-5f;

// Cell maths of lstm_cell_fwd_kernel (same arguments, h_out = raw h) plus y into y_out (dense, optional) and / or y_scatter (MLP-order
// rows, optional), and the row statistics mean / rstd (optional) the backward reads.  Two-pass variance over the h just written.
__global__ void __launch_bounds__(256) lstm_cell_ln_fwd_kernel(float* __restrict__ gates, const float* cin, float* c_out,
                                                              float* h_out, float* __restrict__ y_out, float* __restrict__ y_scatter, int spc,
                                                              int64_t scatter_stride, float* __restrict__ hin_next, float* __restrict__ cin_next,
                                                              const uint8_t* __restrict__ done_next, int d_rpc, int64_t d_stride,
                                                              const float* __restrict__ ln_w, const float* __restrict__ ln_b,
                                                              float* __restrict__ mean_out, float* __restrict__ rstd_out, int S, int Hd) {
    const int lane = threadIdx.x & 31;
    const int s = blockIdx.x * LN_ROWS_PER_CTA + (threadIdx.x >> 5);
    if (s >= S) return;
    const int64_t base = (int64_t)s * Hd;
    float* g = gates + (int64_t)s * 4 * Hd;
    float m = 1.0f;
    if (hin_next && done_next) m = 1.0f - (float)done_next[chunk_row(s, d_rpc, d_stride)];
    float sum = 0.f;
    for (int k = lane; k < Hd; k += 32) {
        const float i = sigmoidf_(g[k]), f = sigmoidf_(g[Hd + k]), gg = tanhf(g[2 * Hd + k]), o = sigmoidf_(g[3 * Hd + k]);
        g[k] = i; g[Hd + k] = f; g[2 * Hd + k] = gg; g[3 * Hd + k] = o;
        const float c = f * cin[base + k] + i * gg;
        const float h = o * tanhf(c);
        c_out[base + k] = c;
        h_out[base + k] = h;
        if (hin_next) { hin_next[base + k] = h * m; cin_next[base + k] = c * m; }
        sum += h;
    }
    const float mean = warp_sum(sum) / (float)Hd;
    float sq = 0.f;
    for (int k = lane; k < Hd; k += 32) {
        const float d = h_out[base + k] - mean;
        sq += d * d;
    }
    const float rstd = 1.0f / sqrtf(warp_sum(sq) / (float)Hd + LN_EPS);
    if (lane == 0 && mean_out) { mean_out[s] = mean; rstd_out[s] = rstd; }
    float* ys = y_scatter ? y_scatter + ((int64_t)(s / spc) * scatter_stride + (s % spc)) * Hd : nullptr;
    for (int k = lane; k < Hd; k += 32) {
        const float y = (h_out[base + k] - mean) * rstd * ln_w[k] + ln_b[k];
        if (y_out) y_out[base + k] = y;
        if (ys) ys[k] = y;
    }
}

// Backward of one cell step under the LayerNorm.  dy = dY[scatter row]; h = o * tanh(c_t) is recomputed from the stored activations;
//   dh = rstd * (dy*gamma - mean_k(dy*gamma) - xhat * mean_k(dy*gamma*xhat)) + dhin_next * m_next,  dc_in = dcin_next * m_next,
// then the cell backward of lstm_cell_bwd_kernel.
__global__ void __launch_bounds__(256) lstm_cell_ln_bwd_kernel(const float* __restrict__ gates_act, const float* __restrict__ c_t,
                                                              const float* __restrict__ cin, const float* __restrict__ dY, int spc,
                                                              int64_t scatter_stride, const float* __restrict__ dhin_next,
                                                              const float* __restrict__ dcin_next, const uint8_t* __restrict__ done_next,
                                                              int d_rpc, int64_t d_stride, const float* __restrict__ ln_w,
                                                              const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
                                                              float* __restrict__ dgates, float* __restrict__ dcin, int S, int Hd) {
    const int lane = threadIdx.x & 31;
    const int s = blockIdx.x * LN_ROWS_PER_CTA + (threadIdx.x >> 5);
    if (s >= S) return;
    const int64_t base = (int64_t)s * Hd;
    const float* g = gates_act + (int64_t)s * 4 * Hd;
    const float* dy = dY + ((int64_t)(s / spc) * scatter_stride + (s % spc)) * Hd;
    const float mean = mean_in[s], rstd = rstd_in[s];
    float a = 0.f, b = 0.f;
    for (int k = lane; k < Hd; k += 32) {
        const float xhat = (g[3 * Hd + k] * tanhf(c_t[base + k]) - mean) * rstd;
        const float gy = dy[k] * ln_w[k];
        a += gy;
        b += gy * xhat;
    }
    a = warp_sum(a) / (float)Hd;
    b = warp_sum(b) / (float)Hd;
    float m = 1.0f;
    if (done_next) m = 1.0f - (float)done_next[chunk_row(s, d_rpc, d_stride)];
    float* dg = dgates + (int64_t)s * 4 * Hd;
    for (int k = lane; k < Hd; k += 32) {
        const float i = g[k], f = g[Hd + k], gg = g[2 * Hd + k], o = g[3 * Hd + k];
        const float tc = tanhf(c_t[base + k]);
        const float xhat = (o * tc - mean) * rstd;
        float dh = rstd * (dy[k] * ln_w[k] - a - xhat * b);
        float dc = 0.f;
        if (dhin_next) { dh += dhin_next[base + k] * m; dc += dcin_next[base + k] * m; }
        dc += dh * o * (1.0f - tc * tc);
        dg[k] = dc * gg * i * (1.0f - i);
        dg[Hd + k] = dc * cin[base + k] * f * (1.0f - f);
        dg[2 * Hd + k] = dc * i * (1.0f - gg * gg);
        dg[3 * Hd + k] = dh * tc * o * (1.0f - o);
        dcin[base + k] = dc * f;
    }
}

// dgamma / dbeta of one step as row-split partials: split p (blockIdx.y) sums rows [p*rps, min(S, (p+1)*rps)) and writes
// dgamma_part[p*split_stride + k], dbeta_part[p*split_stride + k] (zero for an empty split).  A CTA owns 32 columns (one per lane, so each
// row is one coalesced access per warp); its 16 warps take every 16th row of the split, and warp 0 adds the 16 warp partials in a fixed
// order -- no atomics, bit-reproducible.
constexpr int LN_PG_COLS = 32, LN_PG_WARPS = 16;
__global__ void __launch_bounds__(LN_PG_COLS * LN_PG_WARPS) lstm_ln_param_grad_kernel(const float* __restrict__ gates_act,
                                                                                      const float* __restrict__ c_t,
                                                                                      const float* __restrict__ dY, int spc,
                                                                                      int64_t scatter_stride,
                                                                                      const float* __restrict__ mean_in,
                                                                                      const float* __restrict__ rstd_in,
                                                                                      float* __restrict__ dgamma_part,
                                                                                      float* __restrict__ dbeta_part, int64_t split_stride,
                                                                                      int rps, int S, int Hd) {
    __shared__ float sw[LN_PG_WARPS][LN_PG_COLS + 1], sb[LN_PG_WARPS][LN_PG_COLS + 1];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int k = blockIdx.x * LN_PG_COLS + lane;
    const int p = blockIdx.y;
    const int r1 = min(S, (p + 1) * rps);
    float dgw = 0.f, dgb = 0.f;
    if (k < Hd) {
        for (int s = p * rps + w; s < r1; s += LN_PG_WARPS) {
            const float h = gates_act[(int64_t)s * 4 * Hd + 3 * Hd + k] * tanhf(c_t[(int64_t)s * Hd + k]);
            const float dy = dY[((int64_t)(s / spc) * scatter_stride + (s % spc)) * Hd + k];
            dgw += dy * ((h - mean_in[s]) * rstd_in[s]);
            dgb += dy;
        }
    }
    sw[w][lane] = dgw;
    sb[w][lane] = dgb;
    __syncthreads();
    if (w == 0 && k < Hd) {
        float a = 0.f, b = 0.f;
        for (int j = 0; j < LN_PG_WARPS; ++j) { a += sw[j][lane]; b += sb[j][lane]; }
        dgamma_part[(int64_t)p * split_stride + k] = a;
        dbeta_part[(int64_t)p * split_stride + k] = b;
    }
}

}  // namespace

B200RL_EXPORT int b200rl_lstm_cell_fwd_f32(float* gates, const float* cin, float* c_out, float* h_out, float* h_scatter, int scatter_rpc,
                                           int64_t scatter_stride, float* hin_next, float* cin_next, const uint8_t* done_next,
                                           int done_rpc, int64_t done_stride, int S, int Hd, void* stream) {
    if (!gates || !cin || !c_out || !h_out || S <= 0 || Hd <= 0) return B200RL_EINVAL;
    if ((hin_next == nullptr) != (cin_next == nullptr)) return B200RL_EINVAL;
    if (h_scatter && scatter_rpc <= 0) return B200RL_EINVAL;
    if (done_next && done_rpc <= 0) return B200RL_EINVAL;
    const int64_t n = (int64_t)S * Hd;
    lstm_cell_fwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, as_stream(stream)>>>(gates, cin, c_out, h_out, h_scatter, scatter_rpc > 0 ? scatter_rpc : 1,
                                                                                     scatter_stride, hin_next, cin_next, done_next,
                                                                                     done_rpc > 0 ? done_rpc : 1, done_stride, S, Hd);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_lstm_cell_bwd_f32(const float* gates_act, const float* c_t, const float* cin, const float* dH, int scatter_rpc,
                                           int64_t scatter_stride, const float* dhin_next, const float* dcin_next, const uint8_t* done_next,
                                           int done_rpc, int64_t done_stride, float* dgates, float* dcin, int S, int Hd, void* stream) {
    if (!gates_act || !c_t || !cin || !dgates || !dcin || S <= 0 || Hd <= 0) return B200RL_EINVAL;
    if ((dhin_next == nullptr) != (dcin_next == nullptr)) return B200RL_EINVAL;
    if (dH && scatter_rpc <= 0) return B200RL_EINVAL;          // a dH without its row mapping would read row 0 for every row
    if (done_next && done_rpc <= 0) return B200RL_EINVAL;
    const int64_t n = (int64_t)S * Hd;
    lstm_cell_bwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, as_stream(stream)>>>(gates_act, c_t, cin, dH, scatter_rpc > 0 ? scatter_rpc : 1,
                                                                                     scatter_stride, dhin_next, dcin_next, done_next,
                                                                                     done_rpc > 0 ? done_rpc : 1, done_stride, dgates, dcin, S, Hd);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_rnn_mask_rows_f32(const float* in, int in_rpc, int64_t in_stride, float* out, const uint8_t* done, int done_rpc,
                                           int64_t done_stride, int S, int Hd, void* stream) {
    if (!in || !out || S <= 0 || Hd <= 0 || in_rpc <= 0) return B200RL_EINVAL;
    if (done && done_rpc <= 0) return B200RL_EINVAL;           // a done vector without its row mapping would read done[0] for every row
    const int64_t n = (int64_t)S * Hd;
    rnn_mask_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, as_stream(stream)>>>(in, in_rpc, in_stride, out, done, done_rpc > 0 ? done_rpc : 1,
                                                                                     done_stride, S, Hd);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_lstm_cell_ln_fwd_f32(float* gates, const float* cin, float* c_out, float* h_out, float* y_out, float* y_scatter,
                                              int scatter_rpc, int64_t scatter_stride, float* hin_next, float* cin_next,
                                              const uint8_t* done_next, int done_rpc, int64_t done_stride, const float* ln_w,
                                              const float* ln_b, float* mean, float* rstd, int S, int Hd, void* stream) {
    if (!gates || !cin || !c_out || !h_out || !ln_w || !ln_b || S <= 0 || Hd <= 0) return B200RL_EINVAL;
    if (!y_out && !y_scatter) return B200RL_EINVAL;
    if ((hin_next == nullptr) != (cin_next == nullptr)) return B200RL_EINVAL;
    if ((mean == nullptr) != (rstd == nullptr)) return B200RL_EINVAL;
    if (y_scatter && scatter_rpc <= 0) return B200RL_EINVAL;
    if (done_next && done_rpc <= 0) return B200RL_EINVAL;
    const unsigned grid = (unsigned)((S + LN_ROWS_PER_CTA - 1) / LN_ROWS_PER_CTA);
    lstm_cell_ln_fwd_kernel<<<grid, 32 * LN_ROWS_PER_CTA, 0, as_stream(stream)>>>(gates, cin, c_out, h_out, y_out, y_scatter,
                                                                                 scatter_rpc > 0 ? scatter_rpc : 1, scatter_stride,
                                                                                 hin_next, cin_next, done_next, done_rpc > 0 ? done_rpc : 1,
                                                                                 done_stride, ln_w, ln_b, mean, rstd, S, Hd);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_lstm_cell_ln_bwd_f32(const float* gates_act, const float* c_t, const float* cin, const float* dY, int scatter_rpc,
                                              int64_t scatter_stride, const float* dhin_next, const float* dcin_next,
                                              const uint8_t* done_next, int done_rpc, int64_t done_stride, const float* ln_w,
                                              const float* mean, const float* rstd, float* dgamma_part, float* dbeta_part,
                                              int64_t split_stride, int n_splits, float* dgates, float* dcin, int S, int Hd, void* stream) {
    if (!gates_act || !c_t || !cin || !dY || !ln_w || !mean || !rstd || !dgates || !dcin || S <= 0 || Hd <= 0) return B200RL_EINVAL;
    if (!dgamma_part || !dbeta_part || n_splits <= 0 || n_splits > 65535 || (n_splits > 1 && split_stride < Hd)) return B200RL_EINVAL;
    if ((dhin_next == nullptr) != (dcin_next == nullptr)) return B200RL_EINVAL;
    if (scatter_rpc <= 0 || (done_next && done_rpc <= 0)) return B200RL_EINVAL;
    cudaStream_t st = as_stream(stream);
    const unsigned grid = (unsigned)((S + LN_ROWS_PER_CTA - 1) / LN_ROWS_PER_CTA);
    lstm_cell_ln_bwd_kernel<<<grid, 32 * LN_ROWS_PER_CTA, 0, st>>>(gates_act, c_t, cin, dY, scatter_rpc, scatter_stride, dhin_next,
                                                                   dcin_next, done_next, done_rpc > 0 ? done_rpc : 1, done_stride, ln_w,
                                                                   mean, rstd, dgates, dcin, S, Hd);
    B200RL_LAUNCH_CHECK();
    const int rps = (S + n_splits - 1) / n_splits;
    lstm_ln_param_grad_kernel<<<dim3((unsigned)((Hd + LN_PG_COLS - 1) / LN_PG_COLS), (unsigned)n_splits), LN_PG_COLS * LN_PG_WARPS, 0, st>>>(
        gates_act, c_t, dY, scatter_rpc, scatter_stride, mean, rstd, dgamma_part, dbeta_part, split_stride, rps, S, Hd);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_rnn_train_dones_u8(const uint8_t* dones, const float* valid, uint8_t* out, int H, int N, void* stream) {
    if (!dones || !valid || !out || H <= 0 || N <= 0) return B200RL_EINVAL;
    const int64_t n = (int64_t)H * N;
    rnn_train_dones_kernel<<<(unsigned)((n + 255) / 256), 256, 0, as_stream(stream)>>>(dones, valid, out, n, N);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

#ifdef B200RL_TEST_HOOKS   // test-only host entry points: compiled into tests/libb200rl_testhooks.so (csrc/build.py), not into the product library
// host test entry point (tests/test_rnn_rows_cpu.py): the element function above over HOST arrays; not in include/b200rl.h
B200RL_EXPORT int b200rl_hosttest_rnn_train_dones(const uint8_t* dones, const float* valid, uint8_t* out, int H, int N) {
    for (int64_t i = 0; i < (int64_t)H * N; ++i) out[i] = rnn_train_done(dones, valid, i, N);
    return B200RL_OK;
}
#endif  // B200RL_TEST_HOOKS
