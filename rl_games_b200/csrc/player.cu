// Deterministic categorical head of the discrete player (players.py: PpoPlayerDiscrete, is_deterministic): the reference plays
// torch.argmax(CategoricalMasked(logits, masks).logits) per head (algos_torch/players.py, distributions.py:23-44).
//
// Narrow kernel: one warp per row, for layouts of at most 8 heads of at most 64 actions, so each lane reads at most two logits of a head
// and a five-step shuffle reduction finds the winner; every other layout runs on the wide kernel below (one warp per head).  Reduction
// order: larger value first, then lower index, so ties go to the lowest index as in torch.argmax; NaN counts as larger than any number (torch.argmax returns the first NaN).  A masked action never wins; a head
// with every action masked plays action 0, which is what argmax gives the reference there (every masked logit is -1e8, so after the
// log-softmax normalisation all are equal).
//
// Tests: tests/test_players_gpu.py (exhaustive against torch.argmax at every head layout up to 8 x 64, ties, all-masked heads),
// tests/test_cat_wide_gpu.py (the wide kernel: every head size 65-256, 9 to 1792 heads).
#include "common.cuh"

namespace {

constexpr int ARGMAX_MAXK = 64;
constexpr int ARGMAX_MAXH = 8;
constexpr int ARGMAX_NONE = 0x7fffffff;      // "no legal action seen yet"

struct ArgmaxHeads { int n; int size[ARGMAX_MAXH]; int off[ARGMAX_MAXH]; };

// (va, ia) beats (vb, ib): a legal candidate beats none; NaN beats numbers; then the larger value; equal values: the lower index
__device__ __forceinline__ bool argmax_beats(float va, int ia, float vb, int ib) {
    if (ia == ARGMAX_NONE) return false;
    if (ib == ARGMAX_NONE) return true;
    const bool na = va != va, nb = vb != vb;
    if (na != nb) return na;
    if (!na && va != vb) return va > vb;
    return ia < ib;
}

__global__ void __launch_bounds__(256) categorical_argmax_kernel(const float* __restrict__ logits, int ld, int K, ArgmaxHeads hd,
                                                                 const uint8_t* __restrict__ masks, int64_t* __restrict__ actions, int N) {
    const int row = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= N) return;
    const float* z = logits + (int64_t)row * ld;
    const uint8_t* mk = masks ? masks + (int64_t)row * K : nullptr;
    for (int j = 0; j < hd.n; ++j) {
        float best = 0.f;
        int bi = ARGMAX_NONE;
        for (int k = lane; k < hd.size[j]; k += 32) {
            const int c = hd.off[j] + k;
            if (mk && !mk[c]) continue;
            const float v = z[c];
            if (argmax_beats(v, k, best, bi)) { best = v; bi = k; }
        }
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, best, s);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, s);
            if (argmax_beats(ov, oi, best, bi)) { best = ov; bi = oi; }
        }
        if (lane == 0) actions[(int64_t)row * hd.n + j] = bi == ARGMAX_NONE ? 0 : bi;
    }
}

// any layout: one CTA per row, warp w takes heads w, w + W, ... (W = min(n_heads, 8)); head j covers [off[j], off[j + 1]) of the row
// (off == NULL: one head of K actions).  The per-head scan and reduction are the narrow kernel's.
__global__ void __launch_bounds__(256) categorical_argmax_wide_kernel(const float* __restrict__ logits, int ld, int K, int n_heads,
                                                                      const int* __restrict__ off, const uint8_t* __restrict__ masks,
                                                                      int64_t* __restrict__ actions) {
    const int64_t row = blockIdx.x;
    const int lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    const float* z = logits + row * ld;
    const uint8_t* mk = masks ? masks + row * K : nullptr;
    for (int j = threadIdx.x >> 5; j < n_heads; j += nw) {
        const int o = off ? off[j] : 0, n = off ? off[j + 1] - o : K;
        float best = 0.f;
        int bi = ARGMAX_NONE;
        for (int k = lane; k < n; k += 32) {
            if (mk && !mk[o + k]) continue;
            const float v = z[o + k];
            if (argmax_beats(v, k, best, bi)) { best = v; bi = k; }
        }
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, best, s);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, s);
            if (argmax_beats(ov, oi, best, bi)) { best = ov; bi = oi; }
        }
        if (lane == 0) actions[row * n_heads + j] = bi == ARGMAX_NONE ? 0 : bi;
    }
}

}  // namespace

B200RL_EXPORT int b200rl_categorical_argmax_wide_f32(const float* logits, int ld, int K, int n_heads, const int* head_sizes_host,
                                                     const int* head_offsets_dev, const uint8_t* action_masks, int64_t* actions_out, int N,
                                                     void* stream) {
    if (!logits || !actions_out || N <= 0 || K <= 0 || ld < K) return B200RL_EINVAL;
    int heads = 1;
    if (n_heads > 0 && head_sizes_host) {
        if (!head_offsets_dev) return B200RL_EINVAL;
        int64_t tot = 0;
        for (int j = 0; j < n_heads; ++j) {
            if (head_sizes_host[j] <= 0) return B200RL_EINVAL;
            tot += head_sizes_host[j];
        }
        if (tot != K) return B200RL_EINVAL;
        heads = n_heads;
    }
    const int warps = heads < 8 ? heads : 8;
    categorical_argmax_wide_kernel<<<N, 32 * warps, 0, as_stream(stream)>>>(logits, ld, K, heads, heads > 1 ? head_offsets_dev : nullptr,
                                                                            action_masks, actions_out);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}

B200RL_EXPORT int b200rl_categorical_argmax_f32(const float* logits, int ld, int K, int n_heads, const int* head_sizes_host,
                                                const uint8_t* action_masks, int64_t* actions_out, int N, void* stream) {
    if (!logits || !actions_out || N <= 0 || K <= 0 || ld < K) return B200RL_EINVAL;
    ArgmaxHeads hd{};
    if (n_heads <= 0 || !head_sizes_host) {
        if (K > ARGMAX_MAXK) return B200RL_EINVAL;
        hd.n = 1; hd.size[0] = K; hd.off[0] = 0;
    } else {
        if (n_heads > ARGMAX_MAXH) return B200RL_EINVAL;
        hd.n = n_heads;
        int off = 0;
        for (int j = 0; j < n_heads; ++j) {
            if (head_sizes_host[j] <= 0 || head_sizes_host[j] > ARGMAX_MAXK) return B200RL_EINVAL;
            hd.size[j] = head_sizes_host[j]; hd.off[j] = off; off += head_sizes_host[j];
        }
        if (off != K) return B200RL_EINVAL;
    }
    const int64_t threads = (int64_t)N * 32;
    categorical_argmax_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, as_stream(stream)>>>(logits, ld, K, hd, action_masks,
                                                                                               actions_out, N);
    B200RL_LAUNCH_CHECK();
    return B200RL_OK;
}
