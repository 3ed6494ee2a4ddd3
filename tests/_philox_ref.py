"""Host restatement of the device random numbers (rl_games_b200/csrc/common.cuh): Philox4x32-10 in numpy uint64 arithmetic, the
(0, 1] and [0, 1) mappings of its 32-bit words, Box-Muller in fp64, and the counter layouts the kernels use.  The generator and the
uniform mappings are bit-exact; the normals differ from the device's only by the __logf / __sincosf intrinsics (a few 1e-6).

Counter layout (ctr_lo = row, ctr_hi = the fields below, which must not overlap):
  policy samplers:  epoch << 20 | step << 4 | q      step < 2^16, q < 16 (Gaussian q < 8, categorical head j: q = 8 + j, j < 8)
  synthetic env:    epoch << 20 | step << 10 | q     step < 2^10, q < 2^9 (feature group), bit 9 for the done draw"""
import numpy as np

M32 = np.uint64(0xFFFFFFFF)
PHILOX_M0, PHILOX_M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
PHILOX_W0, PHILOX_W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)

POLICY_STEP_BITS, POLICY_Q_BITS, EPOCH_SHIFT = 16, 4, 20
GAUSS_Q_MAX, CAT_Q0, CAT_MAXH = 8, 8, 8
SYNTH_STEP_BITS, SYNTH_Q_BITS, SYNTH_DONE_BIT = 10, 9, 9
SYNTH_OBS_KEY_XOR, SYNTH_DONE_KEY_XOR = 0x5851F42D4C957F2D, 0x9E3779B97F4A7C15


def _u64(x):
    return np.asarray(x, dtype=np.uint64)


def philox4x32_10(ctr_lo, ctr_hi, key):
    """four uint32 words (as uint64 arrays) of Philox4x32-10; arguments broadcast; ctr_lo / ctr_hi / key are 64-bit values split
    into 32-bit halves exactly as the device does (c0 = low half of ctr_lo, ..., k1 = high half of key)"""
    ctr_lo, ctr_hi, key = np.broadcast_arrays(_u64(ctr_lo), _u64(ctr_hi), _u64(key))
    c0, c1 = ctr_lo & M32, ctr_lo >> np.uint64(32)
    c2, c3 = ctr_hi & M32, ctr_hi >> np.uint64(32)
    k0, k1 = key & M32, key >> np.uint64(32)
    for _ in range(10):
        p0, p1 = PHILOX_M0 * c0, PHILOX_M1 * c2           # 32 x 32 -> 64 bits: exact in uint64
        hi0, lo0 = p0 >> np.uint64(32), p0 & M32
        hi1, lo1 = p1 >> np.uint64(32), p1 & M32
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0, k1 = (k0 + PHILOX_W0) & M32, (k1 + PHILOX_W1) & M32
    return c0, c1, c2, c3


def unit_open(u):
    """u32_to_unit_open: (0, 1], exact in fp32"""
    return ((_u64(u) >> np.uint64(8)).astype(np.float64) + 1.0) * 2.0 ** -24


def unit_closed_open(u):
    """the categorical sampler's uniform: [0, 1), exact in fp32"""
    return (_u64(u) >> np.uint64(8)).astype(np.float64) * 2.0 ** -24


def box_muller(a, b):
    u, v = unit_open(a), unit_open(b)
    r = np.sqrt(-2.0 * np.log(u))
    t = 2.0 * np.pi * v
    return r * np.cos(t), r * np.sin(t)


def policy_counter(epoch, step, q):
    assert 0 <= step < 1 << POLICY_STEP_BITS and 0 <= q < 1 << POLICY_Q_BITS
    return (int(epoch) << EPOCH_SHIFT) | (int(step) << POLICY_Q_BITS) | int(q)


def synth_counter(epoch, step, q, done=False):
    assert 0 <= step < 1 << SYNTH_STEP_BITS and 0 <= q < 1 << SYNTH_Q_BITS
    return (int(epoch) << EPOCH_SHIFT) | (int(step) << (SYNTH_Q_BITS + 1)) | (int(done) << SYNTH_DONE_BIT) | int(q)


def gaussian_eps(seed, n_rows, A, epoch, step):
    """[n_rows, A] fp64: the eps of policy_head_sample(_sd) / tc_mlp_fwd_rollout without a noise tape"""
    rows = np.arange(n_rows, dtype=np.uint64)
    cols = []
    for q in range((A + 3) // 4):
        assert q < GAUSS_Q_MAX
        x, y, z, w = philox4x32_10(rows, policy_counter(epoch, step, q), seed)
        n0, n1 = box_muller(x, y)
        n2, n3 = box_muller(z, w)
        cols += [n0, n1, n2, n3]
    return np.stack(cols, axis=1)[:, :A]


def categorical_uniforms(seed, n_rows, n_heads, epoch, step):
    """[n_heads, n_rows] fp64 (values exact in fp32): the u of categorical_sample without a uniform tape"""
    assert n_heads <= CAT_MAXH
    rows = np.arange(n_rows, dtype=np.uint64)
    return np.stack([unit_closed_open(philox4x32_10(rows, policy_counter(epoch, step, CAT_Q0 + j), seed)[0]) for j in range(n_heads)])


def synth_env_draws(seed, N, D, epoch, step):
    """(obs [N, D] fp64, done uniform [N] fp64 exact in fp32) of synth_env_step"""
    rows = np.arange(N, dtype=np.uint64)
    groups = (D + 3) // 4
    cols = []
    for q in range(groups):
        x, y, z, w = philox4x32_10(rows, synth_counter(epoch, step, q), seed ^ SYNTH_OBS_KEY_XOR)
        n0, n1 = box_muller(x, y)
        n2, n3 = box_muller(z, w)
        cols += [n0, n1, n2, n3]
    obs = np.stack(cols, axis=1)[:, :D]
    u_done = unit_open(philox4x32_10(rows, synth_counter(epoch, step, 0, done=True), seed ^ SYNTH_DONE_KEY_XOR)[0])
    return obs, u_done
