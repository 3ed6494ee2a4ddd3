"""Host restatement of the wide categorical kernels' draw (rl_games_b200/csrc/discrete.cu categorical_sample_wide_kernel, documented in
include/b200rl.h): the Philox counters of heads j >= 8 and the order in which a head's cdf is summed.

Philox: head j of row e draws word x of Philox4x32-10 at ctr_lo = e | (j >> 3) << 32, ctr_hi = policy_counter(epoch, step, 8 + (j & 7)),
keyed by the seed.  For j < 8 that is _philox_ref.categorical_uniforms, bit for bit.

cdf: 32 actions at a time, cdf_k = carry + S(k) in fp32, S the inclusive Hillis-Steele scan of p over the chunk (steps d = 1, 2, 4, 8,
16: x_l += x_{l-d} for l >= d), carry = the cdf at the previous chunk's last action.  action = #{k : cdf_k <= u}, clamped to the last
action with p > 0."""
import numpy as np

from _philox_ref import CAT_Q0, philox4x32_10, policy_counter, unit_closed_open


def wide_counters(rows, j, epoch, step):
    """(ctr_lo, ctr_hi) of head j for the given rows"""
    rows = np.asarray(rows, dtype=np.uint64)
    return rows | (np.uint64(j >> 3) << np.uint64(32)), policy_counter(epoch, step, CAT_Q0 + (j & 7))


def categorical_uniforms_wide(seed, n_rows, n_heads, epoch, step):
    """[n_heads, n_rows] fp64 (values exact in fp32): the u of the wide sampler without a uniform tape"""
    rows = np.arange(n_rows, dtype=np.uint64)
    out = []
    for j in range(n_heads):
        lo, hi = wide_counters(rows, j, epoch, step)
        out.append(unit_closed_open(philox4x32_10(lo, hi, seed)[0]))
    return np.stack(out)


def wide_cdf(p):
    """[B, K] fp32 probabilities -> [B, K] fp32 cdf in the wide kernel's summation order"""
    p = np.asarray(p, dtype=np.float32)
    B, K = p.shape
    out = np.empty_like(p)
    carry = np.zeros(B, dtype=np.float32)
    for c0 in range(0, K, 32):
        x = np.zeros((B, 32), dtype=np.float32)
        n = min(32, K - c0)
        x[:, :n] = p[:, c0:c0 + n]
        for d in (1, 2, 4, 8, 16):
            y = x.copy()
            x[:, d:] = y[:, d:] + y[:, :-d]
        cdf = carry[:, None] + x
        out[:, c0:c0 + n] = cdf[:, :n]
        carry = cdf[:, 31]
    return out


def wide_inverse_cdf(p, u):
    """actions of the wide sampler for fp32 probabilities p [B, K] and uniforms u [B]; also the distance of u to the nearest cdf value,
    under which a one-ulp difference in p could move the action"""
    p = np.asarray(p, dtype=np.float32)
    u = np.asarray(u, dtype=np.float32)
    cdf = wide_cdf(p)
    count = (cdf <= u[:, None]).sum(axis=1)
    last = np.where(p > 0, np.arange(p.shape[1])[None, :], 0).max(axis=1)
    return np.minimum(count, last), np.abs(cdf - u[:, None]).min(axis=1)
