"""The host Philox restatement (tests/_philox_ref.py) against the Random123 known-answer vectors of Philox4x32-10, and the counter
layout of the device samplers: the bit fields of (epoch, step, draw index) may not overlap over their documented ranges, or two
draws of one row would come from the same Philox block."""
import itertools
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _philox_ref as P  # noqa: E402


def _words(ctr, key):
    """Random123 notation: ctr = (c0, c1, c2, c3), key = (k0, k1) -> the device's (ctr_lo, ctr_hi, key) arguments"""
    out = P.philox4x32_10((ctr[1] << 32) | ctr[0], (ctr[3] << 32) | ctr[2], (key[1] << 32) | key[0])
    return [int(w) for w in out]


def test_random123_known_answers():
    assert _words((0, 0, 0, 0), (0, 0)) == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]
    f = 0xFFFFFFFF
    assert _words((f, f, f, f), (f, f)) == [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]
    assert _words((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0)) == \
        [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]


def test_vectorised_matches_scalar():
    rows = np.arange(37, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    vec = P.philox4x32_10(rows, 12345, 0xDEADBEEFCAFEF00D)
    for i in (0, 5, 36):
        one = P.philox4x32_10(int(rows[i]), 12345, 0xDEADBEEFCAFEF00D)
        assert [int(w[i]) for w in vec] == [int(w) for w in one]


def test_uniform_mappings_are_exact_fp32_and_in_range():
    w = np.array([0, 255, 256, 0x7FFFFFFF, 0xFFFFFF00, 0xFFFFFFFF], dtype=np.uint64)
    u_open, u_co = P.unit_open(w), P.unit_closed_open(w)
    assert np.all(u_open > 0) and np.all(u_open <= 1) and u_open[-1] == 1.0
    assert np.all(u_co >= 0) and np.all(u_co < 1) and u_co[0] == 0.0
    assert np.array_equal(u_open.astype(np.float32).astype(np.float64), u_open)
    assert np.array_equal(u_co.astype(np.float32).astype(np.float64), u_co)
    n0, n1 = P.box_muller(w, w[::-1])
    assert np.all(np.isfinite(n0)) and np.all(np.isfinite(n1))


def _field_masks(fields):
    """fields: [(shift, width)] -> the bit masks of each field; asserts they are pairwise disjoint"""
    masks = [((1 << width) - 1) << shift for shift, width in fields]
    for a, b in itertools.combinations(masks, 2):
        assert a & b == 0, (hex(a), hex(b))
    return masks


def test_policy_counter_fields_do_not_overlap():
    # step < 2^16, draw index q < 16; the epoch starts above both
    _field_masks([(0, P.POLICY_Q_BITS), (P.POLICY_Q_BITS, P.POLICY_STEP_BITS), (P.EPOCH_SHIFT, 64 - P.EPOCH_SHIFT)])
    assert P.POLICY_Q_BITS + P.POLICY_STEP_BITS <= P.EPOCH_SHIFT
    # Gaussian draws (q < 8: 4 normals each, up to 32 actions) and categorical heads (q = 8 + j, j < CAT_MAXH) never share a q
    gauss = set(range(P.GAUSS_Q_MAX))
    cat = {P.CAT_Q0 + j for j in range(P.CAT_MAXH)}
    assert not gauss & cat and max(cat) < 1 << P.POLICY_Q_BITS and 4 * P.GAUSS_Q_MAX >= 31
    # the extremes of every field are distinct counters
    seen = {P.policy_counter(e, s, q) for e in (0, 1, (1 << 20) + 1) for s in (0, 1, 7, 65535) for q in range(16)}
    assert len(seen) == 3 * 4 * 16
    assert P.policy_counter(1, 0, 0) == 1 << 20 and P.policy_counter(0, 65535, 15) == (1 << 20) - 1


def test_synth_env_counter_fields_do_not_overlap():
    _field_masks([(0, P.SYNTH_Q_BITS), (P.SYNTH_DONE_BIT, 1), (P.SYNTH_Q_BITS + 1, P.SYNTH_STEP_BITS), (P.EPOCH_SHIFT, 64 - P.EPOCH_SHIFT)])
    assert P.SYNTH_Q_BITS + 1 + P.SYNTH_STEP_BITS <= P.EPOCH_SHIFT
    seen = {P.synth_counter(e, s, q, d) for e in (0, 3) for s in (0, 7, 1023) for q in (0, 1, 511) for d in (False, True)}
    assert len(seen) == 2 * 3 * 3 * 2


def test_draw_helpers_shapes_and_moments():
    eps = P.gaussian_eps(11, 4096, 31, 3, 7)
    assert eps.shape == (4096, 31)
    assert abs(eps.mean()) < 0.01 and abs(eps.var() - 1.0) < 0.02
    # q advances every four actions: columns 4..7 are not a copy of 0..3
    assert not np.allclose(eps[:, :4], eps[:, 4:8])
    u = P.categorical_uniforms(11, 4096, 8, 3, 7)
    assert u.shape == (8, 4096) and abs(u.mean() - 0.5) < 0.01
    obs, ud = P.synth_env_draws(5, 1000, 61, 0, 7)
    assert obs.shape == (1000, 61) and ud.shape == (1000,) and np.all((ud > 0) & (ud <= 1))
