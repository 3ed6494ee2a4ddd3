"""Every layer GEMM and convolution call the agents make (tests/golden/layer_census.json), replayed on fresh random operands and checked
against an fp64 reference element by element.

Each census entry is replayed in the layout the agent gave it: the first layer's chunked arena rows with the recorded chunk stride and
row stride (junk in the rows and columns the call must skip), the weights as a view at the recorded offset of an fp32 arena (plus its
``b200rl_cast_bf16`` twin when the call had one), the weight gradient's dW / db slots at the recorded offsets of split rows of the
recorded stride.  Entries that differ only in M are merged; each is run at M = 1, 127, 128, 129, the largest recorded M and that M + 1,
with the recorded split count, so the trailing splits of the small M are empty.

- The fp64 reference takes the operands the kernel stages: X after the 1/255 scaling and the normaliser in fp32, rounded to bf16 for the
  ``_tc`` entry points, as are the weights and dY (also in the bias-gradient sums).  Each element of the result must satisfy
  ``|got - ref| <= C * sqrt(R) * 2^-24 * (|A| |B|)_ij + TINY``, with R the reduction length (of the split, for weight gradients) and
  ``|A| |B|`` the fp64 product of the absolute operands (plus |bias|; times |act'| for the data gradient).  A max-norm check stays
  alongside.
- Every element the call owns is NaN before the call and finite after it; empty splits hold exact zeros.  Everything around it (the
  padding before and after Y / dX, the other parameter slots of each split row) holds a sentinel that must be unchanged.
- A second identical call is bit-identical; reduce_splits equals the ordered fp32 loop ``acc = acc + part[s]`` bit for bit.

C was calibrated on an NVIDIA H100 80GB HBM3 at a 700 W power limit.  WORST below records the worst observed ratio
|got - ref| / (sqrt(R) 2^-24 |A||B| + TINY) per entry point over the whole census.  The largest is 1.35, for linear_fwd_f32.  C = 5 is
under 4x that.  The tensor-core entry points stay under 1: their bf16 operands are exact in the reference, and the fp32 accumulation of
the wgmma chains is no worse than the CUDA cores' fmaf chains.  The file runs in about 2 minutes on that GPU."""
import json
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from test_conv_tc_gpu import ACTS, _act_grad, bf  # noqa: E402

pytestmark = [pytest.mark.gpu]
DEV = 'cuda:0'
CENSUS = os.path.join(HERE, 'golden', 'layer_census.json')
U = 2.0 ** -24
WORST = {'linear_fwd_f32': 1.347, 'linear_fwd_tc': 0.925, 'linear_bwd_data_f32': 0.814, 'linear_bwd_data_tc': 0.411,       # measured
         'linear_bwd_weight_f32': 1.308, 'linear_bwd_weight_tc': 0.533, 'conv2d_fwd_f32': 0.516, 'conv2d_fwd_tc': 0.238,
         'conv2d_bwd_data_f32': 0.298, 'conv2d_bwd_data_tc': 0.256, 'conv2d_bwd_weight_f32': 1.210, 'conv2d_bwd_weight_tc': 0.468}
C = 5.0
TINY = 4 * U                  # a few ulps of an O(1) activation: tanhf and the fast exponential of the tensor cores' ELU
MAXNORM = 1e-4
SENT = 12345.0                # the sentinel around what a call owns
PAD = 37                      # sentinel elements before and after an output
SLAB = {'linear_bwd_weight_f32': 16, 'linear_bwd_weight_tc': 64, 'conv2d_bwd_weight_f32': 16, 'conv2d_bwd_weight_tc': 64}
EDGE_M = (1, 127, 128, 129)


def _groups():
    """census entries merged over M (first layers on whole-batch rows stay dense at every M): {id: (entry, largest M, configs)}"""
    with open(CENSUS) as f:
        c = json.load(f)
    out = {}
    for e in c['golden'] + c['yaml']:
        a = dict(e['args'])
        M = a.pop('M', None)
        if 'rows_per_chunk' in a and a['rows_per_chunk'] >= M:
            a['rows_per_chunk'] = 'dense'
        key = json.dumps([e['fn'], a, e['ptr']], sort_keys=True)
        if key not in out:
            out[key] = [e, M, []]
        if M is not None and M > out[key][1]:
            out[key][0], out[key][1] = e, M
        out[key][2] += [n for n in e['configs'] if n not in out[key][2]]
    groups = {}
    for key, (e, M, configs) in sorted(out.items()):
        short = ','.join(f'{k}={v}' for k, v in sorted(e['args'].items()) if k not in ('M', 'chunk_stride', 'x_ld'))
        gid = f"{e['fn']}[{short}]"
        i = 1
        while gid in groups:
            i += 1
            gid = f"{e['fn']}[{short}]#{i}"
        groups[gid] = (e, M, configs)
    return groups


GROUPS = _groups() if os.path.exists(CENSUS) else {}


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _chunk_rows(M, rpc, cs):
    m = torch.arange(M, device=DEV)
    return (m // rpc) * cs + m % rpc


def _arena_rows(g, M, rpc, cs, ld, D, u8, align_bytes, normed):
    """(X: the view the kernel reads, rows: [M, D] the logical rows, norm pair or None): the rows sit at their chunk positions in an
    arena of junk, X starts `align_bytes` past a 16-byte boundary"""
    es = 1 if u8 else 4
    off = align_bytes // es
    idx = _chunk_rows(M, rpc, cs)
    n = off + (int(idx.max()) + 1) * ld + 8
    if u8:
        arena = torch.randint(0, 256, (n,), generator=g, dtype=torch.uint8).to(DEV)
    else:
        arena = (torch.rand(n, generator=g).to(DEV) - 0.5) * 2e6          # junk: any read of it blows the bound
    X = arena[off:]
    ridx = (idx[:, None] * ld + torch.arange(D, device=DEV)[None, :])
    if u8:
        rows = torch.randint(0, 256, (M, D), generator=g, dtype=torch.uint8).to(DEV)
    else:
        rows = torch.randn(M, D, generator=g).to(DEV) * 3
    X.view(-1)[ridx.reshape(-1)] = rows.reshape(-1)
    norm = None
    if normed:           # spread so that some elements clamp at +-5 and some fall between 4 and 5
        if u8:
            norm = (torch.rand(D, generator=g).to(DEV) * 0.5, torch.rand(D, generator=g).to(DEV) * 0.25 + 0.05)
        else:
            norm = (torch.randn(D, generator=g).to(DEV) * 0.5, torch.rand(D, generator=g).to(DEV) + 0.5)
    return X, rows, norm


def _staged(rows, norm, tc):
    """what the kernel stages from the rows, in fp64: /255 and the normaliser in fp32, then bf16 on the tensor cores.  The divisor is a
    device tensor: torch multiplies by the reciprocal of a Python scalar, one ulp off the kernel's division, which the bf16 rounding can
    turn into a whole bf16 ulp"""
    v = rows.float() / torch.tensor(255.0, device=rows.device) if rows.dtype == torch.uint8 else rows.float()
    if norm is not None:
        v = torch.clamp((v - norm[0]) / norm[1], -5.0, 5.0)
    return bf(v) if tc else v.double()


def _weights(g, shape, w_mod8, bias, twin):
    """W as a view of an fp32 arena at an element offset = w_mod8 (mod 8), b right after it, and the bf16 twin of the arena"""
    from rl_games_b200 import ops
    n = math.prod(shape)
    off = 8 + w_mod8
    flat = torch.zeros(off + n + shape[0] + 16, device=DEV)
    fan_in = n // shape[0]
    flat[off:off + n] = torch.randn(n, generator=g).to(DEV) / fan_in ** 0.5
    flat[off + n:off + n + shape[0]] = torch.randn(shape[0], generator=g).to(DEV) * 0.1
    W = flat[off:off + n].view(shape)
    b = flat[off + n:off + n + shape[0]] if bias else None
    arena = None
    if twin:
        fb = torch.empty(flat.numel(), dtype=torch.bfloat16, device=DEV)
        ops.cast_bf16(flat, fb)
        arena = (flat, fb)
    return W, b, arena


def _padded(n, fill=float('nan')):
    """a buffer of PAD sentinels, n owned elements (prefilled with `fill`), PAD sentinels"""
    buf = torch.full((n + 2 * PAD,), SENT, device=DEV)
    buf[PAD:PAD + n] = fill
    return buf, buf[PAD:PAD + n]


def _act_fp64(x, act):
    return ACTS[act](x) if act else x


def _bits(t):
    return t.contiguous().view(torch.int32).clone()


class _Ratios:
    """the worst |got - ref| / (sqrt(R) 2^-24 mag + TINY) per entry point over the run"""
    seen = {}

    @classmethod
    def check(cls, fn, what, got, ref, mag, R, maxnorm=True):
        got = got.double()
        assert torch.isfinite(got).all(), f'{what}: an owned element is not written (NaN) or not finite'
        err = (got - ref).abs()
        ratio = (err / (math.sqrt(R) * U * mag + TINY)).max().item()
        cls.seen[fn] = max(cls.seen.get(fn, 0.0), ratio)
        if ratio > C:
            i = int((err / (math.sqrt(R) * U * mag + TINY)).argmax())
            raise AssertionError(f'{what}: element {i}: got {got.reshape(-1)[i].item():.9g}, fp64 {ref.reshape(-1)[i].item():.9g}, '
                                 f'|A||B| {mag.reshape(-1)[i].item():.3g}, R {R}: ratio {ratio:.3g} > C = {C}')
        if not maxnorm:
            return
        scale = ref.abs().max().item() + 1e-30
        assert err.max().item() <= MAXNORM * scale, f'{what}: max-norm error {err.max().item():.3e} at scale {scale:.3e}'


def _check_sentinel(buf, owned_mask, what):
    outside = buf[~owned_mask]
    assert (outside == SENT).all(), f'{what}: {int((outside != SENT).sum())} elements outside the owned range changed'


def _twice(call, reset, out):
    """the call on freshly prefilled outputs, then again: bit-identical"""
    reset()
    call()
    first = _bits(out)
    reset()
    call()
    torch.cuda.synchronize()
    assert torch.equal(first, _bits(out)), 'a second identical call is not bit-identical'


def _split_ranges(fn, P, S):
    rps = -(-P // S)
    rps = -(-rps // SLAB[fn]) * SLAB[fn]
    return rps, [(min(s * rps, P), min((s + 1) * rps, P)) for s in range(S)]


def _wgrad_check(fn, what, part, S, dw_off, db_off, n_w, n_b, dY2, X2, P, wshape):
    """per-split dW = dY_s^T X_s, db = colsum(dY_s) against fp64; empty splits exact zeros; everything else in the rows untouched"""
    rps, ranges = _split_ranges(fn, P, S)
    pad = S * rps - P
    Yp = F.pad(dY2, (0, 0, 0, pad)).view(S, rps, -1)
    Xp = F.pad(X2, (0, 0, 0, pad)).view(S, rps, -1)
    ref = torch.bmm(Yp.transpose(1, 2), Xp)
    mag = torch.bmm(Yp.abs().transpose(1, 2), Xp.abs())
    for s, (lo, hi) in enumerate(ranges):
        got_w = part[s, dw_off:dw_off + n_w].view(wshape[0], -1)
        if hi <= lo:
            assert torch.equal(got_w, torch.zeros_like(got_w)), f'{what}: empty split {s} of {S}: dW not zero'
        else:
            _Ratios.check(fn, f'{what} dW split {s}/{S}', got_w, ref[s], mag[s], hi - lo, maxnorm=False)
        if db_off is not None:
            got_b = part[s, db_off:db_off + n_b]
            if hi <= lo:
                assert torch.equal(got_b, torch.zeros_like(got_b)), f'{what}: empty split {s} of {S}: db not zero'
            else:
                _Ratios.check(fn, f'{what} db split {s}/{S}', got_b, Yp[s].sum(0), Yp[s].abs().sum(0), hi - lo, maxnorm=False)
    # the max-norm check on the sum over the splits (a split's single db element may cancel to nearly nothing)
    for name, got, r in (('dW', part[:, dw_off:dw_off + n_w].double().sum(0), ref.sum(0).reshape(-1)),
                         ('db', part[:, db_off:db_off + n_b].double().sum(0) if db_off is not None else None, Yp.sum((0, 1)))):
        if got is not None:
            err, scale = (got - r).abs().max().item(), r.abs().max().item() + 1e-30
            assert err <= MAXNORM * scale, f'{what} {name}: max-norm error {err:.3e} of the split sum at scale {scale:.3e}'
    owned = torch.zeros_like(part, dtype=torch.bool)
    owned[:, dw_off:dw_off + n_w] = True
    if db_off is not None:
        owned[:, db_off:db_off + n_b] = True
    _check_sentinel(part, owned, what)


def _part_buffer(S, split_stride, dw_off, n_w, db_off, n_b):
    part = torch.full((S, split_stride), SENT, device=DEV)

    def reset():
        part.fill_(SENT)
        part[:, dw_off:dw_off + n_w] = float('nan')
        if db_off is not None:
            part[:, db_off:db_off + n_b] = float('nan')
    return part, reset


# ------------------------------------------------------------------------------------------------------------------- linear
def _linear(fn, e, M, seed):
    from rl_games_b200 import ops
    a, p = e['args'], e['ptr']
    tc = fn.endswith('_tc')
    g = _gen(seed)
    K, N = a['K'], a['Nout']
    what = f'{fn} M={M}'
    if fn.startswith('linear_fwd') or fn.startswith('linear_bwd_weight'):
        rpc = M if a['rows_per_chunk'] >= e['args']['M'] else a['rows_per_chunk']
        X, rows, norm = _arena_rows(g, M, rpc, a['chunk_stride'], a['x_ld'], K, False, p['x_align16'], p['norm'])
        nm, ns = norm if norm is not None else (None, None)
        xin = _staged(rows, norm, tc)
        chunk = dict(rows_per_chunk=rpc, chunk_stride=a['chunk_stride'], x_ld=a['x_ld'], norm_mean=nm, norm_std=ns, M=M)
    if fn.startswith('linear_fwd'):
        W, b, arena = _weights(g, (N, K), p['w_mod8'], p['bias'], p.get('W_bf16'))
        kw = dict(bf16_arena=arena) if tc else {}
        prev = torch.randn(M, N, generator=g).to(DEV) if a['accumulate'] else None
        buf, Y = _padded(M * N)
        Y = Y.view(M, N)

        def reset():
            buf.fill_(SENT)
            Y.copy_(prev) if prev is not None else Y.fill_(float('nan'))
        f = ops.linear_fwd_tc if tc else ops.linear_fwd
        _twice(lambda: f(X, W, b, Y, a['act'], accumulate=bool(a['accumulate']), **chunk, **kw), reset, buf)
        Wd = bf(W) if tc else W.double()
        pre = xin @ Wd.T
        mag = xin.abs() @ Wd.abs().T
        if b is not None:
            pre, mag = pre + b.double(), mag + b.double().abs()
        if prev is not None:
            pre, mag = pre + prev.double(), mag + prev.double().abs()
        _Ratios.check(fn, what, Y, _act_fp64(pre, a['act']), mag, K)
        owned = torch.zeros_like(buf, dtype=torch.bool)
        owned[PAD:PAD + M * N] = True
        _check_sentinel(buf, owned, what)
    elif fn.startswith('linear_bwd_data'):
        W, _, arena = _weights(g, (N, K), p['w_mod8'], False, p.get('W_bf16'))
        kw = dict(bf16_arena=arena) if tc else {}
        dY = torch.randn(M, N, generator=g).to(DEV)
        A_prev = _act_fp64(torch.randn(M, K, generator=g).to(DEV), a['act_prev']).float() if p['A_prev'] else None
        buf, dX = _padded(M * K)
        dX = dX.view(M, K)

        def reset():
            buf.fill_(SENT)
            dX.fill_(float('nan'))
        f = ops.linear_bwd_data_tc if tc else ops.linear_bwd_data
        _twice(lambda: f(dY, W, A_prev, dX, a['act_prev'], M=M, **kw), reset, buf)
        dYd, Wd = (bf(dY), bf(W)) if tc else (dY.double(), W.double())
        d = _act_grad(A_prev.double(), a['act_prev']) if A_prev is not None else torch.ones(M, K, dtype=torch.float64, device=DEV)
        _Ratios.check(fn, what, dX, (dYd @ Wd) * d, (dYd.abs() @ Wd.abs()) * d.abs(), N)
        owned = torch.zeros_like(buf, dtype=torch.bool)
        owned[PAD:PAD + M * K] = True
        _check_sentinel(buf, owned, what)
    else:
        S, ss, dw_off = a['n_splits'], a['split_stride'], p['dw_off']
        db_off = dw_off + p['db_rel'] if p['db'] else None
        part, reset = _part_buffer(S, ss, dw_off, N * K, db_off, N)
        dY = torch.randn(M, N, generator=g).to(DEV)
        f = ops.linear_bwd_weight_tc if tc else ops.linear_bwd_weight
        db_view = part[0, db_off:] if db_off is not None else None
        _twice(lambda: f(dY, X, part[0, dw_off:], db_view, K, N, S, split_stride=ss, **chunk), reset, part)
        _wgrad_check(fn, what, part, S, dw_off, db_off, N * K, N, bf(dY) if tc else dY.double(), xin, M, (N, K))


# ------------------------------------------------------------------------------------------------------------------- conv2d
def _conv(fn, e, M, seed):
    from rl_games_b200 import ops
    a, p = e['args'], e['ptr']
    tc = fn.endswith('_tc')
    g = _gen(seed)
    C_, H, Wd_, Co, KH, KW, st, pad = a['C'], a['H'], a['Wd'], a['Cout'], a['KH'], a['KW'], a['stride'], a['pad']
    geo = (C_, H, Wd_, st, pad)
    Ho, Wo = (H + 2 * pad - KH) // st + 1, (Wd_ + 2 * pad - KW) // st + 1
    L, R, D = Ho * Wo, C_ * KH * KW, C_ * H * Wd_
    what = f'{fn} M={M}'
    if not fn.startswith('conv2d_bwd_data'):
        rpc = M if a['rows_per_chunk'] >= e['args']['M'] else a['rows_per_chunk']
        nhwc = bool(a['x_nhwc'])
        X, rows, norm = _arena_rows(g, M, rpc, a['chunk_stride'], a['x_ld'], D, bool(a['x_u8']), p['x_align16'], p['norm'])
        nm, ns = norm if norm is not None else (None, None)
        v = _staged(rows, norm, tc)
        xin = v.view(M, H, Wd_, C_).permute(0, 3, 1, 2) if nhwc else v.view(M, C_, H, Wd_)
        cols = F.unfold(xin, (KH, KW), stride=st, padding=pad)                  # [M, R, L]
        chunk = dict(nhwc=nhwc, rows_per_chunk=rpc, chunk_stride=a['chunk_stride'], x_ld=a['x_ld'], norm_mean=nm, norm_std=ns)
    if fn.startswith('conv2d_fwd'):
        W, b, arena = _weights(g, (Co, C_, KH, KW), p.get('w_mod8', p.get('wb_mod8')), p['bias'], tc)
        kw = dict(bf16_arena=arena) if tc else {}
        buf, Y = _padded(M * Co * L)
        Y = Y.view(M, Co, Ho, Wo)

        def reset():
            buf.fill_(SENT)
            Y.fill_(float('nan'))
        f = ops.conv2d_fwd_tc if tc else ops.conv2d_fwd
        _twice(lambda: f(X, W, b, Y, geo, a['act'], M, **chunk, **kw), reset, buf)
        W2 = (bf(W) if tc else W.double()).view(Co, R)
        pre, mag = W2 @ cols, W2.abs() @ cols.abs()
        del cols
        if b is not None:
            pre, mag = pre + b.double()[:, None], mag + b.double().abs()[:, None]
        _Ratios.check(fn, what, Y.view(M, Co, L), _act_fp64(pre, a['act']), mag, R)
        owned = torch.zeros_like(buf, dtype=torch.bool)
        owned[PAD:PAD + M * Co * L] = True
        _check_sentinel(buf, owned, what)
    elif fn.startswith('conv2d_bwd_data'):
        W, _, arena = _weights(g, (Co, C_, KH, KW), p.get('w_mod8', p.get('wb_mod8')), False, tc)
        kw = dict(bf16_arena=arena) if tc else {}
        dY = torch.randn(M, Co, Ho, Wo, generator=g).to(DEV)
        A_prev = _act_fp64(torch.randn(M, C_, H, Wd_, generator=g).to(DEV), a['act_prev']).float() if p['A_prev'] else None
        buf, dX = _padded(M * D)
        dX = dX.view(M, C_, H, Wd_)

        def reset():
            buf.fill_(SENT)
            dX.fill_(float('nan'))
        f = ops.conv2d_bwd_data_tc if tc else ops.conv2d_bwd_data
        _twice(lambda: f(dY, W, A_prev, dX, geo, a['act_prev'], M, **kw), reset, buf)
        W2 = (bf(W) if tc else W.double()).view(Co, R)
        dYd = (bf(dY) if tc else dY.double()).view(M, Co, L)
        fold = lambda t: F.fold(t, (H, Wd_), (KH, KW), stride=st, padding=pad)      # noqa: E731
        d = _act_grad(A_prev.double(), a['act_prev']) if A_prev is not None else 1.0
        ref = fold(W2.T @ dYd) * d
        mag = fold(W2.abs().T @ dYd.abs()) * (d.abs() if A_prev is not None else 1.0)
        _Ratios.check(fn, what, dX, ref, mag, Co * KH * KW)
        owned = torch.zeros_like(buf, dtype=torch.bool)
        owned[PAD:PAD + M * D] = True
        _check_sentinel(buf, owned, what)
    else:
        S, ss, dw_off = a['n_splits'], a['split_stride'], p['dw_off']
        db_off = dw_off + p['db_rel'] if p['db'] else None
        part, reset = _part_buffer(S, ss, dw_off, Co * R, db_off, Co)
        dY = torch.randn(M, Co, Ho, Wo, generator=g).to(DEV)
        f = ops.conv2d_bwd_weight_tc if tc else ops.conv2d_bwd_weight
        db_view = part[0, db_off:] if db_off is not None else None
        _twice(lambda: f(dY, X, part[0, dw_off:], db_view, (Co, C_, KH, KW), geo, S, M, ss, **chunk), reset, part)
        dY2 = (bf(dY) if tc else dY.double()).view(M, Co, L).permute(0, 2, 1).reshape(M * L, Co)
        X2 = cols.permute(0, 2, 1).reshape(M * L, R)
        del cols
        _wgrad_check(fn, what, part, S, dw_off, db_off, Co * R, Co, dY2, X2, M * L, (Co, R))


def _reduce(e, seed):
    from rl_games_b200 import ops
    a = e['args']
    n, S, ss = a['n'], a['n_splits'], a['split_stride']
    g = _gen(seed)
    part = torch.randn(S, ss, generator=g).to(DEV) * torch.exp(torch.randn(S, ss, generator=g).to(DEV) * 3)
    buf, out = _padded(n)

    def reset():
        buf.fill_(SENT)
        out.fill_(float('nan'))
    _twice(lambda: ops.reduce_splits(part, out, n, S, split_stride=ss), reset, buf)
    acc = torch.zeros(n, device=DEV)
    for s in range(S):
        acc = acc + part[s, :n]
    assert torch.equal(_bits(out), _bits(acc)), 'reduce_splits differs from the ordered fp32 loop'
    owned = torch.zeros_like(buf, dtype=torch.bool)
    owned[PAD:PAD + n] = True
    _check_sentinel(buf, owned, 'reduce_splits')


@pytest.mark.parametrize('gid', list(GROUPS))
def test_census_entry_matches_fp64_where_it_writes(gid):
    e, M_rec, configs = GROUPS[gid]
    fn = e['fn']
    try:
        if fn == 'reduce_splits_f32':
            _reduce(e, 1)
            return
        for i, M in enumerate(sorted(set(EDGE_M) | {M_rec, M_rec + 1})):
            (_conv if fn.startswith('conv2d') else _linear)(fn, e, M, 100 + i)
            torch.cuda.synchronize()
    except AssertionError as ex:
        raise AssertionError(f'{gid} (made by: {", ".join(configs)}): {ex}') from None
    finally:
        torch.cuda.empty_cache()


def test_zz_report_the_worst_ratio_per_entry_point():
    """prints the measured ratios (run with -s); the bound itself is asserted per entry"""
    for fn, r in sorted(_Ratios.seen.items()):
        print(f'census worst ratio {fn}: {r:.3f}')
