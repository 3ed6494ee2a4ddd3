"""The policy heads away from the benchmark's 8 actions, on scratch buffers nobody zeroed, and on the device-RNG path.

A. The fused bf16 tensor-core train step (tc_mlp_fwd_train + tc_mlp_bwd) against the kernel-faithful reference of
   test_tc_faithful_gpu.py (bf16 rounding where the kernels round, exact products, the oracle's loss functions, autograd for
   d(head)) at every kind of action count the kernels branch on: A = 1 .. 15, A % 4 == 0 or not, narrow / native / wide trunks,
   masked rows, chunked arena rows, partial last tiles and CTAs that own several tiles.
B. The tiled scratch buffers (act1..3, d_head, delta1/2, xtile, wpack) filled with 0xFF bytes (bf16 NaN) give the same bytes as
   zero-filled ones: the kernels write every byte a later kernel reads, padding included.
C. The fused rollout forward at the same action counts, through both store branches of its epilogue.
D. The fp32 head kernels (ppo_head_loss, policy_head_sample, their state-dependent-sigma editions) against fp64 autograd at every
   shared-memory regime: head widths up to the last that fits, A up to 31, every activation of the last layer.
E. The device Philox draws against the bit-exact host restatement tests/_philox_ref.py: each sampler without a tape equals the
   same sampler fed the host draws as a tape.
F. The optimiser tail's refresh of the packed bf16 weights equals a fresh pack of the updated parameters, byte for byte."""
import math
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import ppo_oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _philox_ref as PR  # noqa: E402
from test_mlp_tc_gpu import decode_tiles, rel_l2, cosine  # noqa: E402
from test_tc_faithful_gpu import ACTS, NATIVE, bf, mm  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = 'cuda'
ARG_UNSUPPORTED = 'argument error -2'      # B200RL_EUNSUPPORTED


def make_net(g, D, units, A):
    ins, W, b = D, [], []
    for u in units:
        W.append((torch.randn(u, ins, generator=g) / math.sqrt(ins)).to(DEV))
        b.append((torch.randn(u, generator=g) * 0.1).to(DEV))
        ins = u
    Wh = (torch.randn(A + 1, ins, generator=g) / math.sqrt(ins)).to(DEV)
    bh = (torch.randn(A + 1, generator=g) * 0.1).to(DEV)
    logstd = (torch.randn(A, generator=g) * 0.2).to(DEV)
    return W, b, Wh, bh, logstd


def flat_offsets(D, units, A):
    """flat parameter layout of the model (logstd first): name -> offset, total size"""
    offs, o, ins = {}, A, D
    for i, u in enumerate(units):
        offs[f'W{i}'] = o; o += u * ins
        offs[f'b{i}'] = o; o += u
        ins = u
    offs['W_head'] = o; o += (A + 1) * ins
    offs['b_head'] = o; o += A + 1
    return offs, o


def _raises_unsupported(fn):
    try:
        fn()
    except Exception as e:      # B200RLError
        return ARG_UNSUPPORTED in str(e)
    return False


# ================================================================================ A / B: fused train step
def _train_inputs(A, D, units, H, N, epm, masked, seed):
    g = torch.Generator().manual_seed(seed)
    net = make_net(g, D, units, A)
    e0 = 128 if N > epm else 0
    x = dict(obs=(torch.randn(H, N, D, generator=g) * 2 + 0.5), nm=torch.randn(D, generator=g) * 0.3, ns=torch.rand(D, generator=g) + 0.7,
             actions=torch.randn(H, N, A, generator=g), old_mu=torch.randn(H, N, A, generator=g) * 0.5,
             old_sigma=torch.rand(H, N, A, generator=g) + 0.5, old_v=torch.randn(H, N, generator=g), ret=torch.randn(H, N, generator=g),
             old_nlp=torch.randn(H, N, generator=g) * 0.3 + 0.9 * A, adv=torch.randn(H, N, generator=g),
             mask=(torch.rand(H, N, generator=g) < 0.7).float() if masked else None)
    x = {k: (None if v is None else v.to(DEV)) for k, v in x.items()}
    x.update(H=H, N=N, epm=epm, e0=e0, M=H * epm, D=D, units=units, A=A)
    x['inv'] = torch.tensor([1.0 / max(float(x['mask'][:, e0:e0 + epm].sum()), 1.0)], device=DEV) if masked else None
    return net, x


def _rows(x, t):
    """arena tensor [H, N, ...] -> minibatch rows in kernel order (t * epm + e)"""
    return torch.cat([t[k, x['e0']:x['e0'] + x['epm']] for k in range(x['H'])])


def _faithful_reference(net, x, actname, e_clip=0.2, critic_coef=2.0):
    """test_tc_faithful_gpu's recipe for any A and trunk width"""
    _, act_fn, act_grad = ACTS[actname]
    W, b, Wh, bh, logstd = net
    rows = lambda t: _rows(x, t)   # noqa: E731
    xb = bf(torch.clamp((rows(x['obs']) - x['nm']) * (1.0 / x['ns']), -5.0, 5.0))
    Wb, Whb = [bf(w) for w in W], bf(Wh)
    a1 = bf(act_fn(mm(xb, Wb[0]) + b[0]))
    a2 = bf(act_fn(mm(a1, Wb[1]) + b[1]))
    a3 = bf(act_fn(mm(a2, Wb[2]) + b[2]))
    head = (mm(a3, Whb) + bh).requires_grad_()
    ls = logstd.clone().requires_grad_()
    value, mu = head[:, 0:1], head[:, 1:]
    sigma = torch.exp(ls).expand_as(mu)
    nlp = O.neglogp_fn(rows(x['actions']), mu, sigma, ls.expand_as(mu))
    a_l = O.actor_loss(rows(x['old_nlp']), nlp, rows(x['adv']), True, e_clip, smooth=True)
    c_l = O.critic_loss(rows(x['old_v']).unsqueeze(1), value, e_clip, rows(x['ret']).unsqueeze(1), True)
    ent = (0.5 + 0.5 * math.log(2 * math.pi) + ls.expand_as(mu)).sum(-1)
    b_l = (mu * mu).sum(-1)
    mk = None if x['mask'] is None else rows(x['mask'])
    (a_m, c_m, e_m, b_m), _ = O.apply_masks([a_l.unsqueeze(1), c_l, ent.unsqueeze(1), b_l.unsqueeze(1)], mk)
    loss = a_m + 0.5 * c_m * critic_coef - e_m * 0.0 + b_m * 0.0
    loss.backward()
    kl_rows = O.policy_kl(mu.detach(), sigma.detach(), rows(x['old_mu']), rows(x['old_sigma']), reduce=False)
    kl = kl_rows.mean() if mk is None else (kl_rows * mk).sum() / mk.sum().clamp(min=1.0)
    dh = bf(head.grad)
    d3 = bf(mm(dh, Whb.t().contiguous()) * act_grad(a3))
    d2 = bf(mm(d3, Wb[2].t().contiguous()) * act_grad(a2))
    d1 = bf(mm(d2, Wb[1].t().contiguous()) * act_grad(a1))
    grads = {'W_head': mm(dh.t().contiguous(), a3.t().contiguous()), 'b_head': dh.sum(0),
             'W2': mm(d3.t().contiguous(), a2.t().contiguous()), 'b2': d3.sum(0),
             'W1': mm(d2.t().contiguous(), a1.t().contiguous()), 'b1': d2.sum(0),
             'W0': mm(d1.t().contiguous(), xb.t().contiguous()), 'b0': d1.sum(0)}
    return dict(acts=(a1, a2, a3), mu=mu.detach(), sigma=sigma.detach(), stats=[float(a_m), float(c_m), float(e_m), float(b_m), float(kl)],
                dh=dh, dls=ls.grad, d2=d2, d1=d1, grads=grads)


def _run_train_step(ops, net, x, act_id, fill):
    """tc_mlp_fwd_train + ppo_loss_finalize + tc_mlp_bwd + reduce_splits, every scratch buffer pre-filled with the byte `fill`"""
    from rl_games_b200.ops import LossCfg
    W, b, Wh, bh, logstd = net
    D, units, A, M, N, epm, e0 = x['D'], x['units'], x['A'], x['M'], x['N'], x['epm'], x['e0']
    wide = ops.tc_kind(D, units, A) == 2
    sl = lambda t: None if t is None else t[0, e0:]   # noqa: E731
    cfg = LossCfg(0.2, 2.0, 0.0, 1, 2, 1, 1, 1)
    n_tiles = (M + 127) // 128
    tb = ops.tc_tile_bytes(D, units, A)
    buf = lambda n: torch.full((n,), fill, dtype=torch.uint8, device=DEV)   # noqa: E731
    wpack = buf(ops.tc_pack_bytes(D, units, A))
    ops.tc_pack_weights(W[0], W[1], W[2], Wh, D, units, A, wpack)
    act = [buf(n_tiles * tb[i]) for i in range(3)]
    dhead, delta2, delta1 = buf(n_tiles * tb[3]), buf(n_tiles * tb[1]), buf(n_tiles * tb[0])
    xt = None if wide else buf(n_tiles * ops.tc_xtile_bytes(D, units, A))
    mu_t, sg_t = x['old_mu'].clone(), x['old_sigma'].clone()
    partials = torch.zeros(148, ops.loss_partial_stride(), dtype=torch.float64, device=DEV)
    nbt = ops.tc_mlp_fwd_train(sl(x['obs']), epm, N, D, x['nm'], x['ns'], wpack, b, bh, logstd, units, M, A, sl(x['actions']), sl(mu_t),
                               sl(sg_t), sl(x['old_v']), sl(x['ret']), sl(x['old_nlp']), sl(x['adv']), sl(x['mask']), cfg, x['inv'], act,
                               dhead, partials, xtile=xt, activation=act_id)
    stats, dls = torch.zeros(16, device=DEV), torch.empty(A, device=DEV)
    ops.ppo_loss_finalize(partials, nbt, A, torch.tensor([0.0], device=DEV), stats, dls)
    offs, P = flat_offsets(D, units, A)
    part = torch.full((148, P), float('nan'), device=DEV)
    npart = ops.tc_mlp_bwd(sl(x['obs']), epm, N, D, x['nm'], x['ns'], wpack, units, M, A, act, dhead, delta2, delta1, part, P, offs,
                           xtile=xt, activation=act_id)
    grad = torch.zeros(P, device=DEV)
    ops.reduce_splits(part[0, A:], grad[A:], P - A, npart, split_stride=P)
    torch.cuda.synchronize()
    return dict(wpack=wpack, act=act, dhead=dhead, delta2=delta2, delta1=delta1, mu=mu_t, sigma=sg_t, stats=stats, dls=dls, grad=grad,
                offs=offs, n_tiles=n_tiles)


# A, D, units, H, N, epm, masked, activation
TRAIN_CASES = [
    (1, 17, [128, 64, 32], 4, 512, 256, False, 'elu'),
    (1, 60, [256, 128, 64], 1, 1000, 1000, True, 'elu'),           # one chunk of 1000 rows (not a multiple of 128): partial last tile
    (2, 60, [256, 128, 64], 2, 384, 128, True, 'elu'),
    (3, 17, [128, 64, 32], 1, 1000, 1000, True, 'elu'),
    (3, 105, [256, 128, 64], 4, 512, 256, False, 'elu'),
    (5, 105, [256, 128, 64], 2, 384, 128, True, 'elu'),
    (5, 17, [128, 64, 32], 2, 512, 256, False, 'relu'),
    (6, 60, [256, 128, 64], 4, 10240, 10112, True, 'elu'),         # 316 tiles: every CTA owns two or three
    (6, 17, [128, 64, 32], 1, 700, 700, False, 'elu'),
    (7, 60, [128, 64, 32], 2, 384, 128, True, 'relu'),
    (8, 105, [128, 64, 32], 1, 1000, 1000, False, 'elu'),
    (12, 60, [256, 128, 64], 4, 512, 256, True, 'elu'),
    (12, 17, [128, 64, 32], 1, 333, 333, False, 'elu'),
    (15, 17, [128, 64, 32], 4, 10240, 10112, False, 'elu'),        # multi-tile CTAs at the largest action count
    (15, 105, [256, 128, 64], 2, 384, 128, True, 'elu'),
    (15, 60, [256, 128, 64], 1, 1000, 1000, True, 'relu'),
]


@pytest.mark.parametrize('A,D,units,H,N,epm,masked,actname', TRAIN_CASES)
def test_tc_train_step_vs_faithful_reference(A, D, units, H, N, epm, masked, actname):
    from rl_games_b200 import ops
    assert ops.tc_kind(D, units, A) == (2 if D > 64 else 1)
    net, x = _train_inputs(A, D, units, H, N, epm, masked, seed=1000 * A + D + N)
    ref = _faithful_reference(net, x, actname)
    out = _run_train_step(ops, net, x, ACTS[actname][0], 0)
    M, n_tiles, rep = x['M'], out['n_tiles'], {}
    for i, (C, r) in enumerate(zip(units, ref['acts'])):
        full = decode_tiles(out['act'][i], n_tiles, NATIVE[i])[:M]
        if C < NATIVE[i]:
            assert float(full[:, C:].abs().max()) == 0.0, i       # padded units are exactly zero
        rep[f'a{i + 1}'] = rel_l2(full[:, :C], r)
        assert rep[f'a{i + 1}'] < 3e-3, (i, rep)
    got_mu = _rows(x, out['mu'])
    rep['mu_rel_l2'] = rel_l2(got_mu, ref['mu'])
    assert rep['mu_rel_l2'] < 1e-3, rep
    torch.testing.assert_close(got_mu, ref['mu'], rtol=0, atol=6e-3)
    # the minibatch's rows of old_mu / old_sigma are rewritten with the new mu / sigma; every other arena row is untouched
    torch.testing.assert_close(_rows(x, out['sigma']), ref['sigma'], rtol=1e-6, atol=0)
    keep = torch.ones(x['H'], x['N'], dtype=torch.bool, device=DEV)
    keep[:, x['e0']:x['e0'] + epm] = False
    assert torch.equal(out['mu'][keep], x['old_mu'][keep]) and torch.equal(out['sigma'][keep], x['old_sigma'][keep])
    for k in range(5):
        rep[f'stat{k}'] = (float(out['stats'][k]), ref['stats'][k])
        assert float(out['stats'][k]) == pytest.approx(ref['stats'][k], rel=5e-3, abs=2e-5), (k, rep)
    dh_t = decode_tiles(out['dhead'], n_tiles, 16)[:M, :A + 1]
    rep['d_head'] = rel_l2(dh_t, ref['dh'])
    assert rep['d_head'] < 1e-2 and cosine(dh_t, ref['dh']) > 0.9999, rep
    rep['d_logstd'] = rel_l2(out['dls'], ref['dls'])
    assert rep['d_logstd'] < 2e-3, rep
    for name, C, CN, r in (('delta2', units[1], NATIVE[1], ref['d2']), ('delta1', units[0], NATIVE[0], ref['d1'])):
        got = decode_tiles(out[name], n_tiles, CN)[:M, :C]
        rep[name] = rel_l2(got, r)
        assert rep[name] < 1.5e-2 and cosine(got, r) > 0.9999, rep
    for k, r in ref['grads'].items():
        o = out['offs'][k]
        got = out['grad'][o:o + r.numel()].view_as(r)
        rep['g' + k] = rel_l2(got, r)
        assert rep['g' + k] < 1e-2 and cosine(got, r) > 0.9999, (k, rep)
    print('A =', A, (D, units, H, N, epm, masked, actname), {k: (round(v, 6) if isinstance(v, float) else v) for k, v in rep.items()})


def test_tc_train_refuses_tiles_that_straddle_arena_chunks():
    """several chunks whose row count is not a multiple of 128 would put one tile across two chunks: refused before any launch"""
    from rl_games_b200 import ops
    net, x = _train_inputs(3, 17, [128, 64, 32], 2, 400, 200, False, seed=5)
    assert _raises_unsupported(lambda: _run_train_step(ops, net, x, 1, 0))


@pytest.mark.parametrize('A,D,units,H,N,epm,masked', [(3, 17, [128, 64, 32], 1, 1000, 1000, True),
                                                      (6, 105, [256, 128, 64], 2, 384, 128, False),
                                                      (13, 60, [128, 64, 32], 2, 300, 128, True)])
def test_tc_scratch_buffers_need_no_initialisation(A, D, units, H, N, epm, masked):
    """every scratch buffer filled with 0xFF bytes (bf16 NaN) before the calls: finite results, byte-identical to the zero-filled run,
    and the padding the tile layout defines reads back as exactly 0"""
    from rl_games_b200 import ops
    net, x = _train_inputs(A, D, units, H, N, epm, masked, seed=77 + A)
    z = _run_train_step(ops, net, x, 1, 0)
    f = _run_train_step(ops, net, x, 1, 0xFF)
    M, n_tiles = x['M'], z['n_tiles']
    assert torch.isfinite(f['grad']).all() and torch.isfinite(f['stats']).all() and torch.isfinite(f['dls']).all()
    assert torch.equal(f['wpack'], z['wpack'])
    for k in ('mu', 'sigma', 'stats', 'dls', 'grad'):
        assert torch.equal(f[k], z[k]), k
    dh = decode_tiles(f['dhead'], n_tiles, 16)
    assert torch.equal(dh[:M, :A + 1], decode_tiles(z['dhead'], n_tiles, 16)[:M, :A + 1])
    assert float(dh[:M, A + 1:].abs().max()) == 0.0 if A < 15 else True      # d_head columns A+1..15 of live rows
    assert float(dh[M:].abs().max()) == 0.0 if M % 128 else True              # padded rows of the last tile
    for i, C in enumerate(units):
        got, ref = decode_tiles(f['act'][i], n_tiles, NATIVE[i])[:M], decode_tiles(z['act'][i], n_tiles, NATIVE[i])[:M]
        assert torch.equal(got, ref), i
        assert float(got[:, C:].abs().max()) == 0.0 if C < NATIVE[i] else True     # padded units
    for name, C, CN in (('delta2', units[1], NATIVE[1]), ('delta1', units[0], NATIVE[0])):
        got, ref = decode_tiles(f[name], n_tiles, CN)[:M], decode_tiles(z[name], n_tiles, CN)[:M]
        assert torch.equal(got, ref), name
        assert float(got[:, C:].abs().max()) == 0.0 if C < CN else True


# ================================================================================ C: fused rollout
def _rollout_reference(net, obs, nm, ns, noise, actname='elu'):
    W, b, Wh, bh, logstd = net
    act_fn = ACTS[actname][1]
    a = bf(torch.clamp((obs - nm) * (1.0 / ns), -5.0, 5.0))
    for w, bb in zip(W, b):
        a = bf(act_fn(mm(a, bf(w)) + bb))
    head = mm(a, bf(Wh)) + bh
    mu, val = head[:, 1:], head[:, 0]
    val = math.sqrt(4.0 + 1e-5) * torch.clamp(val, -5.0, 5.0) + 1.5
    return mu, val


def _rollout_outs(N, A, offset):
    """row-wide outputs; offset = 1 moves them one float off 16-byte alignment (the scalar store branch)"""
    def rw():
        return torch.full((N * A + offset,), float('nan'), device=DEV)[offset:].view(N, A)
    return dict(a=rw(), m=rw(), s=rw(), e=rw(), nl=torch.full((N,), float('nan'), device=DEV), v=torch.full((N,), float('nan'), device=DEV),
                d=torch.zeros(N, dtype=torch.uint8, device=DEV), valid=torch.full((N,), float('nan'), device=DEV))


@pytest.mark.parametrize('A,D,units,offset', [(1, 60, [256, 128, 64], 0), (3, 17, [128, 64, 32], 0), (6, 105, [256, 128, 64], 0),
                                              (8, 60, [256, 128, 64], 0), (8, 60, [256, 128, 64], 1), (12, 17, [128, 64, 32], 0),
                                              (12, 105, [256, 128, 64], 1), (15, 60, [256, 128, 64], 0)])
def test_tc_rollout_vs_faithful_reference(A, D, units, offset):
    from rl_games_b200 import ops
    N = 1000
    g = torch.Generator().manual_seed(31 * A + D)
    net = make_net(g, D, units, A)
    W, b, Wh, bh, logstd = net
    obs = (torch.randn(N, D, generator=g) * 2).to(DEV)
    nm, ns = (torch.randn(D, generator=g) * 0.3).to(DEV), (torch.rand(D, generator=g) + 0.7).to(DEV)
    noise = torch.randn(N, A, generator=g).to(DEV)
    vm, vv = torch.tensor([1.5], dtype=torch.float64, device=DEV), torch.tensor([4.0], dtype=torch.float64, device=DEV)
    lo, hi = torch.full((A,), -2.0, device=DEV), torch.full((A,), 4.0, device=DEV)
    dones_cur = (torch.rand(N, generator=g) < 0.3).to(torch.uint8).to(DEV)
    prev = (torch.rand(N, generator=g) < 0.3).float().to(DEV)
    wide = ops.tc_kind(D, units, A) == 2
    scratch = torch.full(((N + 127) // 128 * ops.tc_tile_bytes(D, units, A)[0],), 0xFF, dtype=torch.uint8, device=DEV) if wide else None
    wpack = torch.full((ops.tc_pack_bytes(D, units, A),), 0xFF, dtype=torch.uint8, device=DEV)
    ops.tc_pack_weights(W[0], W[1], W[2], Wh, D, units, A, wpack)
    t = _rollout_outs(N, A, offset)
    ops.tc_mlp_fwd_rollout(obs, D, nm, ns, wpack, b, bh, logstd, units, N, A, vm, vv, True, noise, 1, None, 0, t['a'], t['m'], t['s'],
                           t['nl'], t['v'], t['e'], True, lo, hi, dones_cur, t['d'], prev, t['valid'], l1_scratch=scratch)
    torch.cuda.synchronize()
    mu, val = _rollout_reference(net, obs, nm, ns, noise)
    rep = {'mu_rel_l2': rel_l2(t['m'], mu), 'mu_max_abs': float((t['m'] - mu).abs().max()), 'v_rel_l2': rel_l2(t['v'], val)}
    print('rollout A =', A, (D, units, offset), {k: round(v, 6) for k, v in rep.items()})
    assert rep['mu_rel_l2'] < 1e-3 and rep['v_rel_l2'] < 1e-3, rep
    torch.testing.assert_close(t['m'], mu, rtol=0, atol=6e-3)
    torch.testing.assert_close(t['v'], val, rtol=0, atol=1.2e-2)
    sigma = torch.exp(logstd).expand(N, A)
    torch.testing.assert_close(t['s'], sigma, rtol=1e-6, atol=0)
    # action = mu + sigma * eps on the kernel's own mu: only the final fp32 roundings differ
    torch.testing.assert_close(t['a'], t['m'] + t['s'] * noise, rtol=0, atol=1e-6)
    nlp = 0.5 * (noise.double() ** 2).sum(-1) + 0.5 * math.log(2 * math.pi) * A + logstd.double().sum()
    torch.testing.assert_close(t['nl'].double(), nlp, rtol=1e-5, atol=2e-5)
    torch.testing.assert_close(t['e'], torch.clamp(t['a'], -1.0, 1.0) * 3.0 + 1.0, rtol=0, atol=1e-6)
    assert torch.equal(t['d'], dones_cur) and torch.equal(t['valid'], 1.0 - prev)
    v2 = torch.full((N,), float('nan'), device=DEV)
    ops.tc_mlp_fwd_rollout(obs, D, nm, ns, wpack, b, bh, logstd, units, N, A, vm, vv, True, None, 0, None, 0, None, None, None, None, v2,
                           None, False, None, None, None, None, None, None, values_only=True, l1_scratch=scratch)
    torch.cuda.synchronize()
    assert torch.equal(v2, t['v'])


# ================================================================================ D: fp32 head kernels vs fp64 autograd
ACT_LAST = {0: (lambda z: z, lambda a: torch.ones_like(a)), 1: (F.elu, lambda a: torch.where(a > 0, torch.ones_like(a), a + 1.0)),
            2: (torch.relu, lambda a: (a > 0).to(a.dtype)), 3: (torch.tanh, lambda a: 1.0 - a * a)}
E_CLIP, CRITIC_COEF, BOUNDS_COEF, ENT_COEF = 0.2, 2.0, 0.001, 0.01


def _loss_cfg():
    from rl_games_b200.ops import LossCfg
    return LossCfg(E_CLIP, CRITIC_COEF, BOUNDS_COEF, 1, 1, 1, 1, 1)


def _head_loss_inputs(g, A, Hl, HR, act_last, masked, M=700, epm=250, N=300):
    """a_last [M, Hl] (output of the last layer's activation), arena rows in chunks of epm with stride N; with a mask, the second
    128-row block of the minibatch is masked out entirely"""
    a_last = ACT_LAST[act_last][0](torch.randn(M, Hl, generator=g))
    W = torch.randn(HR, Hl, generator=g) / math.sqrt(Hl)
    b = torch.randn(HR, generator=g) * 0.3
    W[A + 1:] *= 0.3            # raw-sigma rows (state-dependent sigma): sigma within about [0.5, 2]
    rows = (M + epm - 1) // epm * N
    actions, old_mu = torch.randn(rows, A, generator=g), torch.randn(rows, A, generator=g) * 0.5
    old_sigma = torch.rand(rows, A, generator=g) + 0.3
    old_v, ret, adv = torch.randn(rows, generator=g), torch.randn(rows, generator=g), torch.randn(rows, generator=g)
    m_ = torch.arange(M)
    ridx = (m_ // epm) * N + m_ % epm
    mask = None
    if masked:
        mask = (torch.rand(rows, generator=g) < 0.8).float()
        mask[ridx[128:256]] = 0.0
    return dict(a_last=a_last, W=W, b=b, actions=actions, old_mu=old_mu, old_sigma=old_sigma, old_v=old_v, ret=ret, adv=adv, mask=mask,
                ridx=ridx, M=M, epm=epm, N=N, A=A, Hl=Hl)


def _ppo_terms(x, head_value, mu, sg, ls, old_nlp):
    """per-row fp64 loss terms and the minibatch weights w = mask / sum(mask)"""
    r = x['ridx']
    nlp = O.neglogp_fn(x['actions'][r].double(), mu, sg, ls)
    a = O.actor_loss(old_nlp[r].double(), nlp, x['adv'][r].double(), True, E_CLIP, smooth=True)
    c = O.critic_loss(x['old_v'][r].double().unsqueeze(1), head_value, E_CLIP, x['ret'][r].double().unsqueeze(1), True).squeeze(1)
    e = (0.5 + 0.5 * math.log(2 * math.pi) + ls).sum(-1)
    bl = O.bound_loss(mu, BOUNDS_COEF)
    kl = O.policy_kl(mu.detach(), sg.detach(), x['old_mu'][r].double(), x['old_sigma'][r].double(), reduce=False)
    if x['mask'] is None:
        w = torch.full((x['M'],), 1.0 / x['M'], dtype=torch.float64)
    else:
        mk = x['mask'][r].double()
        w = mk / mk.sum().clamp(min=1.0)
    return nlp, a, c, e, bl, kl, w


def _sigma_of(head, A, logstd, sd, param, min_sigma, bounds):
    """(sigma, logstd) per row and action, fp64"""
    if sd:
        import _torch_ops_sd as S
        return S.apply_sigma(head[:, A + 1:], param, min_sigma, bounds)
    ls = logstd.expand(head.shape[0], A)
    return torch.exp(ls), ls


def _check_head_loss(ops, A, Hl, act_last, masked, sd=False, param='exp', min_sigma=0.0, bounds=None):
    g = torch.Generator().manual_seed(1000 * A + Hl + 10 * act_last + int(sd))
    HR = 1 + 2 * A if sd else A + 1
    x = _head_loss_inputs(g, A, Hl, HR, act_last, masked)
    logstd = torch.randn(A, generator=g) * 0.2
    # old neglogp = the current one + noise: probability ratios inside and around the clip range
    r = x['ridx']
    with torch.no_grad():
        h0 = x['a_last'].double() @ x['W'].double().t() + x['b'].double()
        sg0, ls0 = _sigma_of(h0, A, logstd.double(), sd, param, min_sigma, bounds)
        old_nlp = torch.randn(x['actions'].shape[0], generator=g) * 0.3 + 0.9 * A
        old_nlp[r] = (O.neglogp_fn(x['actions'][r].double(), h0[:, 1:A + 1], sg0, ls0) + torch.randn(x['M'], generator=g).double() * 0.3).float()
    # ---- fp64 autograd ----
    al = x['a_last'].double().requires_grad_(True)
    W, b = x['W'].double().requires_grad_(True), x['b'].double().requires_grad_(True)
    head = al @ W.t() + b
    head.retain_grad()
    value, mu = head[:, :1], head[:, 1:A + 1]
    lsp = None if sd else logstd.double().requires_grad_(True)
    sg, ls = _sigma_of(head, A, lsp, sd, param, min_sigma, bounds)
    nlp, a, c, e, bl, kl, w = _ppo_terms(x, value, mu, sg, ls, old_nlp)
    loss = (a * w).sum() + 0.5 * CRITIC_COEF * (c * w).sum() - ENT_COEF * (e * w).sum() + BOUNDS_COEF * (bl * w).sum()
    loss.backward()
    d_alast_ref = al.grad * ACT_LAST[act_last][1](al.detach())
    # ---- kernel ----
    M, epm, N = x['M'], x['epm'], x['N']
    d = lambda t: None if t is None else t.to(DEV)   # noqa: E731
    omu, osg = d(x['old_mu']).clone(), d(x['old_sigma']).clone()
    d_head, d_alast = torch.full((M, HR), float('nan'), device=DEV), torch.full((M, Hl), float('nan'), device=DEV)
    partials = torch.zeros(16, ops.loss_partial_stride(), dtype=torch.float64, device=DEV)
    mu_o, v_o, nlp_o = torch.empty(M, A, device=DEV), torch.empty(M, device=DEV), torch.empty(M, device=DEV)
    inv = None if x['mask'] is None else (1.0 / d(x['mask'])[d(x['ridx'])].sum().clamp(min=1.0)).reshape(1)
    ec = torch.tensor([ENT_COEF], device=DEV)
    common = (d(x['actions']), omu, osg, d(x['old_v']), d(x['ret']), d(old_nlp), d(x['adv']), d(x['mask']), epm, N, M, A, _loss_cfg(), inv,
              d_head, d_alast, act_last, partials)
    if sd:
        nb = ops.ppo_head_loss_sd(d(x['a_last']), d(x['W']), d(x['b']), ops.sigma_cfg(param, min_sigma, bounds), ec, *common,
                                  mu_out=mu_o, value_out=v_o, neglogp_out=nlp_o)
    else:
        nb = ops.ppo_head_loss(d(x['a_last']), d(x['W']), d(x['b']), d(logstd), *common, mu_out=mu_o, value_out=v_o, neglogp_out=nlp_o)
    stats, dls = torch.zeros(16, device=DEV), torch.full((A,), float('nan'), device=DEV)
    ops.ppo_loss_finalize(partials, nb, A, torch.zeros(1, device=DEV) if sd else ec, stats, dls)
    torch.cuda.synchronize()
    cpu = lambda t: t.cpu().double()   # noqa: E731
    torch.testing.assert_close(cpu(mu_o), mu.detach(), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(cpu(v_o), value.detach().squeeze(1), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(cpu(nlp_o), nlp.detach(), rtol=1e-5, atol=1e-4)
    # the fp32 neglogp sums A terms; its rounding reaches the gradients through exp(old_nlp - nlp) and the smooth clamp, so the
    # tolerances grow with A (measured at A = 31: 1.6e-6 absolute on d_head, 4.6e-6 on d_logstd)
    k = max(1.0, A / 8)
    torch.testing.assert_close(cpu(d_head), head.grad, rtol=2e-4 * k, atol=2e-7 * k * k)
    torch.testing.assert_close(cpu(d_alast), d_alast_ref, rtol=2e-4 * k, atol=2e-7 * k * k)
    if sd:
        assert torch.equal(dls.cpu(), torch.zeros(A))
    else:
        torch.testing.assert_close(cpu(dls), lsp.grad, rtol=2e-4 * k, atol=1e-6 * k * k)
    ref_stats = [(a * w).sum(), (c * w).sum(), (e * w).sum(), (bl * w).sum(), (kl * w).sum()]
    for k, rs in enumerate(ref_stats):
        assert float(stats[k]) == pytest.approx(float(rs), rel=1e-4, abs=1e-6), (k, float(stats[k]), float(rs))
    torch.testing.assert_close(cpu(omu)[r], mu.detach(), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(cpu(osg)[r], sg.detach(), rtol=1e-5, atol=1e-6)
    keep = torch.ones(x['actions'].shape[0], dtype=torch.bool)
    keep[r] = False
    assert torch.equal(omu.cpu()[keep], x['old_mu'][keep]) and torch.equal(osg.cpu()[keep], x['old_sigma'][keep])


def _loss_smem(A, Hl, sd):
    HR = 1 + 2 * A if sd else A + 1
    return 4 * (128 * (Hl + 1) + HR * Hl + HR + 4 * A + 4 * (8 + A))


def _sample_smem(A, Hl, sd):
    HR = 1 + 2 * A if sd else A + 1
    return 4 * (128 * (Hl + 1) + HR * Hl + HR + 2 * A)


def _first_hl_over(smem, A, sd):
    Hl = 1
    while smem(A, Hl, sd) <= 200 * 1024:
        Hl += 1
    return Hl


@pytest.mark.parametrize('A', [1, 4, 15, 17, 31])
@pytest.mark.parametrize('Hl', [24, 128, 256])
@pytest.mark.parametrize('act_last', [0, 1, 2, 3])
def test_ppo_head_loss_vs_fp64_autograd(A, Hl, act_last):
    from rl_games_b200 import ops
    _check_head_loss(ops, A, Hl, act_last, masked=act_last != 0)


@pytest.mark.parametrize('param,min_sigma,bounds', [('exp', 0.0, None), ('softplus', 0.2, None), ('exp', 0.1, (-1.0, 0.4))])
def test_ppo_head_loss_sd_vs_fp64_autograd_wide(param, min_sigma, bounds):
    from rl_games_b200 import ops
    _check_head_loss(ops, 15, 256, 1, True, sd=True, param=param, min_sigma=min_sigma, bounds=bounds)


@pytest.mark.parametrize('sd', [False, True])
def test_head_loss_largest_supported_width_and_refusal(sd):
    """the last head width that fits in 200 KB of shared memory runs and is right; the next one is refused with no launch"""
    from rl_games_b200 import ops
    A = 15 if sd else 31
    hl = _first_hl_over(_loss_smem, A, sd)
    _check_head_loss(ops, A, hl - 1, 1, True, sd=sd)
    HR = 1 + 2 * A if sd else A + 1
    M = 300
    a_last, W, b = torch.randn(M, hl, device=DEV), torch.randn(HR, hl, device=DEV), torch.zeros(HR, device=DEV)
    d_head = torch.full((M, HR), 7.0, device=DEV)
    f = lambda *s: torch.zeros(*s, device=DEV)   # noqa: E731
    rest = (f(M, A), f(M, A), torch.ones(M, A, device=DEV), f(M), f(M), f(M), f(M), None, M, M, M, A, _loss_cfg(), None, d_head, f(M, hl), 1,
            torch.zeros(16, ops.loss_partial_stride(), dtype=torch.float64, device=DEV))
    if sd:
        call = lambda: ops.ppo_head_loss_sd(a_last, W, b, ops.sigma_cfg('exp'), f(1), *rest)   # noqa: E731
    else:
        call = lambda: ops.ppo_head_loss(a_last, W, b, f(A), *rest)   # noqa: E731
    assert _raises_unsupported(call)
    torch.cuda.synchronize()
    assert torch.equal(d_head, torch.full((M, HR), 7.0, device=DEV))


def _check_sample(ops, A, Hl, sd=False, param='exp', min_sigma=0.0, bounds=None):
    g = torch.Generator().manual_seed(500 + 3 * A + Hl + int(sd))
    N = 515
    HR = 1 + 2 * A if sd else A + 1
    a_last = F.elu(torch.randn(N, Hl, generator=g))
    W, b = torch.randn(HR, Hl, generator=g) / math.sqrt(Hl), torch.randn(HR, generator=g) * 0.3
    logstd = torch.randn(A, generator=g) * 0.3
    noise = torch.randn(N, A, generator=g)
    head = a_last.double() @ W.double().t() + b.double()
    mu, val = head[:, 1:A + 1], head[:, 0]
    if sd:
        import _torch_ops_sd as S
        sg, ls = S.apply_sigma(head[:, A + 1:], param, min_sigma, bounds)
    else:
        ls = logstd.double().expand_as(mu)
        sg = torch.exp(ls)
    act = mu + sg * noise.double()
    nlp = O.neglogp_fn(act, mu, sg, ls)
    val = math.sqrt(4.0 + 1e-5) * val.clamp(-5, 5) + 1.5
    o = {k: torch.full((N, A), float('nan'), device=DEV) for k in ('a', 'm', 's', 'e')}
    nl, v = torch.full((N,), float('nan'), device=DEV), torch.full((N,), float('nan'), device=DEV)
    vm, vv = torch.tensor([1.5], dtype=torch.float64, device=DEV), torch.tensor([4.0], dtype=torch.float64, device=DEV)
    lo, hi = torch.full((A,), -2.0, device=DEV), torch.full((A,), 4.0, device=DEV)
    args = (vm, vv, True, noise.to(DEV), 0, None, 0, o['a'], o['m'], o['s'], nl, v, o['e'], True, lo, hi, None, None, None, None, N, A)
    if sd:
        ops.policy_head_sample_sd(a_last.to(DEV), W.to(DEV), b.to(DEV), ops.sigma_cfg(param, min_sigma, bounds), *args)
    else:
        ops.policy_head_sample(a_last.to(DEV), W.to(DEV), b.to(DEV), logstd.to(DEV), *args)
    torch.cuda.synchronize()
    cpu = lambda t: t.cpu().double()   # noqa: E731
    torch.testing.assert_close(cpu(o['m']), mu, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(cpu(v), val, rtol=1e-5, atol=2e-5)
    torch.testing.assert_close(cpu(o['s']), sg, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(cpu(o['a']), act, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(cpu(nl), nlp, rtol=1e-5, atol=1e-4)
    torch.testing.assert_close(cpu(o['e']), act.clamp(-1, 1) * 3.0 + 1.0, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize('A', [1, 4, 15, 17, 31])
@pytest.mark.parametrize('Hl', [24, 128, 256])
def test_policy_head_sample_vs_fp64(A, Hl):
    from rl_games_b200 import ops
    _check_sample(ops, A, Hl)


@pytest.mark.parametrize('param,min_sigma,bounds', [('exp', 0.0, None), ('softplus', 0.2, None), ('linear', 0.0, None)])
def test_policy_head_sample_sd_vs_fp64_wide(param, min_sigma, bounds):
    from rl_games_b200 import ops
    _check_sample(ops, 15, 256, sd=True, param=param, min_sigma=min_sigma, bounds=bounds)


@pytest.mark.parametrize('sd', [False, True])
def test_policy_head_sample_largest_supported_width_and_refusal(sd):
    from rl_games_b200 import ops
    A = 15 if sd else 31
    hl = _first_hl_over(_sample_smem, A, sd)
    _check_sample(ops, A, hl - 1, sd=sd)
    HR = 1 + 2 * A if sd else A + 1
    N = 300
    v = torch.full((N,), 7.0, device=DEV)
    f = lambda *s: torch.zeros(*s, device=DEV)   # noqa: E731
    rest = (None, None, False, f(N, A), 0, None, 0, f(N, A), f(N, A), f(N, A), f(N), v, None, False, None, None, None, None, None, None, N, A)
    if sd:
        call = lambda: ops.policy_head_sample_sd(f(N, hl), f(HR, hl), f(HR), ops.sigma_cfg('exp'), *rest)   # noqa: E731
    else:
        call = lambda: ops.policy_head_sample(f(N, hl), f(HR, hl), f(HR), f(A), *rest)   # noqa: E731
    assert _raises_unsupported(call)
    torch.cuda.synchronize()
    assert torch.equal(v, torch.full((N,), 7.0, device=DEV))


# ================================================================================ E: device RNG vs the host Philox
SEEDS = [0, 123456789, 0xDEADBEEFCAFE]
EPOCHS = [0, 3, (1 << 20) + 1]
STEPS = [0, 7, 65535]
# __logf / __sincosf against fp64 log / cos / sin.  The largest gap is at u = 1 - 2^-24, where r = sqrt(-2 ln u) = 3.5e-4 and one ulp of
# the intrinsic log moves r by ~6e-5; a slipped counter field is an O(1) difference.
RNG_ATOL = 2e-4


def _epoch_dev(ep):
    return torch.tensor([ep], dtype=torch.int64, device=DEV)


def _gauss_sampler_case(ops, kind, A, seed):
    """max |action(device eps) - action(host eps as tape)| over the epoch / step grid"""
    N, Hl = 700, 32
    g = torch.Generator().manual_seed(A + seed % 1000)
    if kind == 'tc':
        D, units = 60, [256, 128, 64]
        W, b, Wh, bh, logstd = make_net(g, D, units, A)
        obs, nm, ns = torch.randn(N, D, generator=g).to(DEV), torch.zeros(D, device=DEV), torch.ones(D, device=DEV)
        wpack = torch.empty(ops.tc_pack_bytes(D, units, A), dtype=torch.uint8, device=DEV)
        ops.tc_pack_weights(W[0], W[1], W[2], Wh, D, units, A, wpack)

        def launch(noise, ep, step, o):
            ops.tc_mlp_fwd_rollout(obs, D, nm, ns, wpack, b, bh, logstd, units, N, A, None, None, False, noise, seed, ep, step, o['a'], o['m'],
                                   o['s'], o['nl'], o['v'], None, False, None, None, None, None, None, None)
    else:
        sd = kind == 'sd'
        HR = 1 + 2 * A if sd else A + 1
        a_last = torch.randn(N, Hl, generator=g).to(DEV)
        W, b = (torch.randn(HR, Hl, generator=g) * 0.2).to(DEV), (torch.randn(HR, generator=g) * 0.3).to(DEV)
        logstd = (torch.randn(A, generator=g) * 0.3).to(DEV)

        def launch(noise, ep, step, o):
            rest = (None, None, False, noise, seed, ep, step, o['a'], o['m'], o['s'], o['nl'], o['v'], None, False, None, None, None, None,
                    None, None, N, A)
            if sd:
                ops.policy_head_sample_sd(a_last, W, b, ops.sigma_cfg('softplus', 0.1), *rest)
            else:
                ops.policy_head_sample(a_last, W, b, logstd, *rest)
    worst = 0.0
    for ep in EPOCHS:
        for step in STEPS:
            eps = torch.from_numpy(PR.gaussian_eps(seed, N, A, ep, step)).float().to(DEV)
            dev_o = {k: torch.full((N, A), float('nan'), device=DEV) for k in ('a', 'm', 's')}
            tape_o = {k: torch.full((N, A), float('nan'), device=DEV) for k in ('a', 'm', 's')}
            for o in (dev_o, tape_o):
                o['nl'], o['v'] = torch.empty(N, device=DEV), torch.empty(N, device=DEV)
            launch(None, _epoch_dev(ep), step, dev_o)
            launch(eps, None, 0, tape_o)
            torch.cuda.synchronize()
            assert torch.equal(dev_o['m'], tape_o['m']) and torch.equal(dev_o['s'], tape_o['s'])
            err = float((dev_o['a'] - tape_o['a']).abs().max())
            assert err < RNG_ATOL, (kind, A, seed, ep, step, err)
            worst = max(worst, err)
    return worst


@pytest.mark.parametrize('seed', SEEDS)
@pytest.mark.parametrize('kind,A', [('fp32', 1), ('fp32', 5), ('fp32', 31), ('sd', 15), ('tc', 3), ('tc', 15)])
def test_gaussian_samplers_draw_the_host_philox_normals(kind, A, seed):
    from rl_games_b200 import ops
    worst = _gauss_sampler_case(ops, kind, A, seed)
    print(f'device-RNG max |action error| {kind} A={A} seed={seed}: {worst:.3e}')


@pytest.mark.parametrize('head_sizes,masked', [(None, False), (None, True), ([3, 4, 2], True), ([2] * 8, False)])
def test_categorical_sampler_draws_the_host_philox_uniforms_bit_exact(head_sizes, masked):
    from rl_games_b200 import ops
    N = 1000
    sizes = head_sizes or [7]
    K, nh = sum(sizes), len(sizes)
    g = torch.Generator().manual_seed(K + nh)
    logits = (torch.randn(N, K, generator=g) * 2).to(DEV)
    value = torch.randn(N, 1, generator=g).to(DEV)
    amask = None
    if masked:
        m = torch.rand(N, K, generator=g) < 0.6
        off = 0
        for k in sizes:
            m[torch.arange(N), torch.randint(0, k, (N,), generator=g) + off] = True
            off += k
        amask = m.to(torch.uint8).to(DEV)
    for seed in SEEDS:
        for ep in EPOCHS:
            for step in STEPS:
                u = torch.from_numpy(PR.categorical_uniforms(seed, N, nh, ep, step)).float().contiguous().to(DEV)
                outs = []
                for tape, epd, st in ((None, _epoch_dev(ep), step), (u, None, 0)):
                    a = torch.full((N, nh), -1, dtype=torch.int64, device=DEV)
                    nl, v = torch.empty(N, device=DEV), torch.empty(N, device=DEV)
                    ops.categorical_sample(logits, K, K, value, 1, amask, tape, seed, epd, st, None, None, False, a, nl, v, None, None, None,
                                           None, N, head_sizes=head_sizes)
                    outs.append((a, nl))
                torch.cuda.synchronize()
                assert torch.equal(outs[0][0], outs[1][0]), (head_sizes, seed, ep, step)
                assert torch.equal(outs[0][1], outs[1][1])


@pytest.mark.parametrize('D', [60, 61])
def test_synth_env_draws_the_host_philox(D):
    from rl_games_b200 import ops
    N, A, max_len, p_done = 1000, 3, 50, 0.3
    g = torch.Generator().manual_seed(D)
    worst = 0.0
    for seed in SEEDS:
        for ep in EPOCHS:
            for step in (0, 7, 1023):       # the synthetic env's step field is 10 bits wide
                ep_t0 = torch.randint(0, max_len, (N,), generator=g, dtype=torch.int32)
                ep_t = ep_t0.to(DEV)
                obs, rew = torch.full((N, D), float('nan'), device=DEV), torch.empty(N, device=DEV)
                dones, tos = torch.full((N,), 7, dtype=torch.uint8, device=DEV), torch.full((N,), 7, dtype=torch.uint8, device=DEV)
                acts = torch.randn(N, A, generator=g).to(DEV)
                ops.synth_env_step(acts, obs, rew, dones, tos, ep_t, N, D, A, max_len, p_done, seed, _epoch_dev(ep), step)
                torch.cuda.synchronize()
                obs_h, u_done = PR.synth_env_draws(seed, N, D, ep, step)
                err = float((obs.cpu().double() - torch.from_numpy(obs_h)).abs().max())
                assert err < RNG_ATOL, (D, seed, ep, step, err)
                worst = max(worst, err)
                term = torch.from_numpy(u_done.astype(np.float32) <= np.float32(p_done))
                t = ep_t0 + 1
                to = t >= max_len
                done = to | term
                assert torch.equal(dones.cpu(), done.to(torch.uint8))
                assert torch.equal(tos.cpu(), (to & ~term).to(torch.uint8))
                assert torch.equal(ep_t.cpu(), torch.where(done, torch.zeros_like(t), t))
    print(f'device-RNG max |obs error| synth env D={D}: {worst:.3e}')


def test_fp32_and_fused_rollouts_draw_the_same_eps():
    """the same (seed, epoch, step) gives the same eps on both rollout paths (sigma = 1: action - mu is eps up to one rounding)"""
    from rl_games_b200 import ops
    N, A, D, units = 1000, 8, 60, [256, 128, 64]
    g = torch.Generator().manual_seed(8)
    W, b, Wh, bh, _ = make_net(g, D, units, A)
    logstd = torch.zeros(A, device=DEV)
    obs, nm, ns = torch.randn(N, D, generator=g).to(DEV), torch.zeros(D, device=DEV), torch.ones(D, device=DEV)
    wpack = torch.empty(ops.tc_pack_bytes(D, units, A), dtype=torch.uint8, device=DEV)
    ops.tc_pack_weights(W[0], W[1], W[2], Wh, D, units, A, wpack)
    a3 = torch.randn(N, units[2], generator=g).to(DEV)
    for seed, ep, step in ((5, 0, 0), (123456789, 3, 7), (0xDEADBEEFCAFE, (1 << 20) + 1, 65535)):
        o = [{k: torch.empty(N, A, device=DEV) for k in ('a', 'm', 's')} for _ in range(2)]
        for x in o:
            x['nl'], x['v'] = torch.empty(N, device=DEV), torch.empty(N, device=DEV)
        ops.policy_head_sample(a3, Wh, bh, logstd, None, None, False, None, seed, _epoch_dev(ep), step, o[0]['a'], o[0]['m'], o[0]['s'],
                               o[0]['nl'], o[0]['v'], None, False, None, None, None, None, None, None, N, A)
        ops.tc_mlp_fwd_rollout(obs, D, nm, ns, wpack, b, bh, logstd, units, N, A, None, None, False, None, seed, _epoch_dev(ep), step,
                               o[1]['a'], o[1]['m'], o[1]['s'], o[1]['nl'], o[1]['v'], None, False, None, None, None, None, None, None)
        torch.cuda.synchronize()
        e0, e1 = o[0]['a'] - o[0]['m'], o[1]['a'] - o[1]['m']
        torch.testing.assert_close(e0, e1, rtol=0, atol=2e-6)
        eps = torch.from_numpy(PR.gaussian_eps(seed, N, A, ep, step)).float().to(DEV)
        torch.testing.assert_close(e1, eps, rtol=0, atol=RNG_ATOL)


# ================================================================================ F: packed-weight refresh in the optimiser tail
@pytest.mark.parametrize('A,D', [(3, 17), (15, 105)])
def test_reduce_adam_pack_refresh_equals_fresh_pack(A, D):
    from rl_games_b200 import ops
    from rl_games_b200.ops import OptCfg
    units = [128, 64, 32]
    offs, P = flat_offsets(D, units, A)
    g = torch.Generator().manual_seed(A * D)
    params = (torch.randn(P, generator=g) * 0.1).to(DEV)

    def views(p):
        ins, Ws = D, []
        for i, u in enumerate(units):
            Ws.append(p[offs[f'W{i}']:offs[f'W{i}'] + u * ins].view(u, ins))
            ins = u
        Ws.append(p[offs['W_head']:offs['W_head'] + (A + 1) * ins].view(A + 1, ins))
        return Ws

    def pack(p, fill=0):
        w = torch.full((ops.tc_pack_bytes(D, units, A),), fill, dtype=torch.uint8, device=DEV)
        ops.tc_pack_weights(*views(p), D, units, A, w)
        return w
    wpack = pack(params, 0xFF)
    wpack0 = wpack.clone()
    tab = ops.tc_pack_table(D, units, A, offs)
    cfg = OptCfg(0.9, 0.999, 1e-8, 0.0, 1.0, 0.008, 1e-6, 1e-2, 1.5, 1.0, 1, 0)
    n_splits = 7
    exp_avg, exp_avg_sq, grads = torch.zeros(P, device=DEV), torch.zeros(P, device=DEV), torch.zeros(P, device=DEV)
    state = torch.tensor([3e-3, 0.0, 0.0, 0.0], dtype=torch.float64, device=DEV)
    counter, stats, kl = torch.zeros(1, dtype=torch.int32, device=DEV), torch.zeros(16, device=DEV), torch.zeros(1, device=DEV)
    nrm, bar = torch.zeros(148, dtype=torch.float64, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV)
    p_before = params.clone()
    for it in range(3):
        part = torch.full((n_splits, P), float('nan'), device=DEV)
        part[:, A:] = (torch.randn(n_splits, P - A, generator=g) * 0.01).to(DEV)
        lpart = (torch.rand(5, ops.loss_partial_stride(), generator=g, dtype=torch.float64) * 0.01).to(DEV)
        ops.reduce_adam(part, n_splits, P, lpart, 5, A, torch.tensor([0.0], device=DEV), stats, kl, grads, params, exp_avg, exp_avg_sq, P,
                        state, cfg, counter, nrm, bar, wpack=wpack, pack_table=tab)
        torch.cuda.synchronize()
        assert not torch.equal(params, p_before)
        assert torch.equal(wpack, pack(params)), it
    assert not torch.equal(wpack, wpack0)
