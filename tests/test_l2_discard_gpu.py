"""The optimiser's reducer (reduce_adam_kernel) drops the lines of the split-gradient rows it has consumed from L2 (tc::l2_discard)
instead of letting them be written back.  A discard is only correct if nothing reads those bytes before their next write: the
backward kernel's flush of the next minibatch.  tests/libb200rl_l2poison.so (csrc/build.py::build_l2_poison) turns every discard
into a store of 0xFF bytes, NaN in fp32, so a read that comes too early poisons the result deterministically.  Each case runs once
with the product library and once with the poison library (one subprocess each, B200RL_LIB_PATH) and must give finite outputs that
are byte-identical between the two."""
import math
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBS = {'product': os.path.join(ROOT, 'rl_games_b200', 'libb200rl.so'), 'poison': os.path.join(ROOT, 'tests', 'libb200rl_l2poison.so')}
D, UNITS, A = 60, [256, 128, 64], 8


def _updates(M, n_updates, out):
    """n_updates minibatch updates of the c2 network on one M-row minibatch: training forward + loss, fused backward, fused
    reduce + clip + Adam + weight repack; parameters, Adam state, stats and the loss partials of every update go to `out`"""
    import torch
    from rl_games_b200 import ops
    from rl_games_b200.ops import LossCfg, OptCfg
    dev = 'cuda'
    g = torch.Generator().manual_seed(M)
    rnd = lambda *s: torch.randn(*s, generator=g)   # noqa: E731
    offs, o, ins = {}, A, D
    for i, u in enumerate(UNITS):
        offs['W%d' % i] = o; o += u * ins
        offs['b%d' % i] = o; o += u
        ins = u
    offs['W_head'] = o; o += (A + 1) * ins
    offs['b_head'] = o; o += A + 1
    P = o
    params = torch.zeros(P)
    ins = D
    for i, u in enumerate(UNITS):
        params[offs['W%d' % i]:offs['W%d' % i] + u * ins] = rnd(u * ins) / math.sqrt(ins)
        params[offs['b%d' % i]:offs['b%d' % i] + u] = 0.1 * rnd(u)
        ins = u
    params[offs['W_head']:offs['W_head'] + (A + 1) * ins] = rnd((A + 1) * ins) / math.sqrt(ins)
    params = params.to(dev)
    view = lambda k, n, r=None: params[offs[k]:offs[k] + n] if r is None else params[offs[k]:offs[k] + n].view(r, -1)   # noqa: E731
    Ws = [view('W%d' % i, u * c, u) for i, (u, c) in enumerate(zip(UNITS, [D] + UNITS[:-1]))]
    Wh = view('W_head', (A + 1) * UNITS[-1], A + 1)
    bs, bh, logstd = [view('b%d' % i, u) for i, u in enumerate(UNITS)], view('b_head', A + 1), params[:A]
    obs = rnd(M, D).to(dev); nm = (0.1 * rnd(D)).to(dev); ns = (1.0 + 0.1 * rnd(D).abs()).to(dev)
    actions = rnd(M, A).to(dev); mu = torch.zeros(M, A, device=dev); sg = torch.ones(M, A, device=dev)
    old_v, ret, adv = rnd(M).to(dev), rnd(M).to(dev), rnd(M).to(dev)
    old_nlp = torch.full((M,), 9.0, device=dev)
    lcfg = LossCfg(0.2, 2.0, 0.0, 1, 2, 1, 1, 1)
    ocfg = OptCfg(0.9, 0.999, 1e-8, 0.0, 1.0, 0.008, 1e-6, 1e-2, 1.5, 1.0, 1, 1)
    n_tiles = (M + 127) // 128
    tb = ops.tc_tile_bytes(D, UNITS, A)
    u8 = lambda n: torch.zeros(n, dtype=torch.uint8, device=dev)   # noqa: E731
    wpack = u8(ops.tc_pack_bytes(D, UNITS, A))
    ops.tc_pack_weights(*Ws, Wh, D, UNITS, A, wpack)
    tab = ops.tc_pack_table(D, UNITS, A, offs)
    act, dhead, delta2, delta1 = [u8(n_tiles * tb[i]) for i in range(3)], u8(n_tiles * tb[3]), u8(n_tiles * tb[1]), u8(n_tiles * tb[0])
    xt = u8(n_tiles * ops.tc_xtile_bytes(D, UNITS, A))
    lpart = torch.zeros(ops.NUM_SMS, ops.loss_partial_stride(), dtype=torch.float64, device=dev)
    stride = (P + 31) // 32 * 32
    part = torch.zeros(ops.NUM_SMS, stride, device=dev)
    m1, m2, grads = torch.zeros(P, device=dev), torch.zeros(P, device=dev), torch.zeros(P, device=dev)
    state = torch.tensor([3e-4, 0.0, 0.0, 0.0], dtype=torch.float64, device=dev)
    counter, kl = torch.zeros(1, dtype=torch.int32, device=dev), torch.zeros(1, device=dev)
    nrm, bar = torch.zeros(ops.NUM_SMS, dtype=torch.float64, device=dev), torch.zeros(1, dtype=torch.int64, device=dev)
    ec = torch.tensor([0.001], device=dev)
    res = {}
    for u in range(n_updates):
        stats = torch.zeros(16, device=dev)
        nb = ops.tc_mlp_fwd_train(obs, M, 0, D, nm, ns, wpack, bs, bh, logstd, UNITS, M, A, actions, mu, sg, old_v, ret, old_nlp, adv,
                                  None, lcfg, None, act, dhead, lpart, xtile=xt)
        npart = ops.tc_mlp_bwd(obs, M, 0, D, nm, ns, wpack, UNITS, M, A, act, dhead, delta2, delta1, part, stride, offs, xtile=xt)
        ops.reduce_adam(part, npart, stride, lpart, nb, A, ec, stats, kl, grads, params, m1, m2, P, state, ocfg, counter, nrm, bar,
                        wpack=wpack, pack_table=tab)
        res['stats%d' % u] = stats
        res['loss_partials%d' % u] = lpart[:nb].clone()
        res['grads%d' % u] = grads.clone()
    res.update(params=params, exp_avg=m1, exp_avg_sq=m2, state=state, wpack=wpack, old_mu=mu, old_sigma=sg)
    torch.cuda.synchronize()
    for k, v in res.items():
        np.save(os.path.join(out, k + '.npy'), v.cpu().numpy())


def _epochs(out):
    """three whole `train_epoch`s of a c2-geometry agent (mixed precision: the fused tensor-core update) on a device tape env"""
    import torch
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    from oracle import ppo_oracle as O
    from test_agent_gpu import TapeEnvGPU, make_agent
    N, H, mb = 1024, 16, 4096
    obs_tape, done_tape, tout_tape = O.make_tapes(3 * H + 1, N, D, seed=5)
    params = O.init_params(D, UNITS, A, seed=6)
    agent = make_agent({'mini_epochs': 2, 'mixed_precision': True}, N, H, D, A, UNITS, mb, TapeEnvGPU(obs_tape, done_tape, tout_tape, A), params)
    assert agent.use_tc
    g = torch.Generator().manual_seed(8)
    stats = []
    for _ in range(3):
        agent.epoch_num += 1
        agent.train_epoch(noise=torch.randn(H, N, A, generator=g).to('cuda'))
        stats.append(agent.last_stats.clone())
    torch.cuda.synchronize()
    np.save(os.path.join(out, 'stats.npy'), torch.stack(stats).cpu().numpy())
    for k, v in agent.model.state_dict().items():
        np.save(os.path.join(out, 'sd_' + k + '.npy'), v.detach().cpu().numpy())


def _run_both(case):
    import torch
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    if not os.path.exists(LIBS['poison']):
        from rl_games_b200.csrc import build as _b
        _b.build_l2_poison(verbose=False)
    tmp = tempfile.mkdtemp(prefix='l2_discard_')
    for name, lib in LIBS.items():
        r = subprocess.run([sys.executable, os.path.abspath(__file__)] + case + [os.path.join(tmp, name)], cwd=ROOT, text=True,
                           capture_output=True, env=dict(os.environ, B200RL_LIB_PATH=lib))
        assert r.returncode == 0, (name, r.stdout[-3000:], r.stderr[-3000:])
    names = sorted(os.listdir(os.path.join(tmp, 'product')))
    assert names and names == sorted(os.listdir(os.path.join(tmp, 'poison')))
    for f in names:
        x, y = np.load(os.path.join(tmp, 'product', f)), np.load(os.path.join(tmp, 'poison', f))
        if x.dtype.kind == 'f':
            assert np.isfinite(y).all(), f
        assert x.shape == y.shape and x.tobytes() == y.tobytes(), f


# c2 minibatch (256 tiles: 128 CTAs x 2), a partial last tile, fewer tiles than CTAs (1 tile per CTA), 3 tiles per CTA
@pytest.mark.gpu
@pytest.mark.parametrize('M', [32768, 1000, 5120, 3 * 132 * 128])
def test_l2_discard_updates_match_product(M):
    _run_both(['--updates', str(M)])


@pytest.mark.gpu
def test_l2_discard_train_epochs_match_product():
    _run_both(['--epochs'])


if __name__ == '__main__':
    sys.path.insert(0, ROOT)
    os.makedirs(sys.argv[-1], exist_ok=True)
    if sys.argv[1] == '--updates':
        _updates(int(sys.argv[2]), 4, sys.argv[-1])
    else:
        _epochs(sys.argv[-1])
