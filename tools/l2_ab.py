"""A/B of the L2 cache policy of the minibatch update (evict_first / evict_last hints, split-gradient lines discarded by the reducer):
the library of an earlier commit against the one in the tree, in ONE command on one GPU.

    python tools/l2_ab.py --bytes                  # no GPU needed: the update's global-memory traffic from the c2 shapes (an estimate)
    python tools/tc_ab.py --build-base <commit>    # no GPU needed: that commit's csrc -> rl_games_b200/libb200rl_base.so (git-ignored)
    python tools/l2_ab.py [--rounds 6] [--out DIR] # on the GPU

(a) `bench.py --dump-outputs` once per library: every array (stats, parameters, experience) must be equal bit for bit;
(b) the update's kernels alone at the c2 minibatch shape: the training forward, the fused backward and reduce_adam, each timed with
    CUDA events around 200 launches, and the three in sequence (one subprocess per library, alternating, B200RL_LIB_PATH);
(c) `bench.py --skip-e2e --skip-cpu --steps 20 --warmup 5` alternately base / new, --rounds times each: value, ms_per_step, c5.
The card's name, power limit and clocks are read in the same call.  Fails without a GPU."""
import json
import math
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from tc_ab import LIBS, run   # noqa: E402

D, UNITS, A = 60, [256, 128, 64], 8
M = 32768          # c2 minibatch: 16384 envs x 16 steps / 8 minibatches


def bytes_table():
    """MB moved by one c2 minibatch update, from the tile shapes of mlp_tc.cu (bf16 128-row INTERLEAVE tiles) and the split rows"""
    t = M // 128
    x, a1, a2, a3, dh = 128 * 64 * 2, 128 * UNITS[0] * 2, 128 * UNITS[1] * 2, 128 * UNITS[2] * 2, 128 * 16 * 2
    P = A + sum(u * c + u for u, c in zip(UNITS, [D] + UNITS[:-1])) + (A + 1) * UNITS[-1] + A + 1
    splits = (t + (t + 131) // 132 - 1) // ((t + 131) // 132)
    rows = [('forward: obs read', M * D * 4), ('forward: arena rows (read + old_mu / old_sigma write)', M * (4 * 4 + 3 * A * 4)),
            ('forward: writes xt, a1, a2, a3, d_head', t * (x + a1 + a2 + a3 + dh)),
            ('backward phase 1: reads d_head, a3, a2, a1', t * (dh + a3 + a2 + a1)), ('backward phase 1: writes d2, d1', t * (a2 + a1)),
            ('backward phase 2: reads d2, d1, a1, xt', t * (a2 + a1 + a1 + x)),
            ('split partials: flush write (%d rows x %d params)' % (splits, P), splits * P * 4), ('split partials: reduce_adam read', splits * P * 4)]
    tot = 0
    print('c2 minibatch update, %d rows (%d tiles): bytes from the shapes, NOT measured' % (M, t))
    for name, b in rows:
        print('  %-58s %6.1f MB' % (name, b / 1e6))
        tot += b
    print('  %-58s %6.1f MB  = %.0f us at the data-sheet 3.35 TB/s' % ('total', tot / 1e6, tot / 3.35e12 * 1e6))


def time_kernels(out):
    """the update's three kernels alone on a seeded c2 minibatch with the library B200RL_LIB_PATH names: us per launch"""
    import torch
    from rl_games_b200 import ops
    from rl_games_b200.ops import LossCfg, OptCfg
    dev = 'cuda'
    g = torch.Generator().manual_seed(1)
    rnd = lambda *s: torch.randn(*s, generator=g)   # noqa: E731
    offs, o, ins = {}, A, D
    for i, u in enumerate(UNITS):
        offs['W%d' % i] = o; o += u * ins
        offs['b%d' % i] = o; o += u
        ins = u
    offs['W_head'] = o; o += (A + 1) * ins
    offs['b_head'] = o; o += A + 1
    P = o
    params = (0.05 * rnd(P)).to(dev)
    Ws = [params[offs['W%d' % i]:offs['W%d' % i] + u * c].view(u, c) for i, (u, c) in enumerate(zip(UNITS, [D] + UNITS[:-1]))]
    Wh = params[offs['W_head']:offs['W_head'] + (A + 1) * UNITS[-1]].view(A + 1, -1)
    bs, bh = [params[offs['b%d' % i]:offs['b%d' % i] + u] for i, u in enumerate(UNITS)], params[offs['b_head']:offs['b_head'] + A + 1]
    obs = rnd(M, D).to(dev); nm = torch.zeros(D, device=dev); ns = torch.ones(D, device=dev)
    actions = rnd(M, A).to(dev); mu = torch.zeros(M, A, device=dev); sg = torch.ones(M, A, device=dev)
    old_v, ret, adv = rnd(M).to(dev), rnd(M).to(dev), rnd(M).to(dev)
    old_nlp = torch.full((M,), 9.0, device=dev)
    lcfg = LossCfg(0.2, 2.0, 0.0, 1, 2, 1, 1, 1)
    ocfg = OptCfg(0.9, 0.999, 1e-8, 0.0, 1.0, 0.008, 1e-6, 1e-2, 1.5, 1.0, 1, 1)
    t = M // 128
    tb = ops.tc_tile_bytes(D, UNITS, A)
    u8 = lambda n: torch.zeros(n, dtype=torch.uint8, device=dev)   # noqa: E731
    wpack = u8(ops.tc_pack_bytes(D, UNITS, A))
    ops.tc_pack_weights(*Ws, Wh, D, UNITS, A, wpack)
    tab = ops.tc_pack_table(D, UNITS, A, offs)
    act, dhead, d2, d1 = [u8(t * tb[i]) for i in range(3)], u8(t * tb[3]), u8(t * tb[1]), u8(t * tb[0])
    xt = u8(t * ops.tc_xtile_bytes(D, UNITS, A))
    lpart = torch.zeros(ops.NUM_SMS, ops.loss_partial_stride(), dtype=torch.float64, device=dev)
    part = torch.zeros(ops.NUM_SMS, (P + 3) // 4 * 4, device=dev)     # the agent's row stride
    m1, m2, grads = torch.zeros(P, device=dev), torch.zeros(P, device=dev), torch.zeros(P, device=dev)
    state = torch.tensor([3e-4, 0.0, 0.0, 0.0], dtype=torch.float64, device=dev)
    counter, kl, stats = torch.zeros(1, dtype=torch.int32, device=dev), torch.zeros(1, device=dev), torch.zeros(16, device=dev)
    nrm, bar = torch.zeros(ops.NUM_SMS, dtype=torch.float64, device=dev), torch.zeros(1, dtype=torch.int64, device=dev)
    ec = torch.tensor([0.0], device=dev)
    nb = [0]

    def fwd():
        nb[0] = ops.tc_mlp_fwd_train(obs, M, 0, D, nm, ns, wpack, bs, bh, params[:A], UNITS, M, A, actions, mu, sg, old_v, ret, old_nlp,
                                     adv, None, lcfg, None, act, dhead, lpart, xtile=xt)

    def bwd():
        nb.append(ops.tc_mlp_bwd(obs, M, 0, D, nm, ns, wpack, UNITS, M, A, act, dhead, d2, d1, part, part.shape[1], offs, xtile=xt))

    def radam():
        ops.reduce_adam(part, nb[-1], part.shape[1], lpart, nb[0], A, ec, stats, kl, grads, params, m1, m2, P, state, ocfg, counter, nrm,
                        bar, wpack=wpack, pack_table=tab)

    def update():
        fwd(); bwd(); radam()
    res = {}
    for name, fn in (('update', update), ('fwd_train', fwd), ('bwd', bwd), ('reduce_adam', radam), ('update_again', update)):
        for _ in range(20):
            fn()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(200):
            fn()
        e.record()
        torch.cuda.synchronize()
        res[name] = s.elapsed_time(e) / 200 * 1e3
        del nb[1:]
    with open(out, 'w') as f:
        json.dump(res, f)


def smi():
    return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip()


def main():
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit('l2_ab: no GPU')
    for k, p in LIBS.items():
        if not os.path.exists(p):
            sys.exit('l2_ab: %s library %s is missing (python tools/tc_ab.py --build-base <commit>)' % (k, p))
    rounds = int(sys.argv[sys.argv.index('--rounds') + 1]) if '--rounds' in sys.argv else 6
    out = sys.argv[sys.argv.index('--out') + 1] if '--out' in sys.argv else tempfile.mkdtemp(prefix='l2_ab_')
    print('card (name, power limit, SM clock, max SM clock):', smi())
    bytes_table()
    # ---- (a) outputs of the benchmarked workload ----
    ok = True
    for lib in LIBS:
        r = run(lib, [os.path.join(ROOT, 'bench.py'), '--gpus', '1', '--skip-e2e', '--skip-cpu', '--steps', '3', '--warmup', '1',
                      '--dump-outputs', os.path.join(out, 'dump_' + lib)], capture_output=True)
        if r.returncode:
            sys.exit('l2_ab: bench.py --dump-outputs failed for %s:\n%s\n%s' % (lib, r.stdout[-2000:], r.stderr[-2000:]))
    names = sorted(f for f in os.listdir(os.path.join(out, 'dump_base')) if f.endswith('.npy'))
    nd = [f for f in names if not np.array_equal(np.load(os.path.join(out, 'dump_base', f)), np.load(os.path.join(out, 'dump_new', f)),
                                                 equal_nan=True)]
    print('bench.py --dump-outputs: %d arrays, %d differ %s' % (len(names), len(nd), nd[:10]))
    ok &= not nd and bool(names)
    # ---- (b) kernels alone, alternating ----
    kt = {'base': [], 'new': []}
    for rep in range(3):
        for lib in ('base', 'new'):
            f = os.path.join(out, 'k_%s_%d.json' % (lib, rep))
            run(lib, [os.path.abspath(__file__), '--time', f], check=True)
            kt[lib].append(json.load(open(f)))
    for k in kt['base'][0]:
        b, n = [r[k] for r in kt['base']], [r[k] for r in kt['new']]
        print('%-14s us/launch  base %s  new %s   new/base %.3f' % (k, ' '.join('%.1f' % v for v in b), ' '.join('%.1f' % v for v in n),
                                                              sum(n) / sum(b)))
    # ---- (c) benchmark, alternating ----
    rows = {'base': [], 'new': []}
    for rep in range(rounds):
        for lib in ('base', 'new'):
            r = run(lib, [os.path.join(ROOT, 'bench.py'), '--gpus', '1', '--skip-e2e', '--skip-cpu', '--steps', '20', '--warmup', '5'],
                    capture_output=True)
            line = next((json.loads(ln) for ln in reversed(r.stdout.splitlines()) if ln.startswith('{') and '"metric"' in ln), None)
            if r.returncode or line is None:
                sys.exit('l2_ab: bench.py failed for %s:\n%s\n%s' % (lib, r.stdout[-2000:], r.stderr[-2000:]))
            rows[lib].append((line['value'], line['ms_per_step'], (line.get('c5') or {}).get('value', float('nan'))))
            print('%-4s round %d: value %.4g env-steps/s, %.3f ms/step, c5 %.4g, clocks %s'
                  % (lib, rep, line['value'], line['ms_per_step'], rows[lib][-1][2], json.dumps(line.get('clocks'))))
    wins = sum(n[1] < b[1] for b, n in zip(rows['base'], rows['new']))
    for i, what in enumerate(('value', 'ms_per_step', 'c5 value')):
        b, n = [r[i] for r in rows['base']], [r[i] for r in rows['new']]
        print('%-12s base mean %.5g (spread %.3g)   new mean %.5g (spread %.3g)   new/base %.3f'
              % (what, sum(b) / len(b), max(b) - min(b), sum(n) / len(n), max(n) - min(n), sum(n) / sum(b)))
    print('rounds with a lower c2 ms_per_step: %d of %d' % (wins, rounds))
    print('card after the runs:', smi())
    sys.exit(0 if ok else 'l2_ab: outputs differ')


if __name__ == '__main__':
    if '--bytes' in sys.argv:
        bytes_table()
    elif '--time' in sys.argv:
        time_kernels(sys.argv[sys.argv.index('--time') + 1])
    else:
        main()
