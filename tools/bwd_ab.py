"""A/B of the fused MLP backward kernel: the library of an earlier commit against the one in the tree, in ONE command on one GPU.

    python tools/bwd_ab.py --build-base <commit>    # no GPU needed: that commit's csrc -> rl_games_b200/libb200rl_base.so (git-ignored)
    python tools/bwd_ab.py [--out DIR]              # on the GPU

(a) runs the fused forward + backward once per library on the same seeded c2 minibatch (one subprocess per library, B200RL_LIB_PATH
    selects it) and compares delta1, delta2 and the column-summed split-gradient array element by element;
(b) runs `bench.py --skip-e2e --skip-cpu --steps 20 --warmup 5` alternately base / new, three times each, and prints per run the
    value, ms_per_step, the tc_mlp_bwd kernel entry, the c5 value and the clocks.
Fails without a GPU."""
import json
import math
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PKG = os.path.join(ROOT, 'rl_games_b200')
LIBS = {'base': os.path.join(PKG, 'libb200rl_base.so'), 'new': os.path.join(PKG, 'libb200rl.so')}


def build_base(commit):
    from rl_games_b200.csrc import build as b
    tmp = tempfile.mkdtemp(prefix='bwd_ab_base_')
    files = subprocess.run(['git', '-C', ROOT, 'ls-tree', '-r', '--name-only', commit, 'rl_games_b200/csrc', 'include'],
                           capture_output=True, text=True, check=True).stdout.split()
    for f in files:
        if f.endswith(('.cu', '.cuh', '.h')):
            os.makedirs(os.path.dirname(os.path.join(tmp, f)), exist_ok=True)
            with open(os.path.join(tmp, f), 'w') as fh:
                fh.write(subprocess.run(['git', '-C', ROOT, 'show', '%s:%s' % (commit, f)], capture_output=True, text=True, check=True).stdout)
    objs = []
    for f in sorted(x for x in files if x.endswith('.cu')):
        objs.append(os.path.join(tmp, os.path.basename(f)[:-3] + '.o'))
        subprocess.check_call([b.NVCC] + b.FLAGS + ['-c', os.path.join(tmp, f), '-o', objs[-1]])
    subprocess.check_call([b.NVCC, '-shared', '-gencode', 'arch=compute_90a,code=sm_90a', '-o', LIBS['base']] + objs + ['-lcuda'])
    print(LIBS['base'])


def dump(out):
    """fused forward + backward on a seeded c2 minibatch with the library B200RL_LIB_PATH names; writes delta1, delta2, grad to `out`"""
    import numpy as np
    import torch
    from rl_games_b200 import ops
    from rl_games_b200.ops import LossCfg
    DEV = 'cuda'
    D, UNITS, A = 60, [256, 128, 64], 8
    H, N, epm = 16, 16384, 2048
    M = H * epm
    g = torch.Generator().manual_seed(1)
    rnd = lambda *s: torch.randn(*s, generator=g)   # noqa: E731
    ins, W, b = D, [], []
    for u in UNITS:
        W.append((rnd(u, ins) / math.sqrt(ins)).to(DEV)); b.append((0.1 * rnd(u)).to(DEV)); ins = u
    Wh = (rnd(A + 1, ins) / math.sqrt(ins)).to(DEV); bh = torch.zeros(A + 1, device=DEV)
    logstd = torch.zeros(A, device=DEV)
    obs = rnd(H, N, D).to(DEV); nm = torch.zeros(D, device=DEV); ns = torch.ones(D, device=DEV)
    actions = rnd(H, N, A).to(DEV); mu = torch.zeros(H, N, A, device=DEV); sg = torch.ones(H, N, A, device=DEV)
    old_v = rnd(H, N).to(DEV); ret = rnd(H, N).to(DEV)
    old_nlp = torch.full((H, N), 9.0, device=DEV); adv = rnd(H, N).to(DEV)
    cfg = LossCfg(0.2, 2.0, 0.0, 1, 2, 1, 1, 1)
    n_tiles = M // 128
    tb = ops.tc_tile_bytes(D, UNITS, A)
    wpack = torch.zeros(ops.tc_pack_bytes(D, UNITS, A), dtype=torch.uint8, device=DEV)
    ops.tc_pack_weights(W[0], W[1], W[2], Wh, D, UNITS, A, wpack)
    act = [torch.zeros(n_tiles * tb[i], dtype=torch.uint8, device=DEV) for i in range(3)]
    dhead = torch.zeros(n_tiles * tb[3], dtype=torch.uint8, device=DEV)
    partials = torch.zeros(132, ops.loss_partial_stride(), dtype=torch.float64, device=DEV)
    delta2 = torch.zeros(n_tiles * tb[1], dtype=torch.uint8, device=DEV); delta1 = torch.zeros(n_tiles * tb[0], dtype=torch.uint8, device=DEV)
    P = A + sum(w.numel() + x.numel() for w, x in zip(W, b)) + Wh.numel() + bh.numel()
    offs, o, ins = {}, A, D
    for i, u in enumerate(UNITS):
        offs['W%d' % i] = o; o += u * ins
        offs['b%d' % i] = o; o += u
        ins = u
    offs['W_head'] = o; o += (A + 1) * ins
    offs['b_head'] = o
    part = torch.zeros(132, P, device=DEV)
    xt = torch.zeros(n_tiles * ops.tc_xtile_bytes(D, UNITS, A), dtype=torch.uint8, device=DEV)
    sl = lambda t: t[0]   # noqa: E731
    ops.tc_mlp_fwd_train(sl(obs), epm, N, D, nm, ns, wpack, b, bh, logstd, UNITS, M, A, sl(actions), sl(mu), sl(sg), sl(old_v),
                         sl(ret), sl(old_nlp), sl(adv), None, cfg, None, act, dhead, partials, xtile=xt)
    npart = ops.tc_mlp_bwd(sl(obs), epm, N, D, nm, ns, wpack, UNITS, M, A, act, dhead, delta2, delta1, part, P, offs, xtile=xt)
    torch.cuda.synchronize()
    os.makedirs(out, exist_ok=True)
    np.save(os.path.join(out, 'delta1.npy'), delta1.cpu().numpy())
    np.save(os.path.join(out, 'delta2.npy'), delta2.cpu().numpy())
    # rows summed in index order in float64: the same sum for both libraries when the rows are equal
    np.save(os.path.join(out, 'grad.npy'), part[:npart, A:].double().sum(0).cpu().numpy())
    np.save(os.path.join(out, 'part.npy'), part[:npart, A:].cpu().numpy())


def run(lib, args, **kw):
    env = dict(os.environ, B200RL_LIB_PATH=LIBS[lib])
    return subprocess.run([sys.executable] + args, env=env, cwd=ROOT, text=True, **kw)


def main():
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit('bwd_ab: no GPU')
    for k, p in LIBS.items():
        if not os.path.exists(p):
            sys.exit('bwd_ab: %s library %s is missing (python tools/bwd_ab.py --build-base <commit>)' % (k, p))
    out = sys.argv[sys.argv.index('--out') + 1] if '--out' in sys.argv else tempfile.mkdtemp(prefix='bwd_ab_')
    print(subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip())
    # ---- (a) outputs ----
    for lib in LIBS:
        run(lib, [os.path.abspath(__file__), '--dump', os.path.join(out, lib)], check=True)
    ok = True
    for name in ('delta1', 'delta2', 'part', 'grad'):
        x, y = np.load(os.path.join(out, 'base', name + '.npy')), np.load(os.path.join(out, 'new', name + '.npy'))
        if name.startswith('delta'):
            nd = int((x != y).sum())
            print('%-7s %d bytes, %d differ' % (name, x.size, nd))
            ok &= nd == 0
        else:
            rel = float(np.max(np.abs(x - y) / np.maximum(np.abs(x), 1e-6)))
            print('%-7s %d values, %d differ bitwise, max |diff| / max(|base|, 1e-6) = %.3g' % (name, x.size, int((x != y).sum()), rel))
            ok &= rel <= 1e-6
    # ---- (b) benchmark, alternating ----
    rows = {'base': [], 'new': []}
    for rep in range(3):
        for lib in ('base', 'new'):
            r = run(lib, [os.path.join(ROOT, 'bench.py'), '--gpus', '1', '--skip-e2e', '--skip-cpu', '--steps', '20', '--warmup', '5'],
                    capture_output=True)
            line = next((json.loads(ln) for ln in reversed(r.stdout.splitlines()) if ln.startswith('{') and '"metric"' in ln), None)
            if r.returncode or line is None:
                sys.exit('bwd_ab: bench.py failed for %s:\n%s\n%s' % (lib, r.stdout[-2000:], r.stderr[-2000:]))
            k = next(x for x in line['kernels'] if x['call'].endswith('tc_mlp_bwd'))
            rows[lib].append((line['value'], line['ms_per_step'], k['ms'] / k['launches'] * 1e3, (line.get('c5') or {}).get('value', float('nan'))))
            print('%-4s run %d: value %.4g env-steps/s, %.3f ms/step, tc_mlp_bwd %.4f ms / %d launches = %.1f us (share %.3f), c5 %.4g, clocks %s'
                  % (lib, rep, line['value'], line['ms_per_step'], k['ms'], k['launches'], k['ms'] / k['launches'] * 1e3, k['share'],
                     rows[lib][-1][3], json.dumps(line['clocks'])))
    for i, what in enumerate(('value', 'ms_per_step', 'tc_mlp_bwd us/launch', 'c5 value')):
        b, n = [r[i] for r in rows['base']], [r[i] for r in rows['new']]
        print('%-22s base mean %.5g (spread %.3g)   new mean %.5g (spread %.3g)   new/base %.3f'
              % (what, sum(b) / 3, max(b) - min(b), sum(n) / 3, max(n) - min(n), sum(n) / sum(b)))
    sys.exit(0 if ok else 'bwd_ab: outputs differ beyond fp32 last-bit size')


if __name__ == '__main__':
    if '--build-base' in sys.argv:
        build_base(sys.argv[sys.argv.index('--build-base') + 1])
    elif '--dump' in sys.argv:
        dump(sys.argv[sys.argv.index('--dump') + 1])
    else:
        main()
