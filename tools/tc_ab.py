"""A/B of the fused tensor-core MLP kernels: the library of an earlier commit against the one in the tree, in ONE command on one GPU.

    python tools/tc_ab.py --build-base <commit>    # no GPU needed: that commit's csrc -> rl_games_b200/libb200rl_base.so (git-ignored)
    python tools/tc_ab.py [--out DIR]              # on the GPU

(a) runs the training forward + loss and the fused backward once per library on the same seeded c2 minibatch, and one rollout forward
    (plus a values_only call) at N = 16384 (one subprocess per library, B200RL_LIB_PATH selects it), and compares byte for byte the
    a1 / a2 / a3 / d_head / X tiles, the loss partials, the rewritten old_mu / old_sigma, the rollout outputs and delta1 / delta2, then
    the split-gradient array element by element;
(b) runs `bench.py --skip-e2e --skip-cpu --steps 20 --warmup 5` alternately base / new, three times each, and prints per run the
    value, ms_per_step, the tc_mlp_fwd_train / tc_mlp_fwd_rollout / tc_mlp_bwd kernel entries, the c5 value and the clocks.
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
CALLS = ('tc_mlp_fwd_train', 'tc_mlp_fwd_rollout', 'tc_mlp_bwd')
LIBS = {'base': os.path.join(PKG, 'libb200rl_base.so'), 'new': os.path.join(PKG, 'libb200rl.so')}


def build_base(commit):
    from rl_games_b200.csrc import build as b
    tmp = tempfile.mkdtemp(prefix='tc_ab_base_')
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
    """training forward + loss, fused backward and a rollout forward on seeded c2 inputs with the library B200RL_LIB_PATH names;
    writes their outputs to `out`"""
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
    nb = ops.tc_mlp_fwd_train(sl(obs), epm, N, D, nm, ns, wpack, b, bh, logstd, UNITS, M, A, sl(actions), sl(mu), sl(sg), sl(old_v),
                              sl(ret), sl(old_nlp), sl(adv), None, cfg, None, act, dhead, partials, xtile=xt)
    npart = ops.tc_mlp_bwd(sl(obs), epm, N, D, nm, ns, wpack, UNITS, M, A, act, dhead, delta2, delta1, part, P, offs, xtile=xt)
    # rollout forward: one launch at N rows (Philox sampling, value denormalisation, clipped env actions), then values_only
    ro = rnd(N, D).to(DEV)
    vm, vv = torch.tensor([1.5], dtype=torch.float64, device=DEV), torch.tensor([4.0], dtype=torch.float64, device=DEV)
    lo, hi = torch.full((A,), -1.0, device=DEV), torch.full((A,), 1.0, device=DEV)
    dones_cur = (torch.rand(N, generator=g) < 0.3).to(torch.uint8).to(DEV)
    r = {k: torch.zeros(N, A, device=DEV) for k in ('actions', 'mus', 'sigmas', 'env_actions')}
    r.update(neglogp=torch.zeros(N, device=DEV), values=torch.zeros(N, device=DEV), dones=torch.zeros(N, dtype=torch.uint8, device=DEV),
             values_only=torch.zeros(N, device=DEV))
    ops.tc_mlp_fwd_rollout(ro, D, nm, ns, wpack, b, bh, logstd, UNITS, N, A, vm, vv, True, None, 7, None, 3, r['actions'], r['mus'],
                           r['sigmas'], r['neglogp'], r['values'], r['env_actions'], True, lo, hi, dones_cur, r['dones'], None, None)
    ops.tc_mlp_fwd_rollout(ro, D, nm, ns, wpack, b, bh, logstd, UNITS, N, A, vm, vv, True, None, 0, None, 0, None, None, None, None,
                           r['values_only'], None, False, None, None, None, None, None, None, values_only=True)
    torch.cuda.synchronize()
    os.makedirs(out, exist_ok=True)
    fwd = dict(a1=act[0], a2=act[1], a3=act[2], dhead=dhead, xtile=xt, loss_partials=partials[:nb], old_mu=mu[0], old_sigma=sg[0],
               **{'rollout_' + k: v for k, v in r.items()})
    for k, v in fwd.items():
        np.save(os.path.join(out, k + '.npy'), v.cpu().numpy())
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
        sys.exit('tc_ab: no GPU')
    for k, p in LIBS.items():
        if not os.path.exists(p):
            sys.exit('tc_ab: %s library %s is missing (python tools/tc_ab.py --build-base <commit>)' % (k, p))
    out = sys.argv[sys.argv.index('--out') + 1] if '--out' in sys.argv else tempfile.mkdtemp(prefix='tc_ab_')
    print(subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip())
    # ---- (a) outputs ----
    for lib in LIBS:
        run(lib, [os.path.abspath(__file__), '--dump', os.path.join(out, lib)], check=True)
    ok = True
    exact = ('a1', 'a2', 'a3', 'dhead', 'xtile', 'loss_partials', 'old_mu', 'old_sigma', 'rollout_actions', 'rollout_mus', 'rollout_sigmas',
             'rollout_neglogp', 'rollout_values', 'rollout_env_actions', 'rollout_dones', 'rollout_values_only', 'delta1', 'delta2')
    for name in exact + ('part', 'grad'):
        x, y = np.load(os.path.join(out, 'base', name + '.npy')), np.load(os.path.join(out, 'new', name + '.npy'))
        if name in exact:      # compared as bytes: equal bit patterns (NaN included)
            nd = int((x.view(np.uint8) != y.view(np.uint8)).sum()) if x.shape == y.shape else -1
            print('%-20s %d bytes, %d differ' % (name, x.nbytes, nd))
            ok &= nd == 0
        else:
            rel = float(np.max(np.abs(x - y) / np.maximum(np.abs(x), 1e-6)))
            print('%-20s %d values, %d differ bitwise, max |diff| / max(|base|, 1e-6) = %.3g' % (name, x.size, int((x != y).sum()), rel))
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
            nan = {'ms': float('nan'), 'launches': 1, 'share': float('nan')}      # a call outside the printed top 12
            ks = [next((x for x in line['kernels'] if x['call'].endswith(c)), nan) for c in CALLS]
            rows[lib].append((line['value'], line['ms_per_step']) + tuple(k['ms'] / k['launches'] * 1e3 for k in ks) +
                             ((line.get('c5') or {}).get('value', float('nan')),))
            print('%-4s run %d: value %.4g env-steps/s, %.3f ms/step, c5 %.4g, clocks %s'
                  % (lib, rep, line['value'], line['ms_per_step'], rows[lib][-1][-1], json.dumps(line['clocks'])))
            for c, k in zip(CALLS, ks):
                print('       %-18s %.4f ms / %d launches = %.1f us (share %.3f)' % (c, k['ms'], k['launches'], k['ms'] / k['launches'] * 1e3, k['share']))
    for i, what in enumerate(('value', 'ms_per_step') + tuple(c + ' us/launch' for c in CALLS) + ('c5 value',)):
        b, n = [r[i] for r in rows['base']], [r[i] for r in rows['new']]
        print('%-30s base mean %.5g (spread %.3g)   new mean %.5g (spread %.3g)   new/base %.3f'
              % (what, sum(b) / 3, max(b) - min(b), sum(n) / 3, max(n) - min(n), sum(n) / sum(b)))
    sys.exit(0 if ok else 'tc_ab: outputs differ beyond fp32 last-bit size')


if __name__ == '__main__':
    if '--build-base' in sys.argv:
        build_base(sys.argv[sys.argv.index('--build-base') + 1])
    elif '--dump' in sys.argv:
        dump(sys.argv[sys.argv.index('--dump') + 1])
    else:
        main()
