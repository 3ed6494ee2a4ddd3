"""Stage-by-stage clock64() timeline of the fused tensor-core forward+loss kernel (CTA 0), c2 minibatch shape.

    python tools/tc_stage_timing.py --build      # here (no GPU): builds rl_games_b200/libb200rl_timing.so with -DB200RL_TC_TIMING
    B200RL_LIB_PATH=$PWD/rl_games_b200/libb200rl_timing.so python tools/tc_stage_timing.py     # on the GPU box

The instrumented library is a measurement build only; the product library never contains the stamps."""
import ctypes
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
LABELS = {
    'fwd': ['tile start', 'X staged', 'layer 1 done', 'layer 2 done', 'layer 3 done', 'head done', 'lossA done', 'lossB done'],
    'bwd1': ['tile start', 'loads landed', 'MMA a done', 'd3 epi done', 'MMA b done', 'd2 epi done', 'MMA c half done', 'd1 epi done'],
    'bwd2': ['half start', 'loads landed', 'half done'],
    'bwd2_old': ['tile start', 'X staged', 'loads landed', 'MMAs+bias done'],
}
TAIL = {'fwd': ['kernel end'], 'bwd1': ['flush done'], 'bwd2': ['last MMAs done', 'flush done'], 'bwd2_old': ['last MMAs done', 'flush done']}


VARIANTS = {          # name -> extra -D flags for A/B builds (e.g. the forward kernel's pieces)
    'new': [],
}


def build(variants=('new',)):
    import concurrent.futures as cf
    from rl_games_b200.csrc import build as b
    b.build(verbose=False)
    timed = ('mlp_tc.cu', 'adam.cu')          # the sources that carry opt-in stamps (the relu / tanh units are linked as they are)
    base = [os.path.join(b.OBJ, s[:-3] + '.o') for s in b._sources() if s not in timed]

    def one(job):
        src, name, flags = job
        obj = os.path.join(b.OBJ, '%s_timing_%s.o' % (src[:-3], name))
        subprocess.check_call([b.NVCC] + b.FLAGS + ['-DB200RL_TC_TIMING'] + flags + ['-c', os.path.join(b.HERE, src), '-o', obj])
        return obj
    jobs = [('adam.cu', 'new', [])] + [('mlp_tc.cu', v, VARIANTS[v]) for v in variants]
    with cf.ThreadPoolExecutor(max_workers=6) as ex:
        objs = list(ex.map(one, jobs))
    for v, obj in zip(variants, objs[1:]):
        out = os.path.join(b.PKG, 'libb200rl_timing.so' if v == 'new' else 'libb200rl_timing_%s.so' % v)
        subprocess.check_call([b.NVCC, '-shared', '-gencode', 'arch=compute_90a,code=sm_90a', '-o', out] + base + [objs[0], obj] + ['-lcuda'])
        print(out)


def main():
    import torch
    from rl_games_b200 import ops, _lib
    from rl_games_b200.ops import LossCfg
    DEV = 'cuda'
    D, UNITS, A = 60, [256, 128, 64], 8
    H, N, epm = 16, 16384, 2048
    M = H * epm
    g = torch.Generator().manual_seed(1)
    ins, W, b = D, [], []
    for u in UNITS:
        W.append((torch.randn(u, ins, generator=g) / math.sqrt(ins)).to(DEV)); b.append(torch.zeros(u, device=DEV)); ins = u
    Wh = (torch.randn(A + 1, ins, generator=g) / math.sqrt(ins)).to(DEV); bh = torch.zeros(A + 1, device=DEV)
    logstd = torch.zeros(A, device=DEV)
    obs = torch.randn(H, N, D, device=DEV); nm = torch.zeros(D, device=DEV); ns = torch.ones(D, device=DEV)
    actions = torch.randn(H, N, A, device=DEV); mu = torch.zeros(H, N, A, device=DEV); sg = torch.ones(H, N, A, device=DEV)
    old_v = torch.randn(H, N, device=DEV); ret = torch.randn(H, N, device=DEV)
    old_nlp = torch.full((H, N), 9.0, device=DEV); adv = torch.randn(H, N, device=DEV)
    cfg = LossCfg(0.2, 2.0, 0.0, 1, 2, 1, 1, 1)
    n_tiles = M // 128
    tb = ops.tc_tile_bytes(D, UNITS, A)
    wpack = torch.zeros(ops.tc_pack_bytes(D, UNITS, A), dtype=torch.uint8, device=DEV)
    ops.tc_pack_weights(W[0], W[1], W[2], Wh, D, UNITS, A, wpack)
    act = [torch.zeros(n_tiles * tb[i], dtype=torch.uint8, device=DEV) for i in range(3)]
    dhead = torch.zeros(n_tiles * tb[3], dtype=torch.uint8, device=DEV)
    partials = torch.zeros(132, ops.loss_partial_stride(), dtype=torch.float64, device=DEV)
    sl = lambda t: t[0]   # noqa: E731
    lib = _lib.lib.load()
    fn = lib.b200rl_debug_tc_stamps
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p]
    buf = (ctypes.c_longlong * 384)()
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

    def show(kind, base):
        n = buf[base]
        st = [buf[base + 1 + i] for i in range(n)]
        lab = LABELS[kind]
        head = ['kernel start'] + (['setup (bars)', 'loads issued', 'barrier 1', 'prologue done'] if kind == 'fwd' else [])
        names = head + lab * ((n - len(head) - len(TAIL[kind])) // len(lab)) + TAIL[kind]
        print('  [%s] CTA0: %d stamps, total %.1f us @1.965GHz' % (kind, n, (st[-1] - st[0]) / 1965.0))
        for i in range(1, n):
            print('    %-16s +%7.2f us' % (names[i] if i < len(names) else '?', (st[i] - st[i - 1]) / 1965.0))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=DEV)
    for it in range(4):
        flush.fill_(it)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ops.tc_mlp_fwd_train(sl(obs), epm, N, D, nm, ns, wpack, b, bh, logstd, UNITS, M, A, sl(actions), sl(mu), sl(sg), sl(old_v),
                             sl(ret), sl(old_nlp), sl(adv), None, cfg, None, act, dhead, partials, xtile=xt)
        e1.record()
        # default: single-buffered weight-gradient phase fed with the forward's bf16 X tiles; --no-xt: X re-derived from the fp32
        # observations; --pipelined: the two-stage-ring kernel
        ops.tc_mlp_bwd(sl(obs), epm, N, D, nm, ns, wpack, UNITS, M, A, act, dhead, delta2, delta1, part, P, offs,
                       xtile=None if '--no-xt' in sys.argv else xt, pipelined_wgrad='--pipelined' in sys.argv)
        e2 = torch.cuda.Event(enable_timing=True)
        e2.record()
        torch.cuda.synchronize()
        assert fn(ctypes.cast(buf, ctypes.c_void_p)) == 0
        print('iter %d: fwd+loss %.1f us, bwd1+bwd2 %.1f us (events)' % (it, e0.elapsed_time(e1) * 1e3, e1.elapsed_time(e2) * 1e3))
        if it == 3:
            show('fwd', 0); show('bwd1', 128); show('bwd2' if '--pipelined' in sys.argv else 'bwd2_old', 256)
    # ---- fused reduce + finalise + clip + Adam tail on the partial rows the backward just wrote (L2-hot, like in the real step) ----
    ra = lib.b200rl_debug_ra_stamps
    ra.restype = ctypes.c_int
    ra.argtypes = [ctypes.c_void_p]
    rbuf = (ctypes.c_longlong * 32)()
    from rl_games_b200.ops import OptCfg
    Ppad = (P + 3) // 4 * 4
    part4 = torch.randn(132, Ppad, device=DEV) * 1e-3
    flat, m1, m2, grad = torch.randn(P, device=DEV) * 0.1, torch.zeros(P, device=DEV), torch.zeros(P, device=DEV), torch.zeros(P, device=DEV)
    state = torch.tensor([3e-4, 0.0, 0.0, 0.0], dtype=torch.float64, device=DEV)
    cfg_o = OptCfg(0.9, 0.999, 1e-8, 0.0, 1.0, 0.008, 1e-6, 1e-2, 1.5, 1.0, 1, 1)
    counter, bar = torch.zeros(1, dtype=torch.int32, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV)
    nrm, stats, kl, ec = torch.zeros(132, dtype=torch.float64, device=DEV), torch.zeros(16, device=DEV), torch.zeros(1, device=DEV), torch.zeros(1, device=DEV)
    for it in range(4):
        part4.mul_(1.0)          # rewrite the partial rows so that they sit in L2 as after the backward kernel
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ops.reduce_adam(part4, 132, Ppad, partials, 132, A, ec, stats, kl, grad, flat, m1, m2, P, state, cfg_o, counter, nrm, bar)
        e1.record()
        torch.cuda.synchronize()
        assert ra(ctypes.cast(rbuf, ctypes.c_void_p)) == 0
        if it == 3:
            names = ['kernel start', 'finalise branch', 'split reduction', 'grid barrier', 'Adam slice', 'kernel end']
            print('  [reduce_adam] %.1f us by events; CTA0:' % (e0.elapsed_time(e1) * 1e3))
            for i in range(1, 6):
                print('    %-16s +%7.2f us' % (names[i], (rbuf[i] - rbuf[i - 1]) / 1965.0))


if __name__ == '__main__':
    if '--build-variants' in sys.argv:
        build(tuple(VARIANTS))
    elif '--build' in sys.argv:
        build()
    else:
        main()
