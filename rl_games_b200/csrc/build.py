"""Build libb200rl.so (sm_90a only) with nvcc.  In-tree output: rl_games_b200/libb200rl.so
(git-ignored).  Cross-compiles without a GPU.

A second, TEST-ONLY library tests/libb200rl_testhooks.so is the same objects with the translation units that hold
`#ifdef B200RL_TEST_HOOKS` host entry points (b200rl_hosttest_*: per-thread kernel bodies run over host arrays by the CPU
tests) recompiled with that macro.  The product library does not export them and nothing in rl_games_b200/ loads the
test library.

A third, TEST-ONLY library tests/libb200rl_l2poison.so recompiles the translation units that drop dead lines from L2
(tc::l2_discard) with B200RL_L2_DISCARD_POISON: every discard becomes a store of 0xFF bytes (NaN in fp32 and bf16), so a read
after a discard shows up as NaN in the tests instead of as a timing-dependent stale value."""
import concurrent.futures as cf
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
OUT = os.path.join(PKG, 'libb200rl.so')
OBJ = os.path.join(HERE, '_obj')
HOOKS_OUT = os.path.join(os.path.dirname(PKG), 'tests', 'libb200rl_testhooks.so')
HOOKS_DEFINE = 'B200RL_TEST_HOOKS'
POISON_OUT = os.path.join(os.path.dirname(PKG), 'tests', 'libb200rl_l2poison.so')
POISON_DEFINE = 'B200RL_L2_DISCARD_POISON'
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
         '-Xcompiler', '-fPIC', '-Xcompiler', '-fvisibility=hidden', '--expt-relaxed-constexpr']


def _sources():
    return sorted(f for f in os.listdir(HERE) if f.endswith('.cu'))


def _digest(path):
    h = hashlib.sha1()
    extra = [os.path.join(HERE, 'mlp_tc.cu')] if os.path.basename(path) in ('mlp_tc_relu.cu', 'mlp_tc_tanh.cu') else []     # they #include it
    for dep in [path] + extra + [os.path.join(HERE, f) for f in sorted(os.listdir(HERE)) if f.endswith(('.cuh', '.h'))] + \
            [os.path.join(os.path.dirname(PKG), 'include', 'b200rl.h')]:
        with open(dep, 'rb') as f:
            h.update(f.read())
    h.update(' '.join(FLAGS).encode())
    return h.hexdigest()


def _has_hooks(src):
    with open(os.path.join(HERE, src)) as f:
        return ('#ifdef ' + HOOKS_DEFINE) in f.read()


def _uses_discard(src):
    with open(os.path.join(HERE, src)) as f:
        return 'l2_discard(' in f.read()


def _compile(src, hooks=False, poison=False):
    path = os.path.join(HERE, src)
    obj = os.path.join(OBJ, src[:-3] + ('.hooks.o' if hooks else '.poison.o' if poison else '.o'))
    stamp = obj + '.sha1'
    dig = _digest(path) + ('+hooks' if hooks else '+poison' if poison else '')
    if os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dig:
        return obj, False
    cmd = [NVCC] + FLAGS + (['-D' + HOOKS_DEFINE] if hooks else []) + (['-D' + POISON_DEFINE] if poison else []) + ['-c', path, '-o', obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('nvcc failed for %s:\n%s\n%s' % (src, r.stdout, r.stderr))
    with open(stamp, 'w') as f:
        f.write(dig)
    return obj, True


def build(verbose=True):
    os.makedirs(OBJ, exist_ok=True)
    srcs = _sources()
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        res = list(ex.map(_compile, srcs))
    objs = [o for o, _ in res]
    rebuilt = any(ch for _, ch in res) or not os.path.exists(OUT)
    if rebuilt:
        cmd = [NVCC, '-shared', '-gencode', 'arch=compute_90a,code=sm_90a', '-o', OUT] + objs + ['-lcuda']
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('link failed:\n%s\n%s' % (r.stdout, r.stderr))
    if verbose:
        print('libb200rl: %s (%d sources, %s)' % (OUT, len(srcs), 'rebuilt' if rebuilt else 'up to date'))
    return OUT


def build_test_hooks(verbose=True):
    """tests/libb200rl_testhooks.so: the product objects, with the hook-carrying translation units recompiled with -DB200RL_TEST_HOOKS.
    Loaded only by the CPU tests (tests/_torch_ops.py::_host_lib and the *_rows_cpu tests)."""
    build(verbose=False)
    srcs = _sources()
    hook_srcs = [s for s in srcs if _has_hooks(s)]
    with cf.ThreadPoolExecutor(max_workers=min(8, max(1, len(hook_srcs)))) as ex:
        res = list(ex.map(lambda s: _compile(s, hooks=True), hook_srcs))
    objs = [o for o, _ in res] + [os.path.join(OBJ, s[:-3] + '.o') for s in srcs if s not in hook_srcs]
    if any(ch for _, ch in res) or not os.path.exists(HOOKS_OUT) or os.path.getmtime(HOOKS_OUT) < os.path.getmtime(OUT):
        cmd = [NVCC, '-shared', '-gencode', 'arch=compute_90a,code=sm_90a', '-o', HOOKS_OUT] + objs + ['-lcuda']
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('link failed:\n%s\n%s' % (r.stdout, r.stderr))
    if verbose:
        print('test hooks: %s (%s recompiled with -D%s)' % (HOOKS_OUT, ', '.join(hook_srcs), HOOKS_DEFINE))
    return HOOKS_OUT


def build_l2_poison(verbose=True):
    """tests/libb200rl_l2poison.so: the product objects, with the translation units that call tc::l2_discard recompiled with
    -DB200RL_L2_DISCARD_POISON.  Loaded only by the GPU tests (tests/test_l2_discard_gpu.py, through B200RL_LIB_PATH)."""
    build(verbose=False)
    srcs = _sources()
    poison_srcs = [s for s in srcs if _uses_discard(s)]
    with cf.ThreadPoolExecutor(max_workers=min(8, max(1, len(poison_srcs)))) as ex:
        res = list(ex.map(lambda s: _compile(s, poison=True), poison_srcs))
    objs = [o for o, _ in res] + [os.path.join(OBJ, s[:-3] + '.o') for s in srcs if s not in poison_srcs]
    if any(ch for _, ch in res) or not os.path.exists(POISON_OUT) or os.path.getmtime(POISON_OUT) < os.path.getmtime(OUT):
        cmd = [NVCC, '-shared', '-gencode', 'arch=compute_90a,code=sm_90a', '-o', POISON_OUT] + objs + ['-lcuda']
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('link failed:\n%s\n%s' % (r.stdout, r.stderr))
    if verbose:
        print('L2-discard poison: %s (%s recompiled with -D%s)' % (POISON_OUT, ', '.join(poison_srcs), POISON_DEFINE))
    return POISON_OUT


if __name__ == '__main__':
    build()
    build_test_hooks()
    build_l2_poison()
