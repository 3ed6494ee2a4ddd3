"""Developer tool: which device functions changed since <commit>?  Rebuilds every csrc/*.cu of that commit into a scratch directory with
the product's flags and compares the SASS of each kernel with the current objects (names / addresses normalised).  Used at the end of a
round without GPU time left to show that hardware-validated kernels are byte-identical to what was validated.
Usage: python tools/sass_vs_commit.py <commit>   (run rl_games_b200/csrc/build.py first)"""
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17', '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr']


def funcs(obj):
    txt = subprocess.run(['cuobjdump', '-sass', obj], capture_output=True, text=True).stdout
    out, cur = {}, None
    for line in txt.splitlines():
        m = re.search(r'Function : (\S+)', line)
        if m:
            cur = re.sub(r'_GLOBAL__N__[0-9a-f]+_\d+_\w+?_cu_[0-9a-f]+', 'NS', m.group(1))
            out[cur] = []
        elif cur is not None:
            # addresses dropped, whitespace collapsed: a longer object widens cuobjdump's address column, which pads every line
            ln = re.sub(r'\s+', ' ', re.sub(r'/\*[0-9a-f]{4,}\*/', '', line)).strip()
            if ln:
                out[cur].append(ln)
    return out


def main():
    commit = sys.argv[1]
    tmp = tempfile.mkdtemp(prefix='sass_old_')
    os.makedirs(os.path.join(tmp, 'rl_games_b200', 'csrc'))
    os.makedirs(os.path.join(tmp, 'include'))
    files = subprocess.run(['git', '-C', ROOT, 'ls-tree', '-r', '--name-only', commit, 'rl_games_b200/csrc', 'include'],
                           capture_output=True, text=True, check=True).stdout.split()
    for f in files:
        if f.endswith(('.cu', '.cuh', '.h')):
            with open(os.path.join(tmp, f), 'w') as fh:
                fh.write(subprocess.run(['git', '-C', ROOT, 'show', f'{commit}:{f}'], capture_output=True, text=True, check=True).stdout)
    changed = 0
    for f in sorted(x for x in files if x.endswith('.cu')):
        name = os.path.basename(f)[:-3]
        new_obj = os.path.join(ROOT, 'rl_games_b200', 'csrc', '_obj', name + '.o')
        old_obj = os.path.join(tmp, name + '.o')
        r = subprocess.run(['nvcc'] + FLAGS + ['-c', os.path.join(tmp, f), '-o', old_obj], capture_output=True, text=True)
        if r.returncode or not os.path.exists(new_obj):
            print(f'{name}: cannot compare ({(r.stderr or "no current object").strip()[:120]})')
            continue
        old, new = funcs(old_obj), funcs(new_obj)
        # a changed signature (extra template argument, arguments packed into a struct) renames a kernel: pair such functions by body
        gone = {k: v for k, v in old.items() if k not in new}
        for k in [k for k in new if k not in old]:
            twin = next((g for g, body in gone.items() if body == new[k]), None)
            if twin is not None:
                print(f'{name:10s} renamed, body identical  {k[:80]}')
                del gone[twin], old[twin]
                del new[k]
        for k in sorted(set(old) | set(new)):
            if k not in old:
                print(f'{name:10s} NEW        {k[:90]}'); changed += 1
            elif k not in new:
                print(f'{name:10s} REMOVED    {k[:90]}'); changed += 1
            elif old[k] != new[k]:
                print(f'{name:10s} DIFFERENT  {k[:90]}  ({len(old[k])} -> {len(new[k])} SASS lines)'); changed += 1
    print(f'{changed} device functions differ from {commit}; every other kernel is byte-identical')


if __name__ == '__main__':
    main()
