"""Developer tool: time the categorical kernels (rollout sample, training loss, player argmax) at wide layouts and at the narrow kernels'
largest ones, against torch doing the same work on the same GPU, and compare their outputs.

Shapes (rows x layout): Discrete(362) (Go 19x19), Discrete(4672) (a chess move encoding), the gym-microrts unit-command Tuple on a 16 x 16
map (1792 heads of [6, 4, 4, 4, 4, 7, 49], 19968 logits), and 64 actions / 8 x 64 on both the narrow and the wide kernels.  Masks: a
random half of each head legal (one action forced).  torch: per head, masked log-softmax and Categorical sampling (as
CategoricalMasked / ModelA2CMultiDiscrete do), the loss's masked log-softmax, entropy and autograd backward, and argmax.

Times are CUDA events around `reps` back-to-back launches, after warm-up; the median of `rounds` alternated rounds.  The card's name and
power limit are read in the same run.
Usage: python tools/cat_wide_ab.py [--rounds 5] [--reps 20] [--out FILE]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from rl_games_b200 import ops  # noqa: E402
from rl_games_b200._lib import lib  # noqa: E402
from oracle import ppo_discrete_oracle as DO  # noqa: E402

DEV = 'cuda:0'
MICRORTS = [6, 4, 4, 4, 4, 7, 49] * 256
SHAPES = [('Discrete(362)', 8192, [362]), ('Discrete(4672)', 2048, [4672]), ('microrts 1792 heads', 512, MICRORTS),
          ('Discrete(64)', 8192, [64]), ('8 x 64', 4096, [64] * 8)]


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else torch.cuda.get_device_name(0)


def timed(fn, reps, rounds):
    for _ in range(3):
        fn()
    out = []
    for _ in range(rounds):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(reps):
            fn()
        e.record()
        torch.cuda.synchronize()
        out.append(s.elapsed_time(e) / reps)
    return sorted(out)[len(out) // 2]


class Case:
    def __init__(self, M, sizes, seed=0):
        g = torch.Generator().manual_seed(seed)
        self.M, self.sizes, self.K, self.nh = M, sizes, sum(sizes), len(sizes)
        self.hs = None if len(sizes) == 1 else sizes
        self.head = (torch.randn(M, 1 + self.K, generator=g) * 2).to(DEV)
        mk = torch.rand(M, self.K, generator=g) < 0.5
        off = 0
        for k in sizes:
            mk[torch.arange(M), off + torch.randint(0, k, (M,), generator=g)] = True
            off += k
        self.mk = mk.to(DEV)
        self.mk8 = self.mk.to(torch.uint8)
        self.u = torch.rand(self.nh, M, generator=g).to(DEV)
        self.acts = torch.zeros(M, self.nh, dtype=torch.int64, device=DEV)
        self.nlp, self.vals = torch.zeros(M, device=DEV), torch.zeros(M, device=DEV)
        self.dl = torch.zeros(M, self.K, device=DEV)
        self.dv = torch.zeros(M, 1, device=DEV)
        self.old_nlp = torch.rand(M, device=DEV) * self.nh
        self.adv, self.old_v, self.ret = (torch.randn(M, generator=g).to(DEV) for _ in range(3))
        self.part = torch.zeros(M, 8, dtype=torch.float64, device=DEV)
        self.cfg = ops.CatLossCfg(0.2, 1.0, 0.01, 1, 0, 1)
        self.amax = torch.zeros(M, self.nh, dtype=torch.int64, device=DEV)
        if self.hs:
            self.tab = ops._head_table(self.hs)[1]
            self.off = ops._head_offsets(self.hs, DEV)

    # ---- the kernels through ops (the layout picks narrow or wide), or the wide entry points forced at a narrow layout ----
    def sample(self, wide=None, u=True):
        if not wide:
            ops.categorical_sample(self.head[:, 1:], 1 + self.K, self.K, self.head, 1 + self.K, self.mk8, self.u if u else None, 1,
                                   None, 0, None, None, False, self.acts, self.nlp, self.vals, None, None, None, None, self.M,
                                   head_sizes=self.hs)
            return
        lib.b200rl_categorical_sample_wide_f32(
            self.head[:, 1:].data_ptr(), 1 + self.K, self.K, self.nh if self.hs else 0, None if not self.hs else ctypes_addr(self.tab),
            None if not self.hs else self.off.data_ptr(), self.head.data_ptr(), 1 + self.K, self.mk8.data_ptr(),
            self.u.data_ptr() if u else None, 1, None, 0, None, None, 0, self.acts.data_ptr(), self.nlp.data_ptr(), self.vals.data_ptr(),
            None, None, None, None, self.M, ops._stream())

    def loss(self, wide=None):
        args = (self.head[:, 1:], 1 + self.K, self.K, self.head, 1 + self.K, self.acts, self.mk8, self.old_v, self.ret, self.old_nlp,
                self.adv, None, self.M, 0, self.M, self.cfg, None, self.dl, self.K, self.dv, 1, self.part)
        if not wide:
            return ops.categorical_loss(*args, head_sizes=self.hs)
        nb = ctypes.c_int(0)
        lib.b200rl_categorical_loss_wide_f32(
            self.head[:, 1:].data_ptr(), 1 + self.K, self.K, self.nh if self.hs else 0, None if not self.hs else ctypes_addr(self.tab),
            None if not self.hs else self.off.data_ptr(), self.head.data_ptr(), 1 + self.K, self.acts.data_ptr(), self.mk8.data_ptr(),
            self.old_v.data_ptr(), self.ret.data_ptr(), self.old_nlp.data_ptr(), self.adv.data_ptr(), None, self.M, 0, self.M,
            ctypes_addr(self.cfg), None, self.dl.data_ptr(), self.K, self.dv.data_ptr(), 1, self.part.data_ptr(), self.M,
            ctypes_addr(nb), ops._stream())
        return nb.value

    def argmax(self, wide=None):
        if not wide:
            ops.categorical_argmax(self.head[:, 1:], 1 + self.K, self.K, self.mk8, self.amax, self.M, head_sizes=self.hs)
            return
        lib.b200rl_categorical_argmax_wide_f32(self.head[:, 1:].data_ptr(), 1 + self.K, self.K, self.nh if self.hs else 0,
                                               None if not self.hs else ctypes_addr(self.tab), None if not self.hs else self.off.data_ptr(),
                                               self.mk8.data_ptr(), self.amax.data_ptr(), self.M, ops._stream())

    # ---- torch on the same GPU, head by head ----
    def _split(self, z):
        return zip(torch.split(z, self.sizes, dim=1), torch.split(self.mk, self.sizes, dim=1))

    def torch_sample(self):
        out = []
        for z, m in self._split(self.head[:, 1:]):
            lg = torch.log_softmax(torch.where(m, z, torch.tensor(-1e8, device=DEV)), -1)
            out.append(torch.distributions.Categorical(logits=lg).sample())
        return out

    def torch_loss(self):
        z = self.head[:, 1:].detach().requires_grad_(True)
        nlp, ent = 0.0, 0.0
        for j, (zz, m) in enumerate(self._split(z)):
            lg = torch.log_softmax(torch.where(m, zz, torch.tensor(-1e8, device=DEV)), -1)
            nlp = nlp - lg.gather(1, self.acts[:, j:j + 1]).squeeze(1)
            ent = ent - torch.where(m, lg.exp() * lg, torch.zeros((), device=DEV)).sum(-1)
        ratio = torch.exp(self.old_nlp - nlp)
        a = torch.max(-self.adv * ratio, -self.adv * ratio.clamp(0.8, 1.2))
        (a.mean() - 0.01 * ent.mean()).backward()
        return z.grad

    def torch_argmax(self):
        return [torch.where(m, z, torch.tensor(float('-inf'), device=DEV)).argmax(-1) for z, m in self._split(self.head[:, 1:])]


def ctypes_addr(x):
    return ctypes.addressof(x)


def compare(c):
    """outputs at this shape: tape-sampled actions against the fp64 inverse-cdf rule (share of rows that agree), argmax against torch;
    wide vs narrow kernels where both run (the loss kernels against fp64: tests/test_cat_wide_gpu.py)"""
    res = {}
    c.sample(u=True)
    torch.cuda.synchronize()
    acts = c.acts.clone()
    agree = []
    for j, (z, m) in enumerate(c._split(c.head[:, 1:])):
        _, p, _ = DO.categorical_masked(z.double(), m)
        agree.append((DO.sample_inverse_cdf(p, c.u[j].double()) == acts[:, j]).float().mean().item())
    res['sample_vs_rule_agree'] = min(agree)
    c.argmax()
    torch.cuda.synchronize()
    res['argmax_vs_torch_equal'] = bool(torch.equal(c.amax, torch.stack(c.torch_argmax(), 1)))
    nb = c.loss()
    torch.cuda.synchronize()
    res['loss_partial_rows'] = nb
    if not ops.categorical_is_wide(c.K, c.hs):
        dl_n, part_n, acts_n, am_n = c.dl.clone(), c.part[:nb].sum(0), acts, c.amax.clone()
        c.sample(wide=True)
        c.argmax(wide=True)
        nbw = c.loss(wide=True)
        torch.cuda.synchronize()
        res['wide_vs_narrow_actions_equal'] = float((c.acts == acts_n).float().mean())
        res['wide_vs_narrow_argmax_equal'] = bool(torch.equal(c.amax, am_n))
        res['wide_vs_narrow_dlogits_max_abs'] = float((c.dl - dl_n).abs().max())
        res['wide_vs_narrow_loss_sums_max_rel'] = float(((c.part[:nbw].sum(0) - part_n).abs() / part_n.abs().clamp(min=1e-12))[:4].max())
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'cat_wide_ab.py times kernels on a GPU'
    torch.backends.cuda.matmul.allow_tf32 = False
    out = {'card': card(), 'rows': {}}
    for name, M, sizes in SHAPES:
        c = Case(M, sizes)
        r = {'M': M, 'heads': len(sizes), 'K': sum(sizes), 'path': 'wide' if ops.categorical_is_wide(c.K, c.hs) else 'narrow'}
        r.update(compare(c))
        tr = max(1, args.reps // 10) if len(sizes) > 8 else args.reps
        r['ms'] = {'sample': timed(lambda: c.sample(u=False), args.reps, args.rounds),
                   'loss': timed(c.loss, args.reps, args.rounds),
                   'argmax': timed(c.argmax, args.reps, args.rounds),
                   'torch_sample': timed(c.torch_sample, tr, args.rounds),
                   'torch_loss': timed(c.torch_loss, tr, args.rounds),
                   'torch_argmax': timed(c.torch_argmax, tr, args.rounds)}
        if r['path'] == 'narrow':
            r['ms'].update({'wide_sample': timed(lambda: c.sample(wide=True, u=False), args.reps, args.rounds),
                            'wide_loss': timed(lambda: c.loss(wide=True), args.reps, args.rounds),
                            'wide_argmax': timed(lambda: c.argmax(wide=True), args.reps, args.rounds)})
        # bytes the loss must move at least: logits and their gradient (fp32), masks (uint8), per row scalars
        r['loss_min_bytes'] = M * (9 * c.K + 8 * c.nh + 28)
        r['loss_GBps'] = r['loss_min_bytes'] / (r['ms']['loss'] * 1e-3) / 1e9
        out['rows'][name] = r
        print(name, json.dumps(r), flush=True)
    print(json.dumps(out))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
