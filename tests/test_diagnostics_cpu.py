"""`use_diagnostics: True` on the CPU: the oracle against the reference's golden runs, the explained-variance kernel's finalisation
(through the test-hook library) against the oracle, and the agents' host logic -- replaying the epoch's read-back stats rows into the
diagnostics object -- with torch stand-ins for every op, against the same golden runs."""
import ctypes
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _diag_oracle as DO  # noqa: E402
import _hooks  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')
RUNS = ['diag_mlp.pt', 'diag_masked_rmsadv.pt', 'diag_lstm.pt', 'diag_discrete.pt']


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def _diag_rows(scalars):
    return [s for s in scalars if s[0].startswith('diagnostics/')]


def _same(a, b, rel):
    if math.isnan(b) or math.isinf(b):
        return (math.isnan(a) and math.isnan(b)) or a == b
    return a == pytest.approx(b, rel=rel, abs=1e-12)


@pytest.mark.parametrize('name', RUNS)
def test_oracle_reproduces_the_reference_diagnostics(name):
    g = _load(name)
    cfg, di = g['config'], g['diag_inputs']
    nmb = g['N'] * g['H'] // g['mb']
    got = DO.scalars(di['mini_batches'], di['epochs'], cfg['mini_epochs'], nmb)
    want = _diag_rows(g['train_loop']['scalars'])
    assert [(t, s) for t, _, s in got] == [(t, s) for t, _, s in want]
    for (t, v, _), (_, rv, _) in zip(got, want):
        assert _same(v, rv, 1e-6), (t, v, rv)


def _finalize(sums, masked):
    lib = _hooks.load()
    fn = lib.b200rl_hosttest_expvar_finalize
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    s = torch.tensor(sums, dtype=torch.float64).reshape(-1, 3).contiguous()
    out = torch.zeros(s.shape[0])
    assert fn(ctypes.c_void_p(s.data_ptr()), s.shape[0], int(masked), ctypes.c_void_p(out.data_ptr())) == 0
    return out


def _sums(v, r, m):
    """what the kernel's two passes accumulate for one minibatch: (n, sum sq dev of y, sum sq dev of r - v) over the valid rows"""
    sel = torch.ones_like(v, dtype=torch.bool) if m is None else m != 0
    v, r = v[sel].double(), r[sel].double()
    y = r if m is None else v
    d = (r.float() - v.float()).double()
    n = float(sel.sum())
    return [n, float(((y - y.mean()) ** 2).sum()) if n else 0.0, float(((d - d.mean()) ** 2).sum()) if n else 0.0]


@pytest.mark.parametrize('masked', [False, True])
def test_kernel_finalisation_matches_the_oracle(masked):
    g = torch.Generator().manual_seed(5)
    for trial in range(20):
        B = [64, 7, 2, 300][trial % 4]
        v, r = torch.randn(B, generator=g), torch.randn(B, generator=g) * 1.5 + 0.3
        m = (torch.rand(B, generator=g) < 0.7).float() if masked else None
        if masked and m.sum() < 2:
            m[:2] = 1.0
        got = _finalize(_sums(v, r, m), masked)[0]
        ref = DO.explained_variance(v.unsqueeze(1), r.unsqueeze(1), m)
        torch.testing.assert_close(got, ref.float(), rtol=2e-5, atol=2e-6)


def test_kernel_finalisation_degenerate_inputs_give_inf_or_nan_like_the_reference():
    c, r = torch.full((6,), 0.5), torch.tensor([1.0, 2.0, 0.0, 1.0, 3.0, -1.0])
    assert _finalize(_sums(c, c, None), False)[0].isnan()                  # 0 / 0
    # var_y = 0 with var_dy > 0: -inf (unmasked y = returns, masked y = values)
    assert _finalize(_sums(r, torch.full((6,), 2.0), None), False)[0] == -math.inf
    ref = DO.explained_variance(r.unsqueeze(1), torch.full((6, 1), 2.0))
    assert ref == -math.inf
    m = torch.ones(6)
    assert _finalize(_sums(c, r, m), True)[0] == -math.inf
    assert DO.explained_variance(c.unsqueeze(1), r.unsqueeze(1), m) == -math.inf
    # sum(m) of 0 and of 1: both variances 0 -> NaN, in the reference too
    for k in (0, 1):
        mk = torch.zeros(6)
        mk[:k] = 1.0
        assert _finalize(_sums(r, c, mk), True)[0].isnan()
        assert DO.explained_variance(r.unsqueeze(1), c.unsqueeze(1), mk).isnan()
    # masked rows are left out: non-finite garbage there changes nothing
    mk = torch.tensor([1.0, 1.0, 0.0, 1.0, 0.0, 1.0])
    rp = r.clone()
    rp[2], rp[4] = float('nan'), float('inf')
    assert torch.equal(_finalize(_sums(c + r, rp, mk), True), _finalize(_sums(c + r, r, mk), True))


# ---------------------------------------------------------------------------------------------------------------- agents' host logic
def explained_variance_stand_in(values, returns, mask, H, N, envs_per_mb, out, n_rep=1):
    """torch stand-in of ops.explained_variance: the oracle over each whole-env minibatch of the arena"""
    n_mb = N // envs_per_mb
    for i in range(n_mb):
        sl = slice(i * envs_per_mb, (i + 1) * envs_per_mb)
        fl = lambda t: t[:, sl].transpose(0, 1).reshape(-1)     # noqa: E731
        ev = DO.explained_variance(fl(values).unsqueeze(1), fl(returns).unsqueeze(1), None if mask is None else fl(mask))
        for k in range(n_rep):
            out[k * n_mb + i] = ev


def _categorical_loss_with_clip_sums(orig):
    """the discrete loss stand-in plus the kernel's partial columns 4 / 5 (sum mask, sum mask * clipped, csrc/discrete.cu), which the
    discrete agent sums for diagnostics/clip_frac"""
    import _torch_ops as T

    def fn(logits, ld, K, values, value_ld, actions, action_masks, old_values_n, returns_n, old_neglogp, advs_n, mask, rows_per_chunk,
           chunk_stride, M, cfg, inv_count, d_logits, d_ld, d_value, dv_ld, partials, head_sizes=None):
        arena = lambda t, w=1: T._rows(t, M, w, rows_per_chunk, chunk_stride, w)      # noqa: E731
        mrow = torch.arange(M)
        z = T._flat(logits)[(mrow * ld).unsqueeze(1) + torch.arange(K).unsqueeze(0)].clone()
        nh = len(head_sizes) if head_sizes else 1
        act = arena(actions, nh)
        am = None if action_masks is None else arena(action_masks, K).bool()
        heads = T._cat_heads(z, am, head_sizes)
        nlp = sum(-h[0].gather(1, act[:, j:j + 1]).squeeze(1) for j, h in enumerate(heads))
        clipped = ((arena(old_neglogp).squeeze(1) - nlp).exp() - 1.0).abs() > cfg.e_clip
        m = torch.ones(M) if mask is None else arena(mask).squeeze(1)
        nb = orig(logits, ld, K, values, value_ld, actions, action_masks, old_values_n, returns_n, old_neglogp, advs_n, mask, rows_per_chunk,
                  chunk_stride, M, cfg, inv_count, d_logits, d_ld, d_value, dv_ld, partials, head_sizes)
        partials[0, 4], partials[0, 5] = float(m.sum()), float((m * clipped.float()).sum())
        return nb
    return fn


def _agent(name, monkeypatch, tmp_path, over):
    g = _load(name)
    keys = ('max_epochs', 'save_frequency', 'save_best_after', 'games_to_track', 'use_diagnostics')
    if name == 'diag_discrete.pt':
        import test_discrete_host_cpu as HD
        agent = HD._build(monkeypatch, tmp_path, g, over={k: g['config'][k] for k in keys if k in g['config']} | over)
        from rl_games_b200 import ops
        monkeypatch.setattr(ops, 'categorical_loss', _categorical_loss_with_clip_sums(ops.categorical_loss))
        tape = g['u']
        orig = agent.train_epoch
        agent.train_epoch = lambda: orig(u=tape[agent.epoch_num - 1])
    else:
        import test_agent_host_cpu as HC
        agent = HC._build(monkeypatch, tmp_path, g, HC._Env(g), over={k: g['config'][k] for k in keys if k in g['config']} | over)
        orig = agent.train_epoch
        agent.train_epoch = lambda: orig(noise=g['noise'][agent.epoch_num - 1])
    from rl_games_b200 import ops
    monkeypatch.setattr(torch.Tensor, 'pin_memory', lambda self: self)
    calls = []

    def ev(*a, **k):
        calls.append(a)
        return explained_variance_stand_in(*a, **k)
    monkeypatch.setattr(ops, 'explained_variance', ev)
    return g, agent, calls


def _run(agent):
    scalars = []
    agent.writer = type('W', (), {'add_scalar': lambda self, tag, v, step=None: scalars.append((tag, float(v), step))})()
    agent.algo_observer.writer = agent.writer
    agent.train()
    return scalars


@pytest.mark.parametrize('name', RUNS)
def test_agent_writes_the_reference_diagnostics(name, monkeypatch, tmp_path):
    g, agent, calls = _agent(name, monkeypatch, tmp_path, {})
    assert agent.diag_on
    scalars = _run(agent)
    ref = g['train_loop']['scalars']
    # every tag the reference writes, at the same steps and in the same order (diagnostics first, in write_stats)
    assert [(t, s) for t, _, s in scalars if not t.endswith('/time')] == [(t, s) for t, _, s in ref if not t.endswith('/time')]
    assert len(calls) == agent.epoch_num == 2
    B = g['mb']
    for (t, v, _), (_, rv, _) in zip(_diag_rows(scalars), _diag_rows(ref)):
        if '/clip_frac/' in t:
            # a row at the clip boundary may flip between two implementations: at most one row per minibatch
            bound = 1.0 / B / (B if g['autoreset'] == 'next_step' else 1)
            assert abs(v - rv) <= bound + 1e-7, (t, v, rv)
        else:
            assert _same(v, rv, 1e-4), (t, v, rv)


@pytest.mark.parametrize('name', ['diag_mlp.pt', 'diag_discrete.pt'])
def test_key_off_launches_nothing_writes_nothing_and_syncs_alike(name, monkeypatch, tmp_path):
    import test_agent_host_cpu as HC
    counts = {}
    for on in (False, True):
        g, agent, calls = _agent(name, monkeypatch, tmp_path / str(on), {'use_diagnostics': on})
        n = {'sync': 0}
        if name == 'diag_discrete.pt':
            monkeypatch.setattr(type(agent), '_sync', staticmethod(lambda: n.__setitem__('sync', n['sync'] + 1)))
        else:
            class _S(HC._Stream):
                def synchronize(self):
                    n['sync'] += 1
            monkeypatch.setattr(torch.cuda, 'current_stream', lambda *a: _S())
        scalars = _run(agent)
        assert agent.diag_on == on and bool(calls) == on
        assert any(t.startswith('diagnostics/') for t, _, _ in scalars) == on
        counts[on] = n['sync']
    assert counts[False] == counts[True] > 0


def test_only_rank_zero_gets_the_diagnostics_object():
    from rl_games_b200.diagnostics import DefaultDiagnostics, PpoDiagnostics, make_diagnostics
    assert type(make_diagnostics(True, 0)) is PpoDiagnostics
    assert type(make_diagnostics(True, 1)) is DefaultDiagnostics
    assert type(make_diagnostics(False, 0)) is DefaultDiagnostics
