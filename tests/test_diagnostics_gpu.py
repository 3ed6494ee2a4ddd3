"""`use_diagnostics: True` on the GPU: the explained-variance kernel against the oracle (masked rows poisoned), the agents' diagnostics
summaries against the reference's golden runs (eager and CUDA graph), and the summaries as pure observers: with the key on and off the
same seeds give the same bits."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _diag_oracle as DO  # noqa: E402
from oracle import ppo_oracle as O  # noqa: E402
from test_agent_gpu import DEV, TapeEnvGPU, make_agent  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')


@pytest.mark.parametrize('masked', [False, True])
def test_explained_variance_kernel_matches_oracle_and_ignores_masked_rows(masked):
    from rl_games_b200 import ops
    H, N, epm, reps = 16, 1024, 256, 3
    g = torch.Generator().manual_seed(11)
    v = (torch.randn(H, N, generator=g) * 0.8 + 0.1).to(DEV)
    r = (v.cpu() + torch.randn(H, N, generator=g) * 0.5).to(DEV)
    m = (torch.rand(H, N, generator=g) < 0.75).float().to(DEV) if masked else None
    nmb = N // epm
    outs = []
    for _ in range(2):
        out = torch.full((reps * nmb * 16,), 7.0, device=DEV)
        ops.explained_variance(v, r, m, H, N, epm, out[9::16], n_rep=reps)
        outs.append(out)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])                     # deterministic merge
    out = outs[0].reshape(reps * nmb, 16)
    assert torch.equal(out[:, :9], torch.full_like(out[:, :9], 7.0)) and torch.equal(out[:, 10:], torch.full_like(out[:, 10:], 7.0))
    for i in range(nmb):
        fl = lambda t: t[:, i * epm:(i + 1) * epm].transpose(0, 1).reshape(-1).cpu()      # noqa: E731
        ref = DO.explained_variance(fl(v).unsqueeze(1), fl(r).unsqueeze(1), None if m is None else fl(m))
        for k in range(reps):
            torch.testing.assert_close(out[k * nmb + i, 9].cpu(), ref, rtol=1e-5, atol=1e-6)
    if masked:      # poison test: non-finite garbage in masked rows changes nothing
        vp, rp = v.clone(), r.clone()
        vp[m == 0], rp[m == 0] = float('nan'), float('inf')
        out_p = torch.zeros(nmb, device=DEV)
        ops.explained_variance(vp, rp, m, H, N, epm, out_p)
        torch.cuda.synchronize()
        assert torch.equal(out_p, out[:nmb, 9])


def _train_continuous(name, graph, over=None):
    g = torch.load(os.path.join(GOLDEN, name), weights_only=False)
    cfg = {k: v for k, v in g['config'].items() if k not in ('device', 'torch_compile', 'train_dir', 'reward_shaper')}
    cfg.update({'b200_cuda_graph': graph, 'lr_schedule': g['config'].get('lr_schedule', None), 'print_stats': False,
                'train_dir': '/tmp/b200_parity_runs'}, **(over or {}))
    env = TapeEnvGPU(g['obs_tape'], g['done_tape'], g['timeout_tape'], g['A'], g['autoreset'])
    agent = make_agent(cfg, g['N'], g['H'], g['D'], g['A'], g['units'], g['mb'], env, g['init_state'], network_over=g.get('network_over'))
    orig = agent.train_epoch
    agent.train_epoch = lambda: orig(noise=g['noise'][agent.epoch_num - 1].to(DEV))
    return g, agent, _run(agent)


def _run(agent):
    rows, stats = [], []
    agent.writer = type('W', (), {'add_scalar': lambda self, tag, v, step=None: rows.append((tag, float(v), step))})()
    agent.algo_observer.writer = agent.writer
    orig = agent.train_epoch

    def epoch():
        res = orig()
        stats.append(agent.last_stats.clone())
        return res
    agent.train_epoch = epoch
    agent.train()
    return [r for r in rows if r[0].startswith('diagnostics/')], stats


def _check_against_golden(g, diag, B, masked):
    want = [r for r in g['train_loop']['scalars'] if r[0].startswith('diagnostics/')]
    assert [(t, s) for t, _, s in diag] == [(t, s) for t, _, s in want]
    for (t, v, _), (_, rv, _) in zip(diag, want):
        if '/clip_frac/' in t:
            # neglogp rounding may flip a row at the clip threshold: at most one row per minibatch (masked: the value is frac / B)
            assert abs(v - rv) <= (1.0 / B) / (B if masked else 1) + 1e-7, (t, v, rv)
        elif math.isfinite(rv):
            assert v == pytest.approx(rv, rel=1e-4, abs=1e-7), (t, v, rv)
        else:
            assert (math.isnan(v) and math.isnan(rv)) or v == rv, (t, v, rv)


def _clip_aggregate(st, nmb, k, B, masked):
    """diagnostics/clip_frac/k from the stats rows' B200RL_STAT_CLIPFRAC column, as the reference aggregates it"""
    c = st[k * nmb:(k + 1) * nmb, 6]
    if masked:
        c = torch.where(st[k * nmb:(k + 1) * nmb, 5] > 0, c / B, torch.full_like(c, float('nan')))
    return float(c.mean())


@pytest.mark.parametrize('name', ['diag_mlp.pt', 'diag_masked_rmsadv.pt', 'diag_lstm.pt'])
def test_fp32_agent_writes_the_reference_diagnostics_with_and_without_cuda_graphs(name):
    res = {}
    for graph in (False, True):
        g, agent, (diag, stats) = _train_continuous(name, graph)
        assert agent.diag_on and not agent.use_tc
        masked = g['autoreset'] == 'next_step'
        _check_against_golden(g, diag, g['mb'], masked)
        nmb = agent.num_minibatches
        last = {t: v for t, v, s in diag if s == 2}
        for k in range(agent.mini_epochs_num):
            a, b = last[f'diagnostics/clip_frac/{k}'], _clip_aggregate(stats[-1], nmb, k, g['mb'], masked)
            assert a == b or (math.isnan(a) and math.isnan(b))
        res[graph] = diag
    assert [(t, s) for t, _, s in res[False]] == [(t, s) for t, _, s in res[True]]
    for (t, a, _), (_, b, _) in zip(res[False], res[True]):
        assert a == b or (math.isnan(a) and math.isnan(b)), t


def test_discrete_agent_writes_the_reference_diagnostics():
    from rl_games_b200.runner import Runner
    from test_discrete_gpu import DiscreteTapeEnvGPU
    g = torch.load(os.path.join(GOLDEN, 'diag_discrete.pt'), weights_only=False)
    env = DiscreteTapeEnvGPU(g)
    config = {k: v for k, v in g['config'].items() if k not in ('device', 'torch_compile')}
    config.update({'device': DEV, 'env_info': env.get_env_info(), 'vec_env': env, 'reward_shaper': {'scale_value': 0.1},
                   'train_dir': '/tmp/b200_parity_runs', 'lr_schedule': g['config'].get('lr_schedule', None)})
    network = {'name': 'actor_critic', 'separate': g['separate'], 'space': {'discrete': None},
               'mlp': {'units': g['units'], 'activation': 'relu', 'initializer': {'name': 'default'}}}
    r = Runner()
    r.load({'params': {'seed': 1, 'algo': {'name': 'a2c_discrete'}, 'model': {'name': 'discrete_a2c'}, 'network': network, 'config': config}})
    r.params['config']['vec_env'] = env
    agent = r.algo_factory.create(r.algo_name, base_name='parity', params=r.params)
    agent.model.load_state_dict({k: v.to(DEV) for k, v in g['init_state'].items()}, strict=False)
    agent.init_tensors()
    agent.obs = agent.env_reset()
    orig = agent.train_epoch
    agent.train_epoch = lambda: orig(u=g['u'][agent.epoch_num - 1].to(DEV))
    diag, _ = _run(agent)
    assert agent.diag_on
    _check_against_golden(g, diag, g['mb'], g['autoreset'] == 'next_step')


def _two_epochs(over, tc):
    """fused wgmma geometry (obs 60, MLP [256,128,64], 8 actions), next_step autoreset (masked rows)"""
    N, H, D, A, units, mb = 512, 8, 60, 8, [256, 128, 64], 2048
    obs_tape, done_tape, tout_tape = O.make_tapes(2 * H + 1, N, D, seed=34)
    noise = torch.randn(2, H, N, A, generator=torch.Generator().manual_seed(10)).to(DEV)
    a = make_agent({'mini_epochs': 2, 'mixed_precision': tc, **over}, N, H, D, A, units, mb,
                   TapeEnvGPU(obs_tape, done_tape, tout_tape, A, 'next_step'), O.init_params(D, units, A, seed=12))
    assert a.use_tc == tc
    out = []
    for ep in range(2):
        a.epoch_num += 1
        a.train_epoch(noise=noise[ep])
        out.append(a.last_stats.clone())
    torch.cuda.synchronize()
    return a, out


@pytest.mark.parametrize('tc', [False, True], ids=['fp32', 'fused-bf16'])
def test_diagnostics_are_observational_only(tc):
    """key on and off, same seeds: bit-identical weights, Adam state, arena and stats columns 0-8 after two epochs"""
    a, sa = _two_epochs({}, tc)
    b, sb = _two_epochs({'use_diagnostics': True}, tc)
    assert b.diag_on and not a.diag_on
    for x, y in zip(sa, sb):
        assert torch.equal(x[:, :9], y[:, :9])
        assert torch.isfinite(y[:, 9]).all() and torch.equal(x[:, 9], torch.zeros_like(x[:, 9]))
    for k in ('flat', 'exp_avg', 'exp_avg_sq'):
        assert torch.equal(getattr(a.model, k), getattr(b.model, k)), k
    for k in ('obses', 'actions', 'mus', 'sigmas', 'neglogpacs', 'values', 'rewards', 'advs_n', 'returns_n', 'old_values_n'):
        assert torch.equal(getattr(a, k), getattr(b, k)), k
    assert len(b.diagnostics.exp_vars) == 2 * b.n_updates          # replayed from the read-back rows; epoch() runs in train()


def test_fused_path_exp_var_equals_fp32_path_with_fp32_rollout():
    """b200_rollout_fp32: the tensor-core agent's first-epoch arena is bit-identical to the fp32 agent's, so is its explained variance"""
    N, H, D, A, units, mb = 512, 8, 60, 8, [256, 128, 64], 2048
    obs_tape, done_tape, tout_tape = O.make_tapes(H + 1, N, D, seed=33)
    params = O.init_params(D, units, A, seed=8)
    noise = torch.randn(H, N, A, generator=torch.Generator().manual_seed(9)).to(DEV)
    ev = {}
    for name, cfg in (('fp32', {'mixed_precision': False}), ('tc', {'mixed_precision': True, 'b200_rollout_fp32': True})):
        a = make_agent({'mini_epochs': 2, 'b200_cuda_graph': False, 'normalize_input': False, 'use_diagnostics': True, **cfg}, N, H, D, A,
                       units, mb, TapeEnvGPU(obs_tape, done_tape, tout_tape, A), params)
        a._rollout(noise)
        a._gae_and_prepare()
        torch.cuda.synchronize()
        assert a.use_tc == (name == 'tc')
        ev[name] = a.stats[:, 9].clone()
    assert torch.isfinite(ev['fp32']).all() and torch.equal(ev['fp32'], ev['tc'])
