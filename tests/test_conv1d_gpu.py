"""The conv1d trunk's kernels (b200rl_conv1d_*: conv.cu's and conv_tc.cu's implicit GEMMs instantiated for one axis) against fp64, and
the discrete agent with a conv1d trunk against the reference's golden runs (tests/golden/gen_golden_conv1d.py).

Geometries are the smac frame-stack shapes: C = 4 stacked frames (and C = 14, a transposed stack's channel count) on L = 285 features
(27m_vs_30m: 4 move + 30 x 5 enemy + 26 x 5 ally + 1 own) and L = 156 (corridor: 4 + 24 x 5 + 5 x 6 + 2), the shipped stacks' filters
up to 1024, k3 s1 p1 ("same") and k3 s2 p1 (strided) first layers, k3 p0 inner layers.
- fp32: fp64 autograd on the same operands; every output within 2e-5 of its max-norm (only the fp32 summation order differs).
- tensor cores: fp64 autograd on the operands rounded to bf16 as the kernels stage them (input after the normaliser, dY, weights from the
  bf16 twin); every output within 1e-4 of its max-norm, the bound of tests/test_conv_tc_gpu.py.
Every output and partial buffer is NaN-filled before the call, so an element the kernel does not write fails."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
pytestmark = [pytest.mark.gpu]
DEV = 'cuda:0'
GOLDEN = os.path.join(HERE, 'golden')

# (C, L, Cout, k, stride, pad)
FIRST = [(4, 285, 256, 3, 1, 1), (4, 156, 64, 3, 2, 1), (14, 156, 64, 3, 2, 1), (14, 285, 256, 3, 1, 1), (3, 17, 5, 5, 3, 2)]
INNER = [(256, 285, 512, 3, 1, 1), (512, 285, 1024, 3, 1, 1), (64, 78, 128, 3, 1, 0), (128, 76, 256, 3, 1, 0), (7, 9, 70, 3, 2, 0)]
ACTS = {0: lambda x: x, 1: F.elu, 2: torch.relu, 3: torch.tanh}
TOL = {False: 2e-5, True: 1e-4}


def bf(t):
    return t.float().to(torch.bfloat16).double()


def _act_grad(a, act):
    return {1: torch.where(a > 0, torch.ones_like(a), a + 1.0), 2: (a > 0).to(a.dtype), 3: 1.0 - a * a}.get(act, torch.ones_like(a))


def _case(geo, first, normed, M, rpc, tc, act=2, seed=0, w_off=8):
    """one forward, weight gradient and (inner layers) data gradient of the kernels of one precision and of the fp64 reference; returns
    {name: (kernel output, reference)} and the kernels' outputs of a second identical call"""
    from rl_games_b200 import layerwise, ops
    C, L, Cout, k, s, p = geo
    g = torch.Generator().manual_seed(seed)
    D = C * L
    if first:          # M rows in an arena of M / rpc chunks, chunk stride rpc + 3 (the other rows hold junk)
        n_chunks, N = M // rpc, rpc + 3
        x = torch.randn(n_chunks, N, D, generator=g) * 2
        rows = x[:, :rpc].reshape(M, D)
    else:
        x, N = None, 0
        rows = torch.relu(torch.randn(M, D, generator=g))
    norm = (torch.rand(D, generator=g) * 0.5, torch.rand(D, generator=g) + 0.5) if normed else None
    Wt = torch.randn(Cout, C, k, generator=g) / (C * k) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.1
    flat = torch.zeros(w_off + Wt.numel() + 5, device=DEV)
    Wv = flat[w_off:w_off + Wt.numel()].view(Wt.shape)
    Wv.copy_(Wt)
    arena = (flat, flat.to(torch.bfloat16))
    rnd = bf if tc else (lambda t: t.double())
    v = rows.float()
    if norm is not None:
        v = torch.clamp((v - norm[0]) / norm[1], -5.0, 5.0)
    xin = rnd(v).to(DEV).view(-1, C, L).requires_grad_(True)
    Wd = rnd(Wt).to(DEV).requires_grad_(True)
    bd = b.double().to(DEV).requires_grad_(True)
    pre = F.conv1d(xin, Wd, bd, stride=s, padding=p)
    y_ref = ACTS[act](pre)
    dY = torch.randn(pre.shape, generator=g).to(DEV)
    pre.backward(rnd(dY.cpu()).to(DEV))
    Lo = pre.shape[2]
    xd = (x if first else rows).to(DEV)
    nm, ns = (norm[0].to(DEV), norm[1].to(DEV)) if normed else (None, None)
    chunk = dict(rows_per_chunk=rpc, chunk_stride=N, x_ld=D, norm_mean=nm, norm_std=ns) if first else {}
    geo4 = (C, L, s, p)
    k_ = layerwise.Kernels(tc=tc, bf16_arena=arena if tc else None)
    # the agent's split rule over the output positions, at least 3 splits (some of them empty on the small geometries)
    S, K = max(3, layerwise.n_splits(M * Lo)), C * k
    stride = Cout * K + Cout + 5
    A_prev = torch.relu(torch.randn(M, C, L, generator=g)).to(DEV)

    def run():
        Y = torch.full((M, Cout, Lo), float('nan'), device=DEV)
        k_.conv1d_fwd(xd, Wv, b.to(DEV), Y, geo4, act, M, **chunk)
        part = torch.full((S, stride), float('nan'), device=DEV)
        k_.conv1d_bwd_weight(dY, xd, part[0, :], part[0, Cout * K:], Wt.shape, geo4, S, M, stride, **chunk)
        out = {'Y': Y, 'dW': part[:, :Cout * K].sum(0).view(Wt.shape), 'db': part[:, Cout * K:Cout * K + Cout].sum(0)}
        if not first:
            dX = torch.full((M, C, L), float('nan'), device=DEV)
            k_.conv1d_bwd_data(dY, Wv, A_prev, dX, geo4, 2, M)
            out['dX'] = dX
        torch.cuda.synchronize()
        return out
    got, again = run(), run()
    ref = {'Y': y_ref.detach(), 'dW': Wd.grad, 'db': bd.grad}
    if not first:
        ref['dX'] = xin.grad * _act_grad(A_prev.double(), 2)
    return {n: (got[n], ref[n]) for n in got}, again


def _check(out, tc, what):
    for name, (got, ref) in out.items():
        scale = ref.abs().max().item() + 1e-12
        err = (got.double() - ref).abs().max().item()
        assert err <= TOL[tc] * scale, f'{what} {name}: max error {err:.3e} at scale {scale:.3e}'


def _same(out, again, what):
    for name, (got, _) in out.items():
        assert torch.equal(got, again[name]), f'{what} {name}: a repeated call differs'


@pytest.mark.parametrize('tc', [False, True])
@pytest.mark.parametrize('normed', [False, True])
@pytest.mark.parametrize('geo', FIRST)
def test_first_conv1d_layer_on_arena_rows_vs_fp64(geo, normed, tc):
    """layer 0 on chunked arena rows (the short C*k reduction of 12 or 42), with and without the input normaliser; repeated calls are
    bit-identical"""
    M, rpc = (1024, 64) if geo[1] > 100 else (133, 7)
    out, again = _case(geo, True, normed, M, rpc, tc, w_off=3)        # odd offset: unaligned twin rows
    _check(out, tc, geo)
    _same(out, again, geo)


@pytest.mark.parametrize('w_off', [5, 8])
@pytest.mark.parametrize('tc', [False, True])
@pytest.mark.parametrize('geo', INNER)
def test_inner_conv1d_layers_vs_fp64(geo, tc, w_off):
    """layers >= 1 on dense [M, C, L] activations: forward, the data gradient with the activation derivative folded in, split weight
    gradients; repeated calls are bit-identical.  w_off = 8 puts the filters 16-byte aligned in the bf16 twin, so the tensor-core forward
    reads them with its vector loader wherever C * k is a multiple of 8; w_off = 5 takes the scalar loader"""
    M = 96 if geo[0] >= 256 else 261
    out, again = _case(geo, False, False, M, 0, tc, act=2 if geo[0] > 8 else 1, w_off=w_off)
    _check(out, tc, geo)
    _same(out, again, geo)


# ------------------------------------------------------------------------------------------------------- the agent against the goldens
def _agent(g, over=None):
    import test_conv1d_cpu as C1
    return C1.make_agent(g, '/tmp/b200_conv1d_runs', over, device=DEV)


def _golden(name):
    g = torch.load(os.path.join(GOLDEN, name), weights_only=False)
    for key in ('obs_tape', 'done_tape', 'timeout_tape', 'mask_tape'):
        if g[key] is not None:
            g[key] = g[key].to(DEV)
    return g


@pytest.mark.parametrize('name', ['agent_conv1d_separate.pt', 'agent_conv1d_shared.pt'])
def test_conv1d_agent_on_fp32_kernels_matches_reference_golden(name):
    """two train_epoch()s of the reference DiscreteA2CAgent with a conv1d trunk vs rl_games_b200's fp32 kernels, at the tolerances of
    tests/test_cnn_gpu.py"""
    g = _golden(name)
    agent = _agent(g)
    fl = lambda t: t.transpose(0, 1).reshape(-1, *t.shape[2:]).cpu()    # noqa: E731
    for ep, ref in enumerate(g['epochs_out']):
        agent.epoch_num += 1
        res = agent.train_epoch(u=g['u'][ep].to(DEV))
        assert (agent.actions.cpu() == ref['mb_actions']).all()
        torch.testing.assert_close(agent.rewards.cpu().unsqueeze(2), ref['mb_rewards'], rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(agent.values.cpu().unsqueeze(2), ref['mb_values'], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(fl(agent.advs_n), ref['advantages'], rtol=2e-4, atol=2e-5)
        torch.testing.assert_close(fl(agent.neglogpacs), ref['old_logp_actions'], rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(torch.stack(res[4]).cpu(), ref['a_losses'], rtol=2e-3, atol=2e-6)
        torch.testing.assert_close(torch.stack(res[5]).cpu(), ref['c_losses'], rtol=2e-3, atol=2e-6)
        torch.testing.assert_close(torch.stack(res[6]).cpu(), ref['entropies'], rtol=1e-4, atol=1e-6)
        torch.testing.assert_close(torch.stack(res[7]).cpu(), ref['kls'], rtol=5e-3, atol=1e-8)
        sd = agent.model.state_dict()
        for k, v in ref['state'].items():
            torch.testing.assert_close(sd[k].cpu().reshape(v.shape).to(v.dtype), v, rtol=1e-3, atol=2e-5, msg=lambda m: k + ': ' + m)


# the tensor-core agent's bounds against the fp32 golden: the conv2d tensor-core agent's (tests/test_conv_tc_cpu.py LOOSE), except the
# weights after the epoch's Adam steps.  Adam divides each gradient element by its own running scale, so bf16 noise on a near-zero
# gradient element becomes a step of up to the learning rate; on an H100 the separate-trunk run's first MLP layer ends 2.8e-2 of its
# max-norm away from the fp32 reference's
LOOSE_STATE = 5e-2


def _near_fp32_golden(agent, g, res, ep):
    import test_conv_tc_cpu as TC
    ref = g['epochs_out'][ep]
    fl = lambda t: t.transpose(0, 1).reshape(-1, *t.shape[2:]).cpu()    # noqa: E731
    assert torch.equal(agent.actions.cpu(), ref['mb_actions'])
    got = {'rewards': (agent.rewards.cpu().unsqueeze(2), ref['mb_rewards']), 'values': (agent.values.cpu().unsqueeze(2), ref['mb_values']),
           'advantages': (fl(agent.advs_n), ref['advantages']), 'old_logp_actions': (fl(agent.neglogpacs), ref['old_logp_actions'])}
    for i, key in ((4, 'a_losses'), (5, 'c_losses'), (6, 'entropies')):
        got[key] = (torch.stack(res[i]).cpu(), ref[key])
    for key, (a, r) in got.items():
        assert TC.max_norm_err(a, r) <= TC.LOOSE[key], (key, TC.max_norm_err(a, r))
    sd = agent.model.state_dict()
    for k, v in ref['state'].items():
        err = TC.max_norm_err(sd[k].cpu().reshape(v.shape), v)
        assert err <= LOOSE_STATE, (k, err)


@pytest.mark.parametrize('name', ['agent_conv1d_separate.pt', 'agent_conv1d_shared.pt'])
def test_conv1d_agent_with_mixed_precision_stays_near_the_fp32_golden(name):
    """the tensor-core agent over the first recorded epoch: the same actions, every recorded quantity within the conv2d tensor-core
    agent's max-norm bounds and the weights within LOOSE_STATE"""
    g = _golden(name)
    agent = _agent(g, {'mixed_precision': True})
    assert agent.wbf is not None
    agent.epoch_num += 1
    res = agent.train_epoch(u=g['u'][0].to(DEV))
    _near_fp32_golden(agent, g, res, 0)


@pytest.mark.parametrize('arm', ['fp32', 'bf16'])
def test_conv1d_player_matches_the_reference_player(arm, tmp_path):
    """the package's PpoPlayerDiscrete (CUDA graph on) replaying the reference player's recorded play (tests/golden/conv1d_player_disc.pt):
    argmax exact on rows with a clear margin, the normalised masked logits within 1e-5 (fp32) or the bf16 bound of
    tests/test_players_gpu.py"""
    import test_conv1d_cpu as C1
    from test_players_gpu import BF16_ATOL, BF16_RTOL
    fx = torch.load(C1.PLAYER_FIXTURE, weights_only=False)
    p = C1.fixture_player(fx, {'mixed_precision': arm == 'bf16'}, tmp_path, device=DEV)
    assert (p.wbf is not None) == (arm == 'bf16')
    atol, rtol = (1e-5, 0.0) if arm == 'fp32' else (BF16_ATOL, BF16_RTOL)
    C1.replay_player(p, fx, DEV, atol=atol, rtol=rtol)
