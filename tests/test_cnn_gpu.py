"""The conv trunk's kernels (rl_games_b200/csrc/conv.cu, moments_update_u8 in stats.cu) against fp64 torch, and the discrete agent with a
conv2d trunk against the reference's golden runs (tests/golden/gen_golden_cnn.py).

Each kernel is run on the Nature-CNN Atari geometry (4x84x84 -> 32@8/4 -> 64@4/2 -> 64@3/1) and on awkward ones (padding, stride 3,
channel counts that are not multiples of 4, output channels past one 64-wide tile, row counts that are not a multiple of the 128-row
tile), on uint8 and fp32 frames, NHWC and NCHW, with and without the normaliser, on chunked arena rows, into split partials; outputs are
NaN-filled beforehand, so that an element the kernel does not write fails."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
pytestmark = [pytest.mark.gpu]
DEV = 'cuda:0'
GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')

# (C, H, W, Cout, k, stride, pad)
NATURE = [(4, 84, 84, 32, 8, 4, 0), (32, 20, 20, 64, 4, 2, 0), (64, 9, 9, 64, 3, 1, 0)]
AWKWARD = [(3, 13, 11, 5, 3, 1, 1), (6, 17, 20, 7, 5, 3, 2), (5, 9, 9, 70, 3, 2, 0), (1, 6, 6, 3, 6, 1, 0)]
ACTS = {0: lambda x: x, 1: F.elu, 2: torch.relu, 3: torch.tanh}


def _act_grad(a, act):
    return {1: torch.where(a > 0, torch.ones_like(a), a + 1.0), 2: (a > 0).to(a.dtype), 3: 1.0 - a * a}.get(act, torch.ones_like(a))


def _arena(g, M, D, u8, rpc):
    """M rows in an arena of n_chunks chunks of rpc rows, chunk stride N = rpc + 3 (other rows hold junk)"""
    n_chunks, N = M // rpc, rpc + 3
    x = torch.randint(0, 256, (n_chunks, N, D), generator=g, dtype=torch.uint8) if u8 else torch.randn(n_chunks, N, D, generator=g) * 2
    rows = x[:, :rpc].reshape(M, D)
    return x, rows, N


def _ref_input(rows, geo, nhwc, norm):
    """the kernel's reading of the rows, in fp32 as the kernel computes it, then fp64"""
    C, H, W = geo[:3]
    v = rows.float() / 255.0 if rows.dtype == torch.uint8 else rows.float()
    if norm is not None:
        v = torch.clamp((v - norm[0]) / norm[1], -5.0, 5.0)
    v = v.double()
    return v.view(-1, H, W, C).permute(0, 3, 1, 2) if nhwc else v.view(-1, C, H, W)


def _case(geo, first, u8, nhwc, normed, M, rpc, act=1, seed=0):
    from rl_games_b200 import ops
    C, H, W, Cout, k, s, p = geo
    g = torch.Generator().manual_seed(seed)
    D = C * H * W
    if first:
        x, rows, N = _arena(g, M, D, u8, rpc)
    else:
        x, rows, N = None, torch.randn(M, D, generator=g), 0
    norm = (torch.rand(D, generator=g) * 0.5, torch.rand(D, generator=g) + 0.5) if normed else None
    Wt = torch.randn(Cout, C, k, k, generator=g) / (C * k * k) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.1
    xin = _ref_input(rows, geo, nhwc and first, norm).requires_grad_(True)
    Wd, bd = Wt.double().requires_grad_(True), b.double().requires_grad_(True)
    pre = F.conv2d(xin, Wd, bd, stride=s, padding=p)
    y_ref = ACTS[act](pre)
    dY = torch.randn(pre.shape, generator=g, dtype=torch.float64)
    pre.backward(dY)
    Ho, Wo = pre.shape[2:]
    d = lambda t: None if t is None else t.to(DEV)   # noqa: E731
    xd = d(x) if first else d(rows)
    nm, ns = (d(norm[0]), d(norm[1])) if normed else (None, None)
    chunk = dict(nhwc=nhwc, rows_per_chunk=rpc, chunk_stride=N, x_ld=D, norm_mean=nm, norm_std=ns) if first else {}
    geo5 = (C, H, W, s, p)
    Y = torch.full((M, Cout, Ho, Wo), float('nan'), device=DEV)
    ops.conv2d_fwd(xd, d(Wt), d(b), Y, geo5, act, M, **chunk)
    S, K = 3, C * k * k
    stride = Cout * K + Cout + 5
    part = torch.full((S, stride), float('nan'), device=DEV)
    ops.conv2d_bwd_weight(d(dY.float()), xd, part[0, :], part[0, Cout * K:], Wt.shape, geo5, S, M, stride, **chunk)
    out = {'Y': (Y, y_ref), 'dW': (part[:, :Cout * K].sum(0).view(Wt.shape), Wd.grad), 'db': (part[:, Cout * K:Cout * K + Cout].sum(0), bd.grad)}
    if not first:
        A_prev = F.elu(torch.randn(M, C, H, W, generator=g))
        dX = torch.full((M, C, H, W), float('nan'), device=DEV)
        ops.conv2d_bwd_data(d(dY.float()), d(Wt), d(A_prev), dX, geo5, 1, M)
        out['dX'] = (dX, xin.grad * _act_grad(A_prev.double(), 1))
    torch.cuda.synchronize()
    return out


def _check(out, rtol=1e-5):
    for name, (got, ref) in out.items():
        scale = ref.abs().max().item() + 1e-12
        err = (got.double().cpu() - ref).abs().max().item()
        assert err <= rtol * scale * 30, f'{name}: max error {err:.3e} at scale {scale:.3e}'


@pytest.mark.parametrize('u8,nhwc,normed', [(True, True, True), (True, False, False), (False, True, False), (False, False, True)])
def test_first_conv_layer_on_arena_frames_vs_fp64(u8, nhwc, normed):
    """layer 0 of the Nature CNN and of the awkward geometries on chunked arena rows"""
    for geo in [NATURE[0]] + AWKWARD:
        M = 21 if geo is NATURE[0] else 133
        _check(_case(geo, True, u8, nhwc, normed, M, rpc=7))


@pytest.mark.parametrize('geo', NATURE[1:] + AWKWARD)
@pytest.mark.parametrize('act', [0, 1, 2, 3])
def test_inner_conv_layers_vs_fp64(geo, act):
    """layers >= 1 on dense NCHW activations: forward, the data gradient with the activation derivative folded in, split weight gradients"""
    _check(_case(geo, False, False, False, False, 37 if geo[1] > 10 else 261, 0, act=act))


def test_repeat_is_bit_identical():
    a = _case(NATURE[1], False, False, False, False, 50, 0, seed=4)
    b = _case(NATURE[1], False, False, False, False, 50, 0, seed=4)
    for k in a:
        assert torch.equal(a[k][0], b[k][0]), k
    a = _case(NATURE[0], True, True, True, True, 14, 7, seed=5)
    b = _case(NATURE[0], True, True, True, True, 14, 7, seed=5)
    for k in a:
        assert torch.equal(a[k][0], b[k][0]), k


def test_bad_geometry_is_an_argument_error_and_writes_nothing():
    """a kernel that does not fit the padded input, stride 0, negative padding, a row stride shorter than a frame: B200RL_EINVAL"""
    from rl_games_b200 import ops
    from rl_games_b200._lib import ptr
    x = torch.zeros(2, 3 * 5 * 5, device=DEV)
    Wt = torch.zeros(4, 3, 7, 7, device=DEV)
    Y = torch.full((2, 4, 1, 1), float('nan'), device=DEV)
    s = torch.cuda.current_stream().cuda_stream
    for k, st, pad, ld in ((7, 1, 0, 75), (3, 0, 0, 75), (3, 1, -1, 75), (3, 1, 0, 74)):
        rc = ops.lib.b200rl_conv2d_fwd_f32(ptr(x), 0, 0, 2, 0, ld, None, None, ptr(Wt), None, ptr(Y), 2, 3, 5, 5, 4, k, k, st, pad, 0, s)
        assert rc == -1, (k, st, pad, ld, rc)
    torch.cuda.synchronize()
    assert torch.isnan(Y).all()


@pytest.mark.parametrize('D,rpc,n_chunks', [(4 * 84 * 84, 64, 4), (37, 5, 3), (1, 300, 1)])
def test_moments_update_u8_vs_fp64(D, rpc, n_chunks):
    from rl_games_b200 import ops
    g = torch.Generator().manual_seed(D)
    N = rpc + 2
    x = torch.randint(0, 256, (n_chunks, N, D), generator=g, dtype=torch.uint8)
    rows = x[:, :rpc].reshape(-1, D).double() / 255.0
    mean0, var0, cnt0 = torch.rand(D, generator=g, dtype=torch.float64), torch.rand(D, generator=g, dtype=torch.float64) + 0.1, 17
    n = rows.shape[0]
    bm, bv = rows.mean(0), rows.var(0, unbiased=False)
    tot = cnt0 + n
    delta = bm - mean0
    m_ref, v_ref = mean0 + delta * n / tot, (var0 * cnt0 + bv * n + delta ** 2 * cnt0 * n / tot) / tot
    mean, var, cnt = mean0.to(DEV), var0.to(DEV), torch.tensor([cnt0], dtype=torch.int64, device=DEV)
    mf, sf = torch.full((D,), float('nan'), device=DEV), torch.full((D,), float('nan'), device=DEV)
    ops.moments_update_u8(x.to(DEV), D, rpc, n_chunks, N, mean, var, cnt, mf, sf)
    torch.cuda.synchronize()
    torch.testing.assert_close(mean.cpu(), m_ref, rtol=1e-6, atol=1e-7)
    torch.testing.assert_close(var.cpu(), v_ref, rtol=1e-5, atol=1e-7)
    assert int(cnt.item()) == tot
    torch.testing.assert_close(mf.cpu(), m_ref.float(), rtol=1e-6, atol=1e-6)
    torch.testing.assert_close(sf.cpu(), torch.sqrt(v_ref.float() + 1e-5), rtol=1e-5, atol=1e-6)


class _FrameEnvGPU:
    def __init__(self, g):
        self.g, self.K, self.i = g, g['K'], 0
        self.obs_tape, self.done_tape, self.tout_tape = g['obs_tape'].to(DEV), g['done_tape'].to(DEV), g['timeout_tape'].to(DEV)
        self.mask_tape = g['mask_tape'].to(DEV) if g['mask_tape'] is not None else None

    def reset(self):
        self.i = 0
        return self.obs_tape[0].clone()

    def get_action_masks(self):
        return self.mask_tape[self.i % self.mask_tape.shape[0]]

    def step(self, actions):
        j0 = self.i % self.obs_tape.shape[0]
        rew = (actions.long() == self.obs_tape[j0].reshape(self.g['N'], -1)[:, :self.K].argmax(dim=-1)).float()
        self.i += 1
        j = self.i % self.obs_tape.shape[0]
        return self.obs_tape[j].clone(), rew, self.done_tape[j].clone(), {'time_outs': self.tout_tape[j].clone()}

    def get_env_info(self):
        from rl_games_b200.common import Box, Discrete
        return {'observation_space': Box(0, 255, tuple(self.obs_tape.shape[2:]), 'uint8'), 'action_space': Discrete(self.K)}


@pytest.mark.parametrize('name', ['agent_cnn_shared.pt', 'agent_cnn_separate.pt'])
def test_cnn_agent_matches_reference_golden(name):
    """two train_epoch()s of the reference DiscreteA2CAgent with a conv2d trunk on uint8 frames vs rl_games_b200's, at the tolerances of
    tests/test_discrete_gpu.py"""
    from rl_games_b200.runner import Runner
    from _cnn_frames import frame_tape
    g = torch.load(os.path.join(GOLDEN, name), weights_only=False)
    g['obs_tape'] = frame_tape(g['T'], g['N'], g['frame_shape'], g['seed'])
    env = _FrameEnvGPU(g)
    config = {k: v for k, v in g['config'].items() if k not in ('device', 'torch_compile')}
    config.update({'device': DEV, 'env_info': env.get_env_info(), 'vec_env': env, 'reward_shaper': {'scale_value': 0.1},
                   'train_dir': '/tmp/b200_parity_runs', 'lr_schedule': None})
    r = Runner()
    r.load({'params': {'seed': 1, 'algo': {'name': 'a2c_discrete'}, 'model': {'name': 'discrete_a2c'}, 'network': g['network'],
                       'config': config}})
    r.params['config']['vec_env'] = env
    agent = r.algo_factory.create(r.algo_name, base_name='parity', params=r.params)
    agent.model.load_state_dict({k: v.to(DEV) for k, v in g['init_state'].items()})
    assert agent.model.param_names() == g['param_order']
    agent.init_tensors()
    agent.obs = agent.env_reset()
    assert agent.obses.dtype == torch.uint8
    fl = lambda t: t.transpose(0, 1).reshape(-1, *t.shape[2:])    # noqa: E731
    for ep, ref in enumerate(g['epochs_out']):
        agent.epoch_num += 1
        res = agent.train_epoch(u=g['u'][ep].to(DEV))
        assert (agent.actions.cpu() == ref['mb_actions']).all()
        torch.testing.assert_close(agent.rewards.cpu().unsqueeze(2), ref['mb_rewards'], rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(agent.values.cpu().unsqueeze(2), ref['mb_values'], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(fl(agent.advs_n).cpu(), ref['advantages'], rtol=2e-4, atol=2e-5)
        torch.testing.assert_close(fl(agent.neglogpacs).cpu(), ref['old_logp_actions'], rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(torch.stack(res[4]).cpu(), ref['a_losses'], rtol=2e-3, atol=2e-6)
        torch.testing.assert_close(torch.stack(res[5]).cpu(), ref['c_losses'], rtol=2e-3, atol=2e-6)
        torch.testing.assert_close(torch.stack(res[6]).cpu(), ref['entropies'], rtol=1e-4, atol=1e-6)
        torch.testing.assert_close(torch.stack(res[7]).cpu(), ref['kls'], rtol=5e-3, atol=1e-8)
        sd = agent.model.state_dict()
        for k, v in ref['state'].items():
            torch.testing.assert_close(sd[k].cpu().reshape(v.shape).to(v.dtype), v, rtol=1e-3, atol=2e-5, msg=lambda m: k + ': ' + m)
