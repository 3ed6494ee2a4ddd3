"""The tensor-core convolutions (rl_games_b200/csrc/conv_tc.cu) against fp64 autograd, and the discrete agent with
``mixed_precision: True`` against a kernel-faithful torch model of the same runs and against the recorded fp32 reference runs.

The fp64 reference takes the operands the kernels stage, rounded to bf16 the same way: the input after the 1/255 scaling and the
normaliser (computed in fp32, as the kernel does), dY, and the weights from the bf16 twin of the parameter arena.  What is left is
the order of the fp32 accumulation, so every output must agree to 1e-4 of its max-norm: a layout or indexing error cannot pass.  Each
output and partial buffer is NaN-filled before the call, so an element the kernel does not write fails."""
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

# (C, H, W, Cout, k, stride, pad)
NATURE = [(4, 84, 84, 32, 8, 4, 0), (32, 20, 20, 64, 4, 2, 0), (64, 9, 9, 64, 3, 1, 0)]
AWKWARD = [(1, 36, 36, 16, 5, 3, 2), (3, 36, 36, 48, 8, 4, 0), (3, 13, 11, 96, 3, 1, 1), (5, 9, 9, 70, 3, 2, 0), (1, 6, 6, 3, 6, 1, 0)]
ACTS = {0: lambda x: x, 1: F.elu, 2: torch.relu, 3: torch.tanh}
TOL = 1e-4


def bf(t):
    return t.float().to(torch.bfloat16).double()


def _act_grad(a, act):
    return {1: torch.where(a > 0, torch.ones_like(a), a + 1.0), 2: (a > 0).to(a.dtype), 3: 1.0 - a * a}.get(act, torch.ones_like(a))


def _case(geo, first, u8, nhwc, normed, M, rpc, act=1, seed=0, w_off=8):
    """one forward, weight gradient and (layers >= 1) data gradient of the tensor-core kernels and of the fp64 reference"""
    from rl_games_b200 import layerwise, ops
    C, H, W, Cout, k, s, p = geo
    g = torch.Generator().manual_seed(seed)
    D = C * H * W
    if first:          # M rows in an arena of M / rpc chunks, chunk stride rpc + 3 (the other rows hold junk)
        n_chunks, N = M // rpc, rpc + 3
        x = torch.randint(0, 256, (n_chunks, N, D), generator=g, dtype=torch.uint8) if u8 else torch.randn(n_chunks, N, D, generator=g) * 2
        rows = x[:, :rpc].reshape(M, D)
    else:
        x, N = None, 0
        rows = torch.randn(M, D, generator=g)
    norm = (torch.rand(D, generator=g) * 0.5, torch.rand(D, generator=g) + 0.5) if normed else None
    # the filters live in an fp32 arena at offset w_off, the kernels read them from its bf16 twin
    Wt = torch.randn(Cout, C, k, k, generator=g) / (C * k * k) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.1
    flat = torch.zeros(w_off + Wt.numel() + 5, device=DEV)
    Wv = flat[w_off:w_off + Wt.numel()].view(Wt.shape)
    Wv.copy_(Wt)
    fb = flat.to(torch.bfloat16)
    arena = (flat, fb)
    # the reference: the kernel's fp32 reading of the input, rounded to bf16, then fp64 on the device
    v = rows.float() / 255.0 if rows.dtype == torch.uint8 else rows.float()
    if norm is not None:
        v = torch.clamp((v - norm[0]) / norm[1], -5.0, 5.0)
    v = bf(v).to(DEV)
    xin = (v.view(-1, H, W, C).permute(0, 3, 1, 2) if nhwc and first else v.view(-1, C, H, W)).requires_grad_(True)
    Wd = bf(Wt).to(DEV).requires_grad_(True)
    bd = b.double().to(DEV).requires_grad_(True)
    pre = F.conv2d(xin, Wd, bd, stride=s, padding=p)
    y_ref = ACTS[act](pre)
    dY = torch.randn(pre.shape, generator=g).to(DEV)
    pre.backward(bf(dY))
    Ho, Wo = pre.shape[2:]
    xd = (x if first else rows).to(DEV)
    nm, ns = (norm[0].to(DEV), norm[1].to(DEV)) if normed else (None, None)
    chunk = dict(nhwc=nhwc, rows_per_chunk=rpc, chunk_stride=N, x_ld=D, norm_mean=nm, norm_std=ns) if first else {}
    geo5 = (C, H, W, s, p)
    Y = torch.full((M, Cout, Ho, Wo), float('nan'), device=DEV)
    ops.conv2d_fwd_tc(xd, Wv, b.to(DEV), Y, geo5, act, M, bf16_arena=arena, **chunk)
    # the agent's split rule: a split sums at most ~M*Ho*Wo / 64 output pixels (the tensor cores' fp32 accumulation over one split is
    # what the tolerance allows for); at least 3 splits, some of them empty on the small geometries
    S, K = max(3, layerwise.n_splits(M * Ho * Wo)), C * k * k
    stride = Cout * K + Cout + 5
    part = torch.full((S, stride), float('nan'), device=DEV)
    ops.conv2d_bwd_weight_tc(dY, xd, part[0, :], part[0, Cout * K:], Wt.shape, geo5, S, M, stride, **chunk)
    out = {'Y': (Y, y_ref.detach()), 'dW': (part[:, :Cout * K].sum(0).view(Wt.shape), Wd.grad),
           'db': (part[:, Cout * K:Cout * K + Cout].sum(0), bd.grad)}
    if not first:
        A_prev = F.elu(torch.randn(M, C, H, W, generator=g)).to(DEV)
        dX = torch.full((M, C, H, W), float('nan'), device=DEV)
        ops.conv2d_bwd_data_tc(dY, Wv, A_prev, dX, geo5, 1, M, bf16_arena=arena)
        out['dX'] = (dX, xin.grad * _act_grad(A_prev.double(), 1))
    torch.cuda.synchronize()
    return out


def _check(out, what):
    for name, (got, ref) in out.items():
        scale = ref.abs().max().item() + 1e-12
        err = (got.double() - ref).abs().max().item()
        assert err <= TOL * scale, f'{what} {name}: max error {err:.3e} at scale {scale:.3e}'


@pytest.mark.parametrize('u8,nhwc,normed', [(True, True, True), (True, True, False), (True, False, True), (True, False, False),
                                            (False, True, False), (False, False, True)])
def test_first_conv_layer_on_arena_frames_vs_fp64(u8, nhwc, normed):
    """layer 0 of the Nature CNN at minibatch 2048 and of the awkward geometries, on chunked arena rows"""
    _check(_case(NATURE[0], True, u8, nhwc, normed, 2048, rpc=64), 'nature')
    for i, geo in enumerate(AWKWARD):
        _check(_case(geo, True, u8, nhwc, normed, 133, rpc=7, w_off=3 + i), geo)       # odd offsets: unaligned twin rows


@pytest.mark.parametrize('geo', NATURE[1:])
def test_inner_nature_layers_at_minibatch_2048_vs_fp64(geo):
    _check(_case(geo, False, False, False, False, 2048, 0, act=1), geo)


@pytest.mark.parametrize('geo', AWKWARD)
@pytest.mark.parametrize('act', [0, 1, 2, 3])
def test_inner_conv_layers_vs_fp64(geo, act):
    """layers >= 1 on dense NCHW activations: forward, the data gradient with the activation derivative folded in, split weight gradients"""
    _check(_case(geo, False, False, False, False, 37 if geo[1] > 10 else 261, 0, act=act, w_off=5), geo)


def test_repeat_is_bit_identical():
    for args in ((NATURE[1], False, False, False, False, 300, 0), (NATURE[0], True, True, True, True, 130, 13)):
        a, b = _case(*args, seed=4), _case(*args, seed=4)
        for k in a:
            assert torch.equal(a[k][0], b[k][0]), k


def test_missing_twin_or_bad_geometry_is_an_argument_error_and_writes_nothing():
    from rl_games_b200 import ops
    from rl_games_b200._lib import ptr
    x = torch.zeros(2, 3 * 5 * 5, device=DEV)
    wb = torch.zeros(4 * 3 * 3 * 3, dtype=torch.bfloat16, device=DEV)
    Y = torch.full((2, 4, 3, 3), float('nan'), device=DEV)
    s = torch.cuda.current_stream().cuda_stream
    for w, k, st, ld in ((None, 3, 1, 75), (wb, 7, 1, 75), (wb, 3, 0, 75), (wb, 3, 1, 74)):
        rc = ops.lib.b200rl_conv2d_fwd_tc(ptr(x), 0, 0, 2, 0, ld, None, None, None if w is None else ptr(w), None, ptr(Y), 2, 3, 5, 5, 4,
                                          k, k, st, 0, 0, s)
        assert rc == -1, (k, st, ld, rc)
    torch.cuda.synchronize()
    assert torch.isnan(Y).all()


# ------------------------------------------------------------------------------------------------------------------- agent level
# the kernels against the kernel-faithful model (tests/_torch_ops_conv_tc.py) of the same epoch from the same state: only the fp32
# summation order differs, which now and then moves the bf16 rounding of one operand of a later layer by one bf16 ulp.  One such flip
# feeding the head moves a value by ~1e-3 of the largest value (measured on an H100: up to 2.9e-3 on the shared-trunk golden, up to
# 6e-4 on the others), so the model's state is re-synchronised from the kernels' after every epoch and TIGHT sits between one flip and
# the bf16-vs-fp32 bounds
TIGHT = 5e-3


def _max_norm_err(got, ref):
    return (got.double().cpu() - ref.double().cpu()).abs().max().item() / (ref.double().abs().max().item() + 1e-12)


def _compare_runs(a, b, res_a, res_b):
    assert torch.equal(a.actions, b.actions)
    for name, x, y in (('values', a.values, b.values), ('neglogpacs', a.neglogpacs, b.neglogpacs), ('advs', a.advs_n, b.advs_n),
                       ('a_losses', torch.stack(res_a[4]), torch.stack(res_b[4])), ('c_losses', torch.stack(res_a[5]), torch.stack(res_b[5])),
                       ('entropies', torch.stack(res_a[6]), torch.stack(res_b[6])), ('flat', a.model.flat, b.model.flat)):
        e = _max_norm_err(x, y)
        print(f'{name}: {e:.2e}')
        assert e <= TIGHT, (name, e)
    assert torch.equal(a.wbf, a.model.flat.to(torch.bfloat16))


def _cnn_agent(g, over):
    from rl_games_b200.runner import Runner
    from test_cnn_gpu import _FrameEnvGPU
    env = _FrameEnvGPU(g)
    config = {k: v for k, v in g['config'].items() if k not in ('device', 'torch_compile')}
    config.update({'device': DEV, 'env_info': env.get_env_info(), 'vec_env': env, 'reward_shaper': {'scale_value': 0.1},
                   'train_dir': '/tmp/b200_parity_runs', 'lr_schedule': None})
    config.update(over)
    r = Runner()
    r.load({'params': {'seed': 1, 'algo': {'name': 'a2c_discrete'}, 'model': {'name': 'discrete_a2c'}, 'network': g['network'],
                       'config': config}})
    r.params['config']['vec_env'] = env
    agent = r.algo_factory.create(r.algo_name, base_name='parity', params=r.params)
    agent.model.load_state_dict({k: v.to(DEV) for k, v in g['init_state'].items()})
    agent.init_tensors()
    agent.obs = agent.env_reset()
    return agent


@pytest.mark.parametrize('name', ['agent_cnn_shared.pt', 'agent_cnn_separate.pt'])
def test_cnn_agent_with_mixed_precision_matches_its_model_and_stays_near_the_fp32_golden(name):
    import _torch_ops_conv_tc
    from _cnn_frames import frame_tape
    from test_conv_tc_cpu import check_against_fp32_golden
    g = torch.load(os.path.join(GOLDEN, name), weights_only=False)
    g['obs_tape'] = frame_tape(g['T'], g['N'], g['frame_shape'], g['seed'])
    mp = pytest.MonkeyPatch()
    try:
        a = _cnn_agent(g, {'mixed_precision': True})
        _torch_ops_conv_tc.install_tc_only(mp)          # the model: torch for the tensor-core entry points, kernels for the rest
        b = _cnn_agent(g, {'mixed_precision': True})
        for ep in range(len(g['epochs_out'])):
            a.epoch_num += 1
            b.epoch_num += 1
            res_a = a.train_epoch(u=g['u'][ep].to(DEV))
            res_b = b.train_epoch(u=g['u'][ep].to(DEV))
            _compare_runs(a, b, res_a, res_b)
            check_against_fp32_golden(a, g, res_a, ep, cpu=lambda t: t.cpu())
            b.set_full_state_weights(a.get_full_state_weights(), set_epoch=False)
    finally:
        mp.undo()


def test_mlp_agent_with_masks_and_mixed_precision_matches_its_model():
    """an MLP-only golden run with action masks (tests/test_discrete_gpu.py) on the layer-wise tensor-core GEMMs"""
    import _torch_ops_conv_tc
    from rl_games_b200.runner import Runner
    from test_discrete_gpu import DiscreteTapeEnvGPU
    mp = pytest.MonkeyPatch()
    g = torch.load(os.path.join(GOLDEN, 'agent_discrete_masked.pt'), weights_only=False)

    def make():
        env = DiscreteTapeEnvGPU(g)
        config = {k: v for k, v in g['config'].items() if k not in ('device', 'torch_compile')}
        config.update({'device': DEV, 'env_info': env.get_env_info(), 'vec_env': env, 'reward_shaper': {'scale_value': 0.1},
                       'train_dir': '/tmp/b200_parity_runs', 'lr_schedule': g['config'].get('lr_schedule', None), 'mixed_precision': True})
        network = {'name': 'actor_critic', 'separate': g['separate'], 'space': {'discrete': None},
                   'mlp': {'units': g['units'], 'activation': 'relu', 'initializer': {'name': 'default'}}}
        r = Runner()
        r.load({'params': {'seed': 1, 'algo': {'name': 'a2c_discrete'}, 'model': {'name': 'discrete_a2c'}, 'network': network,
                           'config': config}})
        r.params['config']['vec_env'] = env
        agent = r.algo_factory.create(r.algo_name, base_name='parity', params=r.params)
        agent.model.load_state_dict({k: v.to(DEV) for k, v in g['init_state'].items()}, strict=False)
        agent.init_tensors()
        agent.obs = agent.env_reset()
        return agent
    try:
        a = make()
        _torch_ops_conv_tc.install_tc_only(mp)
        b = make()
        fl = lambda t: t.transpose(0, 1).reshape(-1, *t.shape[2:])    # noqa: E731
        for ep, ref in enumerate(g['epochs_out']):
            a.epoch_num += 1
            b.epoch_num += 1
            res_a = a.train_epoch(u=g['u'][ep].to(DEV))
            res_b = b.train_epoch(u=g['u'][ep].to(DEV))
            _compare_runs(a, b, res_a, res_b)
            b.set_full_state_weights(a.get_full_state_weights(), set_epoch=False)
            # and near the recorded fp32 reference
            assert (a.actions.cpu() == ref['mb_actions']).all()
            assert _max_norm_err(a.values.unsqueeze(2), ref['mb_values']) <= 2e-2
            assert _max_norm_err(fl(a.neglogpacs), ref['dataset']['old_logp_actions']) <= 1e-2
            sd = a.model.state_dict()
            for k in g['param_order']:
                assert _max_norm_err(sd[k], ref['state'][k]) <= 2e-2, k
    finally:
        mp.undo()
