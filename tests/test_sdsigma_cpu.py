"""State-dependent sigma heads (fixed_sigma: False) and the sigma parametrisations (models.py apply_sigma_parametrization) on the CPU:
the kernels' row function through the test-hook library against autograd, the agent's host logic on torch stand-ins against the
reference's golden runs, the parameter layout against the reference's, and what stays refused."""
import ctypes
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from tests import _hooks  # noqa: E402
from test_agent_host_cpu import _CudaLookingStr, _Env, _Event, _Stream  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')
SD_GOLDEN = ['agent_sdsigma.pt', 'agent_sdsigma_softplus.pt']
# fixed sigma in parametrisations mapped outside the kernels: softplus with a floor, exp clamped to logstd_bounds
FIXED_GOLDEN = ['agent_fixedsigma_softplus.pt', 'agent_fixedsigma_bounds.pt']

_CASES = [('exp', 0.0, None), ('exp', 0.0, (-1.0, 0.5)), ('exp', 0.15, None), ('exp', 0.2, (-2.0, 1.0)), ('softplus', 0.0, None),
          ('softplus', 0.2, None), ('linear', 0.0, None), ('linear', 0.2, None), ('scalar', 0.05, None)]


@pytest.mark.parametrize('param,min_sigma,bounds', _CASES)
def test_sigma_param_row_function_matches_autograd(param, min_sigma, bounds):
    import _torch_ops_sd as S
    from rl_games_b200 import ops
    lib = _hooks.load()
    fn = lib.b200rl_hosttest_sigma_param
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    g = torch.Generator().manual_seed(3)
    # around zero, both sides of (and exactly on) the clamp bounds, at the softplus threshold (20 + floor for 'linear')
    special = [-1.0, 0.5, -2.0, 1.0, -1.0001, 0.5001, 19.9, 20.0, 20.1, 20.2, 25.0, -30.0, 0.0]
    raw = torch.cat([torch.randn(500, generator=g) * 3, torch.tensor(special)]).contiguous()
    r = raw.clone().requires_grad_(True)
    sg_ref, ls_ref = S.apply_sigma(r, param, min_sigma, bounds)
    dls_ref, = torch.autograd.grad(ls_ref.sum(), r)
    n = raw.numel()
    sg, ls, dls = torch.zeros(n), torch.zeros(n), torch.zeros(n)
    cfg = ops.sigma_cfg(param, min_sigma, bounds)
    p = lambda t: ctypes.c_void_p(t.data_ptr())    # noqa: E731
    assert fn(p(raw), n, ctypes.addressof(cfg), p(sg), p(ls), p(dls)) == 0
    torch.testing.assert_close(sg, sg_ref.detach(), rtol=2e-6, atol=1e-7)
    torch.testing.assert_close(ls, ls_ref.detach(), rtol=2e-6, atol=1e-7)
    torch.testing.assert_close(dls, dls_ref, rtol=2e-6, atol=1e-7)
    if bounds is not None:        # clamp gradient: 1 on the closed interval, 0 outside
        assert (dls[(raw < bounds[0]) | (raw > bounds[1])] == 0).all()


def _network(units, space_over=None, network_over=None):
    network = {'name': 'actor_critic', 'separate': False,
               'space': {'continuous': {'mu_activation': 'None', 'sigma_activation': 'None', 'mu_init': {'name': 'default'},
                                        'sigma_init': {'name': 'const_initializer', 'val': 0}, 'fixed_sigma': True}},
               'mlp': {'units': list(units), 'activation': 'elu', 'initializer': {'name': 'default'}}}
    network['space']['continuous'].update(space_over or {})
    network.update(network_over or {})
    return network


def _standins(monkeypatch):
    import _torch_ops_sd
    _torch_ops_sd.install_sd(monkeypatch)       # the model's normalisers run on the stand-ins as well


def _sd_keys(n_layers):
    keys = [f'a2c_network.actor_mlp.{2 * i}.{t}' for i in range(n_layers) for t in ('weight', 'bias')]
    return keys + ['a2c_network.value.weight', 'a2c_network.value.bias', 'a2c_network.mu.weight', 'a2c_network.mu.bias',
                   'a2c_network.sigma.weight', 'a2c_network.sigma.bias']


@pytest.mark.parametrize('name', SD_GOLDEN)
def test_state_dict_and_adam_order_follow_the_reference(name, monkeypatch):
    from rl_games_b200.model import B200Model
    _standins(monkeypatch)
    g = torch.load(os.path.join(GOLDEN, name), weights_only=False)
    m = B200Model(_network(g['units'], g['space_over']), g['D'], g['A'], 'cpu', True, True)
    assert not m.a2c_network.fixed_sigma and m.head_rows == 1 + 2 * g['A']
    # parameter order = the reference's named_parameters() order (index keys of the torch Adam state)
    assert m.param_names() == g['param_order'] == _sd_keys(len(g['units']))
    m.load_state_dict(g['init_state'])
    sd = m.state_dict()
    assert 'a2c_network.sigma' not in sd
    for k in g['param_order']:
        assert torch.equal(sd[k], g['init_state'][k]), k
    assert sd['a2c_network.sigma.weight'].shape == (g['A'], g['units'][-1])
    assert torch.equal(m.sigma, torch.zeros(g['A']))           # the dead fixed-sigma block
    osd = m.optimizer_state_dict(3e-4, 1, 0.0)
    assert len(osd['state']) == len(g['param_order'])
    for i, k in enumerate(g['param_order']):
        assert osd['state'][i]['exp_avg'].shape == g['init_state'][k].shape


def test_state_dependent_initialisation_follows_init_state_dependent_sigma_head(monkeypatch):
    from rl_games_b200.model import B200Model
    _standins(monkeypatch)
    torch.manual_seed(0)
    const = B200Model(_network([16, 8], {'fixed_sigma': False, 'sigma_init': {'name': 'const_initializer', 'val': -1.05}}), 6, 3,
                      'cpu', True, True).state_dict()
    assert torch.equal(const['a2c_network.sigma.weight'], torch.zeros(3, 8))
    assert torch.equal(const['a2c_network.sigma.bias'], torch.full((3,), -1.05))
    dflt = B200Model(_network([16, 8], {'fixed_sigma': False, 'sigma_init': {'name': 'default'}}), 6, 3, 'cpu', True, True).state_dict()
    w = dflt['a2c_network.sigma.weight']
    assert w.abs().max() <= 1.0 / 8 ** 0.5 and w.abs().min() > 0          # torch.nn.Linear default init, fan-in 8
    assert torch.equal(dflt['a2c_network.sigma.bias'], torch.zeros(3))


@pytest.mark.parametrize('network_over,match', [({'separate': True}, 'state-dependent sigma with separate'),
                                                 ({'rnn': {'name': 'lstm', 'units': 8, 'layers': 1}}, 'state-dependent sigma with an rnn')])
def test_state_dependent_sigma_refusals(network_over, match, monkeypatch):
    from rl_games_b200.model import B200Model
    _standins(monkeypatch)
    with pytest.raises(NotImplementedError, match=match):
        B200Model(_network([16, 8], {'fixed_sigma': False}, network_over), 6, 3, 'cpu', True, True)


@pytest.mark.parametrize('param,min_sigma,bounds', [('softplus', 0.2, None), ('linear', 0.0, None), ('exp', 0.0, (-0.5, 0.3)),
                                                    ('exp', 0.1, (-0.5, 0.3))])
def test_fixed_sigma_parametrisations_map_the_log_std_the_kernels_read(param, min_sigma, bounds, monkeypatch):
    """fixed sigma, any parametrisation: the kernels read logstd_eff = log(sigma(raw)); sigma_chain = d logstd_eff / d raw"""
    import _torch_ops_sd as S
    from rl_games_b200.model import B200Model
    _standins(monkeypatch)
    over = {'sigma_parametrization': param, 'min_sigma': min_sigma}
    if bounds is not None:
        over['logstd_bounds'] = list(bounds)
    m = B200Model(_network([16, 8], over), 6, 5, 'cpu', True, True)
    assert m.sigma_transform and m.a2c_network.fixed_sigma
    m.sigma.copy_(torch.tensor([-1.0, -0.5, 0.0, 0.3, 0.9]))
    m.refresh_sigma_floor()
    r = m.sigma.clone().requires_grad_(True)
    _, ls = S.apply_sigma(r, param, min_sigma, bounds)
    d, = torch.autograd.grad(ls.sum(), r)
    torch.testing.assert_close(m.logstd_eff, ls.detach(), rtol=1e-6, atol=1e-7)
    torch.testing.assert_close(m.sigma_chain, d, rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize('name', SD_GOLDEN + FIXED_GOLDEN)
@pytest.mark.parametrize('mp', [False, True])
def test_state_dependent_agent_host_logic_matches_reference_golden(name, mp, monkeypatch, tmp_path):
    """fp32 (mp False) and layer-wise tensor-core (mp True) host composition, torch stand-ins for the kernels; the fixed-sigma
    fixtures drive the log-std mapping and its gradient chain (refresh_sigma_floor) through whole updates"""
    import _torch_ops
    import _torch_ops_sd
    from oracle import ppo_oracle as O
    from rl_games_b200.runner import Runner
    _torch_ops_sd.install_sd(monkeypatch)
    monkeypatch.setitem(_torch_ops._USE_HOST_SCHED, 'on', True)
    monkeypatch.setattr(torch.cuda, 'set_device', lambda d: None)
    monkeypatch.setattr(torch.cuda, 'Event', _Event)
    monkeypatch.setattr(torch.cuda, 'current_stream', lambda *a: _Stream())
    monkeypatch.setattr(torch.Tensor, 'pin_memory', lambda self: self)
    g = torch.load(os.path.join(GOLDEN, name), weights_only=False)
    cfgk = g['config']
    env = _Env(g)
    config = {k: v for k, v in cfgk.items() if k not in ('device', 'torch_compile')}
    config.update({'device': _CudaLookingStr('cpu'), 'env_info': env.get_env_info(), 'vec_env': env,
                   'reward_shaper': dict(g.get('reward_shaper') or {'scale_value': 1.0}), 'mixed_precision': mp, 'b200_cuda_graph': False,
                   'train_dir': str(tmp_path), 'lr_schedule': cfgk.get('lr_schedule', None)})
    r = Runner()
    r.load({'params': {'seed': 7, 'algo': {'name': 'a2c_continuous'}, 'model': {'name': 'continuous_a2c_logstd'},
                       'network': _network(g['units'], g['space_over']), 'config': config}})
    r.params['config']['vec_env'] = env
    agent = r.algo_factory.create(r.algo_name, base_name='parity', params=r.params)
    assert not agent.use_tc and agent.gemm_tc == mp          # never the fused kernels: they read the raw log-std / have 16 head rows
    sd_head = not g['space_over'].get('fixed_sigma', True)
    agent.model.load_state_dict(g['init_state'], strict=False)
    agent.init_tensors()
    agent._repack()
    agent.obs = agent.env_reset()
    fl = O.swap_and_flatten01
    for ep, ref in enumerate(g['epochs_out']):
        agent.epoch_num += 1
        agent.train_epoch(noise=g['noise'][ep])
        ds = ref['dataset']
        assert torch.equal(agent.dones_buf, ref['mb_dones'])
        torch.testing.assert_close(agent.values.unsqueeze(2), ref['mb_values'], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(fl(agent.advs_n), ds['advantages'], rtol=2e-4, atol=2e-5)
        torch.testing.assert_close(fl(agent.sigmas), ds['sigma'], rtol=1e-4, atol=1e-6)
        st = agent.last_stats
        torch.testing.assert_close(st[:, 0], ref['a_losses'], rtol=2e-3, atol=2e-6)
        torch.testing.assert_close(st[:, 1], ref['c_losses'], rtol=2e-3, atol=2e-6)
        torch.testing.assert_close(st[:, 2], ref['entropies'], rtol=1e-4, atol=1e-6)
        assert agent.last_lr == pytest.approx(ref['last_lr'], rel=1e-12)
        sd = agent.model.state_dict()
        for k in g['param_order']:
            torch.testing.assert_close(sd[k], ref['state'][k], rtol=1e-3, atol=1e-4, msg=lambda m: k + ': ' + m)
        if sd_head:
            assert torch.equal(agent.model.sigma, torch.zeros(g['A']))    # the dead fixed-sigma block never moves
    ck = agent.get_full_state_weights()
    for i, mref in enumerate(g['epochs_out'][-1]['adam_exp_avg']):
        torch.testing.assert_close(ck['optimizer']['state'][i]['exp_avg'].reshape(mref.shape), mref, rtol=1e-3, atol=1e-7)
