"""Layer-normed LSTM policies (rnn.layer_norm: True) on the CPU: the test-side oracle against the reference's golden runs, the model's
layout / keys / order / initialisation against the reference's, checkpoints both ways, the agent's host logic on torch stand-ins
against the golden runs, a stock YAML with a layer-normed LSTM through the reference's own Runner, and what stays refused."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import _lstm_ln_oracle as LO  # noqa: E402
from test_agent_host_cpu import _CudaLookingStr, _Env, _Event, _Stream  # noqa: E402
from test_oracle_vs_golden import _oracle_from_golden  # noqa: E402

GOLDEN = os.path.join(HERE, 'golden')
LN_GOLDEN = ['agent_lstm_ln.pt', 'agent_lstm_ln_after.pt', 'agent_lstm_ln_after_masked.pt']
ROOT = os.path.dirname(HERE)
REF = os.path.join(ROOT, 'oracle', '_ref')
_need_ref = pytest.mark.skipif(not os.path.isdir(os.path.join(REF, 'rl_games')), reason='reference rl_games not present (oracle/_ref)')


def _load(name):
    g = torch.load(os.path.join(GOLDEN, name), weights_only=False)
    assert g['rnn_layer_norm'] is True
    return g


def _network(units, rnn_units, before_mlp, layer_norm=True, **rnn_over):
    rnn = {'name': 'lstm', 'units': rnn_units, 'layers': 1, 'before_mlp': before_mlp, 'layer_norm': layer_norm, **rnn_over}
    return {'name': 'actor_critic', 'separate': False,
            'space': {'continuous': {'mu_activation': 'None', 'sigma_activation': 'None', 'mu_init': {'name': 'default'},
                                     'sigma_init': {'name': 'const_initializer', 'val': 0}, 'fixed_sigma': True}},
            'mlp': {'units': list(units), 'activation': 'elu', 'initializer': {'name': 'default'}}, 'rnn': rnn}


@pytest.mark.parametrize('name', LN_GOLDEN)
def test_oracle_reproduces_reference_golden(name):
    """two full train_epoch()s of the reference with a layer-normed LSTM vs the test-side oracle, same tapes / noise"""
    g = _load(name)
    assert g['param_order'] == LO.param_names(len(g['units']))
    ag = _oracle_from_golden(g)
    ag = LO.make_agent(ag.env, {k: v for k, v in g['init_state'].items() if k.startswith('a2c_network')}, g['D'], g['A'], g['units'],
                       g['N'], g['H'], g['mb'], ag.cfg)
    ag.obs = ag.env_reset()
    for ep, ref in enumerate(g['epochs_out']):
        out = ag.train_epoch(g['noise'][ep])
        ds = ref['dataset']
        assert torch.equal(ag.buf['dones'], ref['mb_dones'])
        torch.testing.assert_close(ag.buf['values'], ref['mb_values'], rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(ag.dataset['advantages'], ds['advantages'], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(torch.stack(out['a_loss']), ref['a_losses'], rtol=1e-3, atol=1e-6)
        torch.testing.assert_close(torch.stack(out['c_loss']), ref['c_losses'], rtol=1e-3, atol=1e-6)
        assert ag.last_lr == pytest.approx(ref['last_lr'], rel=1e-12)
        for k in g['param_order']:
            torch.testing.assert_close(ag.model.p[k].detach(), ref['state'][k], rtol=1e-4, atol=2e-6, msg=lambda m: k + m)


def _standins(monkeypatch):
    import _torch_ops_ln
    _torch_ops_ln.install_ln(monkeypatch)       # the model's normalisers run on the stand-ins as well


@pytest.mark.parametrize('name', LN_GOLDEN)
def test_layout_keys_order_and_init_follow_the_reference(name, monkeypatch):
    from rl_games_b200.model import B200Model
    _standins(monkeypatch)
    g = _load(name)
    Hd = g['rnn_units']
    torch.manual_seed(0)
    m = B200Model(_network(g['units'], Hd, g['rnn_before_mlp']), g['D'], g['A'], 'cpu', True, True)
    assert m.rnn_layer_norm and m.ln_w.shape == (Hd,) and m.ln_b.shape == (Hd,)
    for n in ('ln_w', 'ln_b'):
        assert m.layout[n][0] % 8 == 0
    # torch.nn.LayerNorm's own initialisation (the mlp initializer does not touch it)
    assert torch.equal(m.ln_w, torch.ones(Hd)) and torch.equal(m.ln_b, torch.zeros(Hd))
    # parameter order = the reference's named_parameters() order (index keys of the torch Adam state)
    assert m.param_names() == g['param_order']
    m.load_state_dict(g['init_state'])
    sd = m.state_dict()
    for k in g['param_order']:
        assert torch.equal(sd[k], g['init_state'][k]), k
    assert torch.equal(m.ln_b, g['init_state']['a2c_network.layer_norm.bias'])
    osd = m.optimizer_state_dict(3e-4, 1, 0.0)
    assert len(osd['state']) == len(g['param_order'])
    for i, k in enumerate(g['param_order']):
        assert osd['state'][i]['exp_avg'].shape == g['init_state'][k].shape
    # without the option nothing changes: no LayerNorm tensors, no keys
    plain = B200Model(_network(g['units'], Hd, g['rnn_before_mlp'], layer_norm=False), g['D'], g['A'], 'cpu', True, True)
    assert not plain.rnn_layer_norm and plain.ln_w is None and 'ln_w' not in plain.layout
    assert not any('layer_norm' in k for k in plain.param_names())


@pytest.mark.parametrize('rnn_over,network_over,match', [
    ({'concat_input': True}, {}, "rnn: only a single-layer 'lstm'"),
    ({'concat_output': True}, {}, "rnn: only a single-layer 'lstm'"),
    ({'layers': 2}, {}, "rnn: only a single-layer 'lstm'"),
    ({'name': 'gru'}, {}, "rnn: only a single-layer 'lstm'"),
    ({}, {'separate': True}, 'separate actor/critic trunks with an rnn'),
    ({}, {'space': {'continuous': {'fixed_sigma': False}}}, 'state-dependent sigma with an rnn')])
def test_what_stays_refused_with_layer_norm(rnn_over, network_over, match, monkeypatch):
    from rl_games_b200.model import B200Model
    _standins(monkeypatch)
    net = _network([16, 8], 8, True, **rnn_over)
    net.update(network_over)
    with pytest.raises(NotImplementedError, match=match):
        B200Model(net, 6, 3, 'cpu', True, True)


def _host_agent(g, monkeypatch, tmp_path, mp):
    from rl_games_b200.runner import Runner
    import _torch_ops
    _standins(monkeypatch)
    monkeypatch.setitem(_torch_ops._USE_HOST_SCHED, 'on', True)
    monkeypatch.setattr(torch.cuda, 'set_device', lambda d: None)
    monkeypatch.setattr(torch.cuda, 'Event', _Event)
    monkeypatch.setattr(torch.cuda, 'current_stream', lambda *a: _Stream())
    monkeypatch.setattr(torch.Tensor, 'pin_memory', lambda self: self)
    cfgk = g['config']
    env = _Env(g)
    config = {k: v for k, v in cfgk.items() if k not in ('device', 'torch_compile')}
    config.update({'device': _CudaLookingStr('cpu'), 'env_info': env.get_env_info(), 'vec_env': env,
                   'reward_shaper': dict(g.get('reward_shaper') or {'scale_value': 1.0}), 'mixed_precision': mp, 'b200_cuda_graph': False,
                   'train_dir': str(tmp_path), 'lr_schedule': cfgk.get('lr_schedule', None)})
    r = Runner()
    r.load({'params': {'seed': 7, 'algo': {'name': 'a2c_continuous'}, 'model': {'name': 'continuous_a2c_logstd'},
                       'network': _network(g['units'], g['rnn_units'], g['rnn_before_mlp']), 'config': config}})
    r.params['config']['vec_env'] = env
    agent = r.algo_factory.create(r.algo_name, base_name='parity', params=r.params)
    assert agent.is_rnn and agent.model.rnn_layer_norm and not agent.use_tc and agent.gemm_tc == mp
    agent.model.load_state_dict(g['init_state'], strict=False)
    agent.init_tensors()
    agent._repack()
    agent.obs = agent.env_reset()
    return agent


@pytest.mark.parametrize('name', LN_GOLDEN)
@pytest.mark.parametrize('mp', [False, True])
def test_agent_host_logic_matches_reference_golden(name, mp, monkeypatch, tmp_path):
    """fp32 (mp False) and layer-wise tensor-core (mp True) host composition on torch stand-ins: the rollout's LayerNorm output, the
    window forward's scatter, BPTT through the LayerNorm and dgamma / dbeta through the step split rows, against the reference"""
    from oracle import ppo_oracle as O
    g = _load(name)
    agent = _host_agent(g, monkeypatch, tmp_path, mp)
    fl = O.swap_and_flatten01
    for ep, ref in enumerate(g['epochs_out']):
        agent.epoch_num += 1
        agent.train_epoch(noise=g['noise'][ep])
        ds = ref['dataset']
        assert torch.equal(agent.dones_buf, ref['mb_dones'])
        torch.testing.assert_close(agent.values.unsqueeze(2), ref['mb_values'], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(fl(agent.advs_n), ds['advantages'], rtol=2e-4, atol=2e-5)
        st = agent.last_stats
        torch.testing.assert_close(st[:, 0], ref['a_losses'], rtol=2e-3, atol=2e-6)
        torch.testing.assert_close(st[:, 1], ref['c_losses'], rtol=2e-3, atol=2e-6)
        assert agent.last_lr == pytest.approx(ref['last_lr'], rel=1e-12)
        sd = agent.model.state_dict()
        for k in g['param_order']:
            torch.testing.assert_close(sd[k], ref['state'][k], rtol=1e-3, atol=1e-4, msg=lambda m: k + ': ' + m)
    ck = agent.get_full_state_weights()
    for i, mref in enumerate(g['epochs_out'][-1]['adam_exp_avg']):
        torch.testing.assert_close(ck['optimizer']['state'][i]['exp_avg'].reshape(mref.shape), mref, rtol=1e-3, atol=1e-7)


def _ref_network(params, D, A):
    """the reference's A2CBuilder network for `params['network']` (oracle/_ref)"""
    for p in (os.path.join(HERE, 'golden', '_stubs'), REF):
        if p not in sys.path:
            sys.path.insert(0, p)
    from rl_games.algos_torch.network_builder import A2CBuilder
    b = A2CBuilder()
    b.load(params)
    return b.build('a2c', actions_num=A, input_shape=(D,), num_seqs=1, value_size=1)


@_need_ref
@pytest.mark.parametrize('name', ['agent_lstm_ln.pt', 'agent_lstm_ln_after.pt'])
def test_checkpoints_load_both_ways(name, monkeypatch, tmp_path):
    """ours -> the reference's network (load_state_dict strict, same forward), and the golden's reference state -> ours (resume)"""
    from rl_games_b200.model import B200Model
    g = _load(name)
    _standins(monkeypatch)
    net = _network(g['units'], g['rnn_units'], g['rnn_before_mlp'])
    m = B200Model(net, g['D'], g['A'], 'cpu', True, True)
    m.load_state_dict(g['epochs_out'][-1]['state'])          # a trained reference state resumes here
    for k in g['param_order']:
        assert torch.equal(m.state_dict()[k], g['epochs_out'][-1]['state'][k])
    with torch.no_grad():
        m.ln_w.add_(torch.linspace(-0.2, 0.2, g['rnn_units']))
    ref = _ref_network(net, g['D'], g['A'])
    sd = {k[len('a2c_network.'):]: v for k, v in m.state_dict().items() if k.startswith('a2c_network.')}
    ref.load_state_dict(sd, strict=True)
    assert [n for n, _ in ref.named_parameters()] == [k[len('a2c_network.'):] for k in m.param_names()]
    assert torch.equal(ref.layer_norm.weight.detach(), m.ln_w)


@_need_ref
def test_humanoid_yaml_with_layer_normed_lstm_trains_through_the_reference_runner(monkeypatch, tmp_path):
    """configs/mujoco/humanoid_envpool.yaml (shared trunk, MLP [512, 256, 128]) with rnn {lstm, 256, before_mlp, layer_norm} through
    rl_games_b200.register(<the reference's Runner>), kernels on torch stand-ins, scaled down to a CPU-sized batch; its checkpoint loads
    into the reference's A2CBuilder network, whose forward reproduces the agent's rollout outputs (mu, value)"""
    import yaml
    import rl_games_b200
    for p in (os.path.join(HERE, 'golden', '_stubs'), REF):
        if p not in sys.path:
            sys.path.insert(0, p)
    from rl_games.torch_runner import Runner
    import _torch_ops
    _standins(monkeypatch)
    monkeypatch.setitem(_torch_ops._USE_HOST_SCHED, 'on', True)
    monkeypatch.setattr(torch.cuda, 'set_device', lambda d: None)
    monkeypatch.setattr(torch.cuda, 'Event', _Event)
    monkeypatch.setattr(torch.cuda, 'current_stream', lambda *a: _Stream())
    monkeypatch.setattr(torch.Tensor, 'pin_memory', lambda self: self)
    from rl_games_b200 import ops

    def head_sample(*a, **k):        # the Runner's rollout draws its own noise on the device; the stand-in is handed zeros
        a = list(a)
        if a[7] is None and not k.get('values_only', False):
            a[7] = torch.zeros(a[-2], a[-1])
        return _torch_ops.policy_head_sample(*a, **k)
    monkeypatch.setattr(ops, 'policy_head_sample', head_sample)
    cfg = yaml.safe_load(open(os.path.join(REF, 'rl_games', 'configs', 'mujoco', 'humanoid_envpool.yaml')))
    net = cfg['params']['network']
    assert list(net['mlp']['units']) == [512, 256, 128] and not net.get('separate', False) and 'rnn' not in net
    net['rnn'] = {'name': 'lstm', 'units': 256, 'layers': 1, 'before_mlp': True, 'layer_norm': True}
    c = cfg['params']['config']
    N, H, D, A = 16, 8, 348, 17
    g = {'obs_tape': torch.randn(H + 1, N, D, generator=torch.Generator().manual_seed(4)), 'D': D, 'A': A, 'autoreset': 'same_step',
         'done_tape': torch.zeros(H + 1, N, dtype=torch.uint8), 'timeout_tape': torch.zeros(H + 1, N, dtype=torch.uint8)}
    g['done_tape'][3, :4] = 1
    env = _Env(g)
    c.update({'env_info': env.get_env_info(), 'vec_env': env, 'device': _CudaLookingStr('cpu'), 'max_epochs': 1, 'num_actors': N,
              'horizon_length': H, 'minibatch_size': N * H // 2, 'mini_epochs': 1, 'seq_length': 4, 'train_dir': str(tmp_path),
              'b200_cuda_graph': False, 'torch_compile': False, 'mixed_precision': False})
    runner = Runner()
    rl_games_b200.register(runner)
    runner.load(cfg)
    runner.params['config']['vec_env'] = env
    made = []
    orig_create = runner.algo_factory.create

    def create(name, **kw):
        a = orig_create(name, **kw)
        made.append(a)
        return a
    monkeypatch.setattr(runner.algo_factory, 'create', create)
    runner.run({'train': True, 'play': False, 'checkpoint': None, 'sigma': None})
    agent, = made
    assert agent.epoch_num == 1 and agent.model.rnn_layer_norm and agent.model.rnn_units == 256
    # the reference network, loaded from our checkpoint, on the next rollout step from the agent's carried states
    ck = agent.get_full_state_weights()
    ref = _ref_network(net, D, A)
    ref.load_state_dict({k[len('a2c_network.'):]: v for k, v in ck['model'].items() if k.startswith('a2c_network.')}, strict=True)
    ref.eval()
    obs = agent.obs['obs'] if isinstance(agent.obs, dict) else agent.obs
    h0, c0 = agent.rnn_h.clone(), agent.rnn_c.clone()
    agent.get_action_values(obs, noise=torch.zeros(N, A))
    rms = agent.model.running_mean_std
    x = torch.clamp((obs - rms.running_mean.float()) / torch.sqrt(rms.running_var.float() + 1e-5), -5.0, 5.0)
    with torch.no_grad():
        mu, _, value, _ = ref({'obs': x, 'rnn_states': (h0.unsqueeze(0), c0.unsqueeze(0)), 'seq_length': 1})
    vms = agent.model.value_mean_std
    value = torch.sqrt(vms.running_var.float() + 1e-5) * torch.clamp(value, -5.0, 5.0) + vms.running_mean.float()
    torch.testing.assert_close(agent.mus[0], mu, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(agent.values[0], value.squeeze(1), rtol=1e-4, atol=1e-5)
