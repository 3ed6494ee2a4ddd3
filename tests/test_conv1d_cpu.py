"""The discrete agent with a conv1d trunk (``network.cnn.type: conv1d``, the smac frame-stack configs) on CPU, without the CUDA kernels:
- the model's arena, state-dict keys, parameter order and shapes and seeded initial weights against the reference network;
- the agent's host logic on torch stand-ins of the conv1d kernels (tests/_torch_ops_conv1d.py) against the reference's golden runs on
  frame stacks (tests/golden/gen_golden_conv1d.py);
- checkpoints in both directions with the reference's ModelA2C network;
- what stays refused, and why;
- one epoch, fp32 and ``mixed_precision: True``, every C-ABI call header-checked;
- every smac conv1d YAML of the reference through the reference's own Runner with a frame-stacked multi-agent env;
- the player (PpoPlayerDiscrete) on a rank-2 observation against the reference player's recorded play
  (tests/golden/conv1d_player_disc.pt);
- init_tensors' refusal of a geometry the device has no room for, before it allocates anything."""
import math
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import test_abi_calls_cpu as ABI  # noqa: E402
import test_reference_runner_cpu as RR  # noqa: E402

GOLDEN = os.path.join(HERE, 'golden')
GOLDENS = ['agent_conv1d_separate.pt', 'agent_conv1d_shared.pt']
needs_ref = pytest.mark.skipif(RR.REF is None, reason='reference rl_games not present (oracle/_ref)')


def _ref_path():
    for p in (os.path.join(GOLDEN, '_stubs'), RR.REF):
        if p not in sys.path:
            sys.path.insert(0, p)


def _golden(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


class StackEnv:
    """gen_golden_conv1d.StackTapeVecEnv over the recorded tapes, as a tensor env of the agent"""

    def __init__(self, g):
        self.g, self.K, self.i = g, g['K'], 0

    def reset(self):
        self.i = 0
        return self.g['obs_tape'][0].clone()

    def get_action_masks(self):
        return self.g['mask_tape'][self.i % self.g['mask_tape'].shape[0]]

    def step(self, actions):
        g = self.g
        j0 = self.i % g['obs_tape'].shape[0]
        rew = (actions.long() == g['obs_tape'][j0][:, -1, :self.K].argmax(dim=-1)).float()
        self.i += 1
        j = self.i % g['obs_tape'].shape[0]
        return g['obs_tape'][j].clone(), rew, g['done_tape'][j].clone(), {'time_outs': g['timeout_tape'][j].clone()}

    def get_env_info(self):
        from rl_games_b200.common import Box, Discrete
        info = {'observation_space': Box(-np.inf, np.inf, tuple(self.g['obs_tape'].shape[2:])), 'action_space': Discrete(self.K)}
        if self.g['agents'] > 1:
            info['agents'] = self.g['agents']
        return info


def stand_ins(monkeypatch):
    import _torch_ops_conv1d
    from rl_games_b200 import agent_discrete
    _torch_ops_conv1d.install_conv1d(monkeypatch)
    monkeypatch.setattr(agent_discrete.DiscreteA2CAgent, '_require_cuda', lambda self: None)
    monkeypatch.setattr(agent_discrete.DiscreteA2CAgent, '_sync', staticmethod(lambda: None))


def make_agent(g, tmp_path, over=None, device='cpu'):
    """the golden run's agent with the config overrides `over` (the ops as installed by the caller)"""
    from rl_games_b200.runner import Runner
    env = StackEnv(g)
    config = {k: v for k, v in g['config'].items() if k not in ('device', 'torch_compile')}
    config.update({'device': device, 'env_info': env.get_env_info(), 'vec_env': env, 'reward_shaper': {'scale_value': 0.1},
                   'train_dir': str(tmp_path), 'lr_schedule': None})
    config.update(over or {})
    r = Runner()
    r.load({'params': {'seed': 1, 'algo': {'name': 'a2c_discrete'}, 'model': {'name': 'discrete_a2c'}, 'network': g['network'],
                       'config': config}})
    r.params['config']['vec_env'] = env
    agent = r.algo_factory.create(r.algo_name, base_name='conv1d', params=r.params)
    agent.model.load_state_dict(g['init_state'])
    agent.init_tensors()
    agent.obs = agent.env_reset()
    return agent


def check_epochs(agent, g, tol=1.0):
    """the agent's epochs against the golden reference run (tol scales the tolerances of the float comparisons)"""
    fl = lambda t: t.transpose(0, 1).reshape(-1, *t.shape[2:]).cpu()    # noqa: E731
    for ep, ref in enumerate(g['epochs_out']):
        agent.epoch_num += 1
        res = agent.train_epoch(u=g['u'][ep].to(agent.device_t))
        assert torch.equal(agent.actions.cpu(), ref['mb_actions'])
        torch.testing.assert_close(agent.rewards.unsqueeze(2).cpu(), ref['mb_rewards'], rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(agent.values.unsqueeze(2).cpu(), ref['mb_values'], rtol=1e-4 * tol, atol=1e-5 * tol)
        torch.testing.assert_close(fl(agent.advs_n), ref['advantages'], rtol=2e-4 * tol, atol=2e-5 * tol)
        torch.testing.assert_close(fl(agent.returns_n).unsqueeze(1), ref['returns'], rtol=1e-4 * tol, atol=1e-5 * tol)
        torch.testing.assert_close(fl(agent.neglogpacs), ref['old_logp_actions'], rtol=1e-5 * tol, atol=1e-5 * tol)
        torch.testing.assert_close(torch.stack(res[4]).cpu(), ref['a_losses'], rtol=2e-3 * tol, atol=2e-6 * tol)
        torch.testing.assert_close(torch.stack(res[5]).cpu(), ref['c_losses'], rtol=2e-3 * tol, atol=2e-6 * tol)
        torch.testing.assert_close(torch.stack(res[6]).cpu(), ref['entropies'], rtol=1e-4 * tol, atol=1e-6 * tol)
        torch.testing.assert_close(torch.stack(res[7]).cpu(), ref['kls'], rtol=5e-3 * tol, atol=1e-8 * tol)
        sd = agent.model.state_dict()
        for k, v in ref['state'].items():
            torch.testing.assert_close(sd[k].reshape(v.shape).to(v.dtype).cpu(), v, rtol=1e-4 * tol, atol=1e-5 * tol, msg=k)


@pytest.mark.parametrize('name', GOLDENS)
def test_model_layout_keys_order_shapes_and_seeded_init_match_the_reference(name, monkeypatch):
    from rl_games_b200.agent_discrete import DiscreteModel
    g = _golden(name)
    stand_ins(monkeypatch)
    torch.manual_seed(g['seed'])
    m = DiscreteModel(g['network'], tuple(g['obs_tape'].shape[2:]), g['K'], 'cpu', g['config']['normalize_input'],
                      g['config']['normalize_value'])
    assert m.cnn.conv1d and m.param_names() == g['param_order']
    assert m.conv_params == sum(v.numel() for k, v in g['seeded_state'].items() if '_cnn.' in k)
    sd = m.state_dict()
    assert [k for k in sd if k.startswith('a2c_network.')] == list(g['seeded_state'])
    for k, v in g['seeded_state'].items():
        assert sd[k].shape == v.shape, k
        assert torch.equal(sd[k], v), k          # draw for draw: the reference's construction, probe frame and init loop
    assert sd['a2c_network.actor_cnn.0.weight'].dim() == 3 and sd['a2c_network.actor_cnn.2.weight'].dim() == 3
    if g['config']['normalize_input']:
        assert sd['running_mean_std.running_mean'].shape == tuple(g['obs_tape'].shape[2:])


@pytest.mark.parametrize('name', GOLDENS)
def test_agent_on_stand_ins_reproduces_the_reference_golden_run(name, monkeypatch, tmp_path):
    g = _golden(name)
    stand_ins(monkeypatch)
    agent = make_agent(g, tmp_path)
    assert agent.obses.dtype == torch.float32 and agent.num_agents == g['agents']
    check_epochs(agent, g)


def _ref_model(g):
    _ref_path()
    from rl_games.algos_torch import model_builder
    mb = model_builder.ModelBuilder()
    model = mb.load({'model': {'name': 'discrete_a2c'}, 'network': g['network']})
    return model.build({'actions_num': g['K'], 'input_shape': tuple(g['obs_tape'].shape[2:]), 'num_seqs': g['rows'], 'value_size': 1,
                        'normalize_value': g['config']['normalize_value'], 'normalize_input': g['config']['normalize_input']})


@needs_ref
@pytest.mark.parametrize('name', GOLDENS)
def test_checkpoints_load_both_ways_with_the_reference_network(name, monkeypatch, tmp_path):
    """the agent's checkpoint into the reference's ModelA2C network: its forward on the agent's current observations gives the agent's
    rollout logits and value; a reference state dict resumes on the agent, optimiser state included"""
    g = _golden(name)
    stand_ins(monkeypatch)
    agent = make_agent(g, tmp_path)
    agent.epoch_num += 1
    agent.train_epoch(u=g['u'][0])
    ckpt = str(tmp_path / 'ck')
    agent.save(ckpt)
    state = torch.load(ckpt + '.pth', weights_only=False)
    ref = _ref_model(g)
    ref.load_state_dict(state['model'])
    ref.eval()
    agent.play_steps(u=g['u'][1])
    with torch.no_grad():
        out = ref({'is_train': False, 'obs': agent.obs.reshape(g['rows'], *g['obs_tape'].shape[2:]), 'prev_actions': None})
    lg = agent.r_out[0]
    torch.testing.assert_close(lg, out['logits'] - out['logits'].logsumexp(-1, keepdim=True) + lg.logsumexp(-1, keepdim=True),
                               rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(agent.last_values, out['values'].squeeze(1), rtol=1e-4, atol=1e-5)
    torch.manual_seed(123)
    ref2 = _ref_model(g)
    opt = torch.optim.Adam(ref2.parameters(), lr=1e-4)
    sum(p.sum() for p in ref2.parameters()).backward()
    opt.step()
    b = make_agent(g, tmp_path)
    b.set_full_state_weights({'model': ref2.state_dict(), 'optimizer': opt.state_dict(), 'epoch': 3, 'frame': 7,
                              'last_mean_rewards': 0.0})
    sd = b.model.state_dict()
    for k, v in ref2.state_dict().items():
        assert torch.equal(sd[k], v), k
    for m, p in zip(b.model._param_views(b.model.exp_avg), ref2.parameters()):
        assert torch.equal(m, opt.state[p]['exp_avg'])


# ------------------------------------------------------------------------------------------------------------------------------ refusals
def _net(convs=None, **extra):
    c = {'type': 'conv1d', 'activation': 'relu', 'initializer': {'name': 'default'},
         'convs': convs or [{'filters': 8, 'kernel_size': 3, 'strides': 1, 'padding': 1}]}
    return dict({'name': 'actor_critic', 'separate': True, 'space': {'discrete': None}, 'cnn': c,
                 'mlp': {'units': [8], 'activation': 'relu', 'initializer': {'name': 'default'}}}, **extra)


@pytest.mark.parametrize('shape', [(12,), (8, 8, 3)])
def test_conv1d_on_rank_1_or_rank_3_observations_is_refused(shape, monkeypatch):
    from rl_games_b200.agent_discrete import DiscreteModel
    stand_ins(monkeypatch)
    with pytest.raises(NotImplementedError, match="^'cnn' networks of type 'conv1d' need a rank-2 Box observation"):
        DiscreteModel(_net(), shape, 4, 'cpu', False, False)


def test_uint8_frame_stacks_and_rank_2_observations_without_conv1d_are_refused():
    from rl_games_b200.agent_discrete import discrete_spaces
    from rl_games_b200.common import Box, Discrete
    with pytest.raises(NotImplementedError, match="^'cnn' networks of type 'conv1d' read fp32 observations"):
        discrete_spaces(Box(0, 255, (4, 12), 'uint8'), Discrete(4), _net(), {})
    conv2d = _net()
    conv2d['cnn'] = dict(conv2d['cnn'], type='conv2d')
    for net in (conv2d, {k: v for k, v in _net().items() if k != 'cnn'}):
        with pytest.raises(NotImplementedError, match='only flat Box observations'):
            discrete_spaces(Box(-1, 1, (4, 12)), Discrete(4), net, {})
    assert discrete_spaces(Box(-1, 1, (4, 12)), Discrete(4), _net(), {})[:2] == ((4, 12), torch.float32)


@pytest.mark.parametrize('key,value', [('kernel_size', 2.0), ('kernel_size', [3]), ('strides', '1'), ('padding', 1.5), ('padding', True)])
def test_non_integer_kernel_stride_or_padding_is_refused(key, value, monkeypatch):
    from rl_games_b200.agent_discrete import DiscreteModel
    stand_ins(monkeypatch)
    conv = dict({'filters': 8, 'kernel_size': 3, 'strides': 1, 'padding': 1}, **{key: value})
    with pytest.raises(NotImplementedError, match='conv1d kernel_size / strides / padding must be integers'):
        DiscreteModel(_net([conv]), (4, 12), 4, 'cpu', False, False)


def test_a_stack_that_does_not_fit_and_conv1d_with_an_rnn_are_refused(monkeypatch):
    from rl_games_b200.agent_discrete import DiscreteModel
    stand_ins(monkeypatch)
    # 3m_cnn_torch with transpose: True on 4 frames: (features, 4) -> k3 s2 p1 -> 2 positions -> k3 p0 does not fit
    convs = [{'filters': 64, 'kernel_size': 3, 'strides': 2, 'padding': 1}, {'filters': 128, 'kernel_size': 3, 'strides': 1, 'padding': 0}]
    with pytest.raises(ValueError, match='conv1d kernel 3 does not fit a 2 input with padding 0'):
        DiscreteModel(_net(convs), (30, 4), 4, 'cpu', False, False)
    with pytest.raises(NotImplementedError, match="'rnn' networks are not supported by the discrete"):
        DiscreteModel(_net(rnn={'name': 'lstm', 'units': 8, 'layers': 1}), (4, 12), 4, 'cpu', False, False)


@needs_ref
def test_does_not_fit_where_the_reference_calc_input_size_fails():
    """the reference's own network builder on the same geometry fails in _calc_input_size"""
    _ref_path()
    from rl_games.algos_torch import model_builder
    net = _net([{'filters': 64, 'kernel_size': 3, 'strides': 2, 'padding': 1}, {'filters': 128, 'kernel_size': 3, 'strides': 1, 'padding': 0}])
    model = model_builder.ModelBuilder().load({'model': {'name': 'discrete_a2c'}, 'network': net})
    with pytest.raises(RuntimeError):
        model.build({'actions_num': 4, 'input_shape': (30, 4), 'num_seqs': 1, 'value_size': 1})


# ------------------------------------------------------------------------------------------- one epoch, every C-ABI call header-checked
@pytest.mark.parametrize('mixed_precision', [False, True])
@pytest.mark.parametrize('name', GOLDENS)
def test_one_epoch_makes_header_checked_conv1d_calls(name, mixed_precision, monkeypatch, tmp_path):
    from rl_games_b200 import agent_discrete
    g = _golden(name)
    rec = ABI._patch(monkeypatch)
    monkeypatch.setattr(agent_discrete.DiscreteA2CAgent, '_require_cuda', lambda self: None)
    monkeypatch.setattr(agent_discrete.DiscreteA2CAgent, '_sync', staticmethod(lambda: None))
    agent = make_agent(g, tmp_path, {'mixed_precision': mixed_precision})
    agent.epoch_num += 1
    agent.train_epoch(u=g['u'][0])
    sfx, other = ('tc', 'f32') if mixed_precision else ('f32', 'tc')
    n_conv, trunks = len(g['network']['cnn']['convs']), 2 if g['separate'] else 1
    n_upd = g['config']['mini_epochs'] * (g['rows'] * g['H'] // g['mb'])
    assert rec.calls[f'b200rl_conv1d_fwd_{sfx}'] == trunks * n_conv * (g['H'] + 1 + n_upd)
    assert rec.calls[f'b200rl_conv1d_bwd_weight_{sfx}'] == trunks * n_conv * n_upd
    assert rec.calls[f'b200rl_conv1d_bwd_data_{sfx}'] == trunks * (n_conv - 1) * n_upd
    convs = ('conv1d_fwd', 'conv1d_bwd_data', 'conv1d_bwd_weight', 'conv2d_fwd', 'conv2d_bwd_data', 'conv2d_bwd_weight')
    for op in convs:                                   # no conv of the other precision
        assert rec.calls.get(f'b200rl_{op}_{other}', 0) == 0, op
    for op in convs[3:]:                               # no conv2d of this precision either
        assert rec.calls.get(f'b200rl_{op}_{sfx}', 0) == 0, op
    # the conv gradients reduce from their own split rows over the conv parameters, the MLP's from `part`
    assert agent.cpart.shape == (agent.conv_splits, agent.model.conv_params)
    assert agent.part.shape == (agent.n_splits, agent.model.num_params)
    assert rec.calls['b200rl_reduce_splits_f32'] == 2 * n_upd


def test_init_tensors_bytes_counts_the_27m_update_within_an_h100():
    """27m_vs_30m_torch's geometry (4 frames x 285 features, 1024-filter stack, minibatch 3456, 8 envs x 27 agents) from the byte count
    alone: what init_tensors would allocate, and the model's arena, fit 80 GB"""
    from rl_games_b200 import agent_discrete
    from rl_games_b200.agent_discrete import _ConvTrunk

    class _M:           # the geometry of DiscreteModel without its 150 M parameters
        separate, units = True, [256, 128]
        cnn = _ConvTrunk({'type': 'conv1d', 'convs': [{'filters': f, 'kernel_size': 3, 'strides': 1, 'padding': 1} for f in (256, 512, 1024)]},
                         (4, 285))
        D = 4 * 285
        conv_params = 2 * sum(s[0] * s[1] * s[2] + s[0] for s, _ in cnn.layers)
        num_params = conv_params + 2 * (1024 * 285 * 256 + 256 + 256 * 128 + 128) + 129 * 1 + 128 * 14 + 14 + 1
    a = agent_discrete.DiscreteA2CAgent.__new__(agent_discrete.DiscreteA2CAgent)
    a.model, a.horizon_length, a.num_rows, a.minibatch_size, a.actions_num = _M, 128, 216, 3456, 14
    a.head_sizes, a.use_action_masks, a.mask_autoreset_rows = None, True, False
    for mp, S in ((False, 13), (True, 6)):
        a.n_splits, a.conv_splits, a.mixed_precision = S, 64, mp
        need = a.init_tensors_bytes() + 12 * _M.num_params
        assert 20e9 < need < 60e9, need


# ------------------------------------------------------------------------------------------------------- every smac conv1d YAML
_REFUSED = {'smac/v1/3m_cnn_torch.yaml': 'does not fit'}          # transpose: True on 4 frames: ValueError from the trunk


def _conv1d_yamls():
    if RR.REF is None:
        return []
    base = os.path.join(RR.REF, 'rl_games', 'configs')
    out = []
    for d in ('smac/v1', 'smac/v1/runs'):
        for f in sorted(os.listdir(os.path.join(base, d))):
            if f.endswith('.yaml') and "conv1d" in open(os.path.join(base, d, f)).read():
                out.append(f'{d}/{f}')
    return out


class _StackMAEnv:
    """zero frame stacks Box(frames, features) (or (features, frames) with the wrapper's transpose) for envs * agents rows"""

    def __init__(self, rows, shape, K, agents):
        self.rows, self.shape, self.K, self.agents = rows, shape, K, agents

    def reset(self):
        return torch.zeros((self.rows,) + self.shape)

    def step(self, actions):
        z8 = torch.zeros(self.rows, dtype=torch.uint8)
        return self.reset(), torch.zeros(self.rows), z8, {'time_outs': z8}

    def get_action_masks(self):
        return torch.ones(self.rows, self.K, dtype=torch.uint8)

    def get_env_info(self):
        import gymnasium as gym
        return {'observation_space': gym.spaces.Box(0, 1, self.shape, np.float32), 'action_space': gym.spaces.Discrete(self.K),
                'agents': self.agents}


_FEATURES = 12          # a small feature count every shipped stack accepts untransposed: the CPU buffers stay small


@needs_ref
@pytest.mark.parametrize('rel', _conv1d_yamls())
def test_every_smac_conv1d_yaml_trains_or_gives_its_reason(rel, monkeypatch, tmp_path):
    """each shipped conv1d YAML, unchanged but for what a launcher injects (an env whose observation is the YAML's frame stack, device,
    one epoch): trains one epoch of `runner.run` through the conv1d kernels (every call header-checked), or raises its reason"""
    import yaml
    _ref_path()
    from rl_games.torch_runner import Runner
    import rl_games_b200
    from rl_games_b200 import agent_discrete
    rec = ABI._patch(monkeypatch)
    monkeypatch.setattr(agent_discrete.DiscreteA2CAgent, '_require_cuda', lambda self: None)
    monkeypatch.setattr(agent_discrete.DiscreteA2CAgent, '_sync', staticmethod(lambda: None))
    cfg = yaml.safe_load(open(os.path.join(RR.REF, 'rl_games', 'configs', rel)))
    c, net = cfg['params']['config'], cfg['params']['network']
    ec = c.get('env_config', {})
    frames = ec.get('frames', 4)
    shape = (_FEATURES, frames) if ec.get('transpose') else (frames, _FEATURES)
    N, Hn, mb = c['num_actors'], c['horizon_length'], c['minibatch_size']
    G = mb // math.gcd(Hn * N, mb)          # the fewest agents (at least 2) that make the batch a whole number of minibatches
    G = G * (-(-2 // G))
    env = _StackMAEnv(N * G, shape, 6, G)
    c.update({'env_info': env.get_env_info(), 'vec_env': env, 'device': 'cpu', 'max_epochs': 1, 'train_dir': str(tmp_path),
              'multi_gpu': False})
    c.pop('max_frames', None)
    runner = Runner()
    rl_games_b200.register(runner)
    runner.load(cfg)
    runner.params['config']['vec_env'] = env
    made = []
    orig_create = runner.algo_factory.create
    monkeypatch.setattr(runner.algo_factory, 'create', lambda name, **kw: (made.append(orig_create(name, **kw)), made[-1])[1])
    if rel in _REFUSED:
        with pytest.raises((NotImplementedError, ValueError), match=_REFUSED[rel]):
            runner.run({'train': True, 'play': False, 'checkpoint': None, 'sigma': None})
        return
    runner.run({'train': True, 'play': False, 'checkpoint': None, 'sigma': None})
    agent, = made
    assert type(agent) is agent_discrete.DiscreteA2CAgent and agent.epoch_num == 1 and agent.num_agents == G
    n_conv = len(net['cnn']['convs'])
    n_upd = c['mini_epochs'] * (N * G * Hn // mb)
    trunks = 2 if net.get('separate') else 1
    sfx = 'tc' if c.get('mixed_precision') else 'f32'
    assert rec.calls[f'b200rl_conv1d_fwd_{sfx}'] == trunks * n_conv * (Hn + 1 + n_upd)
    assert rec.calls[f'b200rl_conv1d_bwd_weight_{sfx}'] == trunks * n_conv * n_upd
    assert rec.calls[f'b200rl_conv1d_bwd_data_{sfx}'] == trunks * (n_conv - 1) * n_upd
    assert rec.calls['b200rl_post_step_ma_f32'] == Hn


# ------------------------------------------------------------------------------------------------------------------------------ memory
def test_init_tensors_refuses_a_geometry_the_device_has_no_room_for_before_allocating(monkeypatch, tmp_path):
    """a conv1d agent on a device whose free memory is below init_tensors_bytes plus the epoch's transient allowance: RuntimeError
    naming the bytes, nothing allocated"""
    from rl_games_b200 import agent_discrete
    g = _golden('agent_conv1d_separate.pt')
    stand_ins(monkeypatch)
    agent = make_agent(g, tmp_path)
    need = agent.init_tensors_bytes() + agent.TRANSIENT_BYTES
    assert need > agent.TRANSIENT_BYTES
    agent._tensors_ready = False
    for name in ('obses', 'part', 'cpart', 'r_a', 't_a', 'd_a', 'grad'):
        delattr(agent, name)
    agent.device_t = torch.device('cuda', 0)           # the check only runs on a CUDA device; the device is never touched
    monkeypatch.setattr(torch.cuda, 'mem_get_info', lambda dev=None: (need - 1, 80 * 2 ** 30))
    allocs = []
    monkeypatch.setattr(agent_discrete.torch, 'zeros', lambda *a, **k: allocs.append(a))
    with pytest.raises(RuntimeError, match=f'needs {need} bytes of device memory'):
        agent.init_tensors()
    assert allocs == [] and not hasattr(agent, 'obses')
    monkeypatch.setattr(torch.cuda, 'mem_get_info', lambda dev=None: (need, 80 * 2 ** 30))
    agent._check_memory()                              # exactly enough: accepted


# ------------------------------------------------------------------------------------------------------------------------------ player
PLAYER_FIXTURE = os.path.join(GOLDEN, 'conv1d_player_disc.pt')


def fixture_player(fx, over, tmp_path, device='cpu'):
    """the package's PpoPlayerDiscrete for the fixture's network on its rank-2 Box, restored from the reference player's state dict"""
    from rl_games_b200.common import Box, Discrete
    from rl_games_b200 import players
    params = dict(fx['params'])
    config = dict(params['config'], device_name=device, b200_cuda_graph=device != 'cpu', **over)
    config.update(env_info={'observation_space': Box(-np.inf, np.inf, tuple(fx['obs_shape'])), 'action_space': Discrete(fx['K']),
                            'agents': fx['agents']}, vec_env=None)
    params['config'] = config
    p = players.PpoPlayerDiscrete(params)
    fn = os.path.join(str(tmp_path), 'conv1d_player.pth')
    torch.save(fx['state'], fn)
    p.restore(fn)
    return p


def replay_player(p, fx, device='cpu', atol=1e-5, rtol=0.0):
    """the fixture's tape through the player: the batch is detected from the rank-2 obs shape, the argmax equals the reference's on
    every row with a clear margin, and the normalised masked logits agree within (atol, rtol)"""
    K, clear_rows = fx['K'], 0
    for t in range(fx['obs'].shape[0]):
        obs, mask = fx['obs'][t].to(device), fx['masks'][t].to(device)
        if t == 0:
            assert p.get_batch_size(obs, 1) == obs.shape[0] and p.has_batch_dimension
        a = p.get_masked_action(obs, mask, True)
        clear = fx['clear'][t].to(device)
        got, want = a.reshape(clear.shape), fx['actions'][t].to(device).reshape(clear.shape)
        assert torch.equal(got[clear], want[clear]), (t, got, want)
        clear_rows += int(clear.sum())
        rows = mask.any(dim=1)
        lg = torch.where(mask, p.r_out[0][:, :K], torch.full_like(mask, -float('inf'), dtype=torch.float32))[rows]
        torch.testing.assert_close(torch.log_softmax(lg, -1)[mask[rows]], fx['logits'][t].to(device)[rows][mask[rows]], atol=atol, rtol=rtol)
        p._done_rows(fx['dones'][t].to(device))
    assert clear_rows >= fx['clear'].numel() // 2


def test_player_plays_frame_stacks_like_the_reference_player(monkeypatch, tmp_path):
    """PpoPlayerDiscrete on Box(frames, features) with a conv1d trunk on the torch stand-ins: checkpoint restore (the (C, L)-shaped
    normaliser included), batch detection, masked deterministic actions and logits against the reference player's recorded play"""
    import _torch_ops_conv1d
    import _torch_ops_player
    from rl_games_b200 import ops, players
    _torch_ops_player.install(monkeypatch)
    for name in ('conv1d_fwd', 'conv1d_bwd_data', 'conv1d_bwd_weight'):
        monkeypatch.setattr(ops, name, getattr(_torch_ops_conv1d, name))
    monkeypatch.setattr(players.BasePlayer, '_require_cuda', lambda self: None)
    fx = torch.load(PLAYER_FIXTURE, weights_only=False)
    p = fixture_player(fx, {'mixed_precision': False}, tmp_path)
    assert p.model.cnn.conv1d
    assert torch.equal(p.model.state_dict()['running_mean_std.running_mean'], fx['state']['model']['running_mean_std.running_mean'])
    replay_player(p, fx)
    assert p.obs_buf.shape == (fx['obs'].shape[1], int(np.prod(fx['obs_shape']))) and p.obs_buf.dtype == torch.float32


def test_player_header_checked_calls_in_both_precisions(monkeypatch, tmp_path):
    from rl_games_b200 import players
    rec = ABI._patch(monkeypatch)
    monkeypatch.setattr(players.BasePlayer, '_require_cuda', lambda self: None)
    fx = torch.load(PLAYER_FIXTURE, weights_only=False)
    for mp, sfx in ((False, 'f32'), (True, 'tc')):
        rec.calls.clear()
        p = fixture_player(fx, {'mixed_precision': mp}, tmp_path)
        assert (p.wbf is not None) == mp
        obs = fx['obs'][0]
        p.get_batch_size(obs, 1)
        p.get_masked_action(obs, fx['masks'][0], True)
        n_conv = len(fx['params']['network']['cnn']['convs'])
        assert rec.calls[f'b200rl_conv1d_fwd_{sfx}'] == 2 * n_conv              # separate trunks
        assert rec.calls['b200rl_categorical_argmax_f32'] == 1
