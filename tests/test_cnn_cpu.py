"""The discrete agent with a conv2d trunk (``network.cnn``) on CPU, without the CUDA kernels:
- the model's arena, state-dict keys, parameter order and seeded initial weights against the reference network;
- the agent's host logic on torch stand-ins of the conv kernels (tests/_torch_ops_cnn.py) against the reference's golden runs on uint8
  frames (tests/golden/gen_golden_cnn.py);
- checkpoints in both directions with the reference's ModelA2C network;
- what stays refused, and why;
- every Atari / minigrid YAML of the reference through the reference's own Runner, every C-ABI call header-checked."""
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
GOLDENS = ['agent_cnn_shared.pt', 'agent_cnn_separate.pt']
needs_ref = pytest.mark.skipif(RR.REF is None, reason='reference rl_games not present (oracle/_ref)')


def _ref_path():
    for p in (os.path.join(GOLDEN, '_stubs'), RR.REF):
        if p not in sys.path:
            sys.path.insert(0, p)


class _FrameEnv:
    """gen_golden_cnn.FrameTapeVecEnv over the recorded tapes, as a tensor env of the agent"""

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
        rew = (actions.long() == g['obs_tape'][j0].reshape(g['N'], -1)[:, :self.K].argmax(dim=-1)).float()
        self.i += 1
        j = self.i % g['obs_tape'].shape[0]
        return g['obs_tape'][j].clone(), rew, g['done_tape'][j].clone(), {'time_outs': g['timeout_tape'][j].clone()}

    def get_env_info(self):
        from rl_games_b200.common import Box, Discrete
        return {'observation_space': Box(0, 255, tuple(self.g['obs_tape'].shape[2:]), 'uint8'), 'action_space': Discrete(self.K)}


def _stand_ins(monkeypatch):
    import _torch_ops_cnn
    from rl_games_b200 import agent_discrete
    _torch_ops_cnn.install_cnn(monkeypatch)
    monkeypatch.setattr(agent_discrete.DiscreteA2CAgent, '_require_cuda', lambda self: None)
    monkeypatch.setattr(agent_discrete.DiscreteA2CAgent, '_sync', staticmethod(lambda: None))


def _agent(monkeypatch, tmp_path, g, over=None):
    from rl_games_b200.runner import Runner
    _stand_ins(monkeypatch)
    env = _FrameEnv(g)
    config = {k: v for k, v in g['config'].items() if k not in ('device', 'torch_compile')}
    config.update({'device': 'cpu', 'env_info': env.get_env_info(), 'vec_env': env, 'reward_shaper': {'scale_value': 0.1},
                   'train_dir': str(tmp_path), 'lr_schedule': None})
    config.update(over or {})
    r = Runner()
    r.load({'params': {'seed': 1, 'algo': {'name': 'a2c_discrete'}, 'model': {'name': 'discrete_a2c'}, 'network': g['network'],
                       'config': config}})
    r.params['config']['vec_env'] = env
    agent = r.algo_factory.create(r.algo_name, base_name='cnn', params=r.params)
    agent.model.load_state_dict(g['init_state'])
    agent.init_tensors()
    agent.obs = agent.env_reset()
    return agent


def _golden(name):
    from _cnn_frames import frame_tape
    g = torch.load(os.path.join(GOLDEN, name), weights_only=False)
    g['obs_tape'] = frame_tape(g['T'], g['N'], g['frame_shape'], g['seed'])
    return g


@pytest.mark.parametrize('name', GOLDENS)
def test_model_layout_keys_order_and_seeded_init_match_the_reference(name, monkeypatch):
    from rl_games_b200.agent_discrete import DiscreteModel
    g = _golden(name)
    _stand_ins(monkeypatch)
    shape = tuple(g['obs_tape'].shape[2:])
    torch.manual_seed(g['seed'])
    m = DiscreteModel(g['network'], shape, g['K'], 'cpu', g['config']['normalize_input'], g['config']['normalize_value'])
    assert m.param_names() == g['param_order']
    assert m.param_names()[0] == 'a2c_network.actor_cnn.0.weight'
    assert m.conv_params == sum(v.numel() for k, v in g['seeded_state'].items() if '_cnn.' in k)
    sd = m.state_dict()
    assert [k for k in sd if k.startswith('a2c_network.')] == list(g['seeded_state'])
    for k, v in g['seeded_state'].items():
        assert sd[k].shape == v.shape, k
        assert torch.equal(sd[k], v), k          # draw for draw: the reference's construction, probe frame and init loop


@pytest.mark.parametrize('name', GOLDENS)
def test_agent_on_stand_ins_reproduces_the_reference_golden_run(name, monkeypatch, tmp_path):
    g = _golden(name)
    agent = _agent(monkeypatch, tmp_path, g)
    assert agent.obses.dtype == torch.uint8 and agent.obs.dtype == torch.uint8      # frames stay bytes in the arena
    fl = lambda t: t.transpose(0, 1).reshape(-1, *t.shape[2:])    # noqa: E731
    for ep, ref in enumerate(g['epochs_out']):
        agent.epoch_num += 1
        res = agent.train_epoch(u=g['u'][ep])
        assert torch.equal(agent.actions, ref['mb_actions'])
        torch.testing.assert_close(agent.rewards.unsqueeze(2), ref['mb_rewards'], rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(agent.values.unsqueeze(2), ref['mb_values'], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(fl(agent.advs_n), ref['advantages'], rtol=2e-4, atol=2e-5)
        torch.testing.assert_close(fl(agent.returns_n).unsqueeze(1), ref['returns'], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(fl(agent.neglogpacs), ref['old_logp_actions'], rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(torch.stack(res[4]), ref['a_losses'], rtol=2e-3, atol=2e-6)
        torch.testing.assert_close(torch.stack(res[5]), ref['c_losses'], rtol=2e-3, atol=2e-6)
        torch.testing.assert_close(torch.stack(res[6]), ref['entropies'], rtol=1e-4, atol=1e-6)
        torch.testing.assert_close(torch.stack(res[7]), ref['kls'], rtol=5e-3, atol=1e-8)
        sd = agent.model.state_dict()
        for k, v in ref['state'].items():
            torch.testing.assert_close(sd[k].reshape(v.shape).to(v.dtype), v, rtol=1e-4, atol=1e-5, msg=k)


def _ref_model(g):
    _ref_path()
    from rl_games.algos_torch import model_builder
    mb = model_builder.ModelBuilder()
    model = mb.load({'model': {'name': 'discrete_a2c'}, 'network': g['network']})
    return model.build({'actions_num': g['K'], 'input_shape': tuple(g['obs_tape'].shape[2:]), 'num_seqs': g['N'], 'value_size': 1,
                        'normalize_value': g['config']['normalize_value'], 'normalize_input': g['config']['normalize_input']})


@needs_ref
@pytest.mark.parametrize('name', GOLDENS)
def test_checkpoints_load_both_ways_with_the_reference_network(name, monkeypatch, tmp_path):
    """the agent's checkpoint into the reference's ModelA2C network: its forward on the agent's current frames gives the agent's rollout
    logits and value; a reference state dict resumes on the agent, optimiser state included"""
    g = _golden(name)
    agent = _agent(monkeypatch, tmp_path, g)
    agent.epoch_num += 1
    agent.train_epoch(u=g['u'][0])
    ckpt = str(tmp_path / 'ck')
    agent.save(ckpt)
    state = torch.load(ckpt + '.pth', weights_only=False)
    ref = _ref_model(g)
    ref.load_state_dict(state['model'])
    ref.eval()
    agent.play_steps(u=g['u'][1])          # leaves the forward of the last frames in r_out / last_values
    with torch.no_grad():
        out = ref({'is_train': False, 'obs': agent.obs.reshape(g['N'], *g['obs_tape'].shape[2:]).float() / 255.0, 'prev_actions': None})
    lg = agent.r_out[0]
    torch.testing.assert_close(lg, out['logits'] - out['logits'].logsumexp(-1, keepdim=True) + lg.logsumexp(-1, keepdim=True),
                               rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(agent.last_values, out['values'].squeeze(1), rtol=1e-4, atol=1e-5)
    # the other way: a reference network's weights and a torch Adam state over its parameters
    torch.manual_seed(123)
    ref2 = _ref_model(g)
    opt = torch.optim.Adam(ref2.parameters(), lr=1e-4)
    sum(p.sum() for p in ref2.parameters()).backward()
    opt.step()
    b = _agent(monkeypatch, tmp_path, g)
    b.set_full_state_weights({'model': ref2.state_dict(), 'optimizer': opt.state_dict(), 'epoch': 3, 'frame': 7,
                              'last_mean_rewards': 0.0})
    sd = b.model.state_dict()
    for k, v in ref2.state_dict().items():
        assert torch.equal(sd[k], v), k
    for m, p in zip(b.model._param_views(b.model.exp_avg), ref2.parameters()):
        assert torch.equal(m, opt.state[p]['exp_avg'])
    assert b.model.optimizer_state_dict(1e-4, 1, 0.0)['state'].keys() == opt.state_dict()['state'].keys()


# ------------------------------------------------------------------------------------------------------------------------------ refusals
def _net(**cnn):
    c = {'type': 'conv2d', 'activation': 'relu', 'initializer': {'name': 'default'},
         'convs': [{'filters': 4, 'kernel_size': 3, 'strides': 1, 'padding': 0}]}
    c.update(cnn)
    return {'name': 'actor_critic', 'separate': False, 'space': {'discrete': None}, 'cnn': c,
            'mlp': {'units': [8], 'activation': 'relu', 'initializer': {'name': 'default'}}}


@pytest.mark.parametrize('ctype,reason', [('conv1d', "'cnn' networks of type 'conv1d'"),
                                          ('conv2d_spatial_softargmax', "'cnn' networks.*spatial soft-argmax"),
                                          ('conv2d_flatten', "'cnn' networks.*flatten"), ('coord_conv2d', "'cnn' networks.*coordinate")])
def test_other_cnn_types_are_refused_with_their_reason(ctype, reason, monkeypatch):
    from rl_games_b200.agent_discrete import DiscreteModel
    _stand_ins(monkeypatch)
    with pytest.raises(NotImplementedError, match=reason):
        DiscreteModel(_net(type=ctype), (8, 8, 3), 4, 'cpu', False, False)


def test_cnn_with_rnn_and_bad_shapes_are_refused(monkeypatch):
    from rl_games_b200.agent_discrete import DiscreteModel
    _stand_ins(monkeypatch)
    net = dict(_net(), rnn={'name': 'lstm', 'units': 8, 'layers': 1})
    with pytest.raises(NotImplementedError, match="'rnn' networks are not supported by the discrete"):
        DiscreteModel(net, (8, 8, 3), 4, 'cpu', False, False)
    with pytest.raises(NotImplementedError, match='rank-3 Box observation'):
        DiscreteModel(_net(), (12,), 4, 'cpu', False, False)
    with pytest.raises(NotImplementedError, match='must be integers'):
        DiscreteModel(_net(convs=[{'filters': 4, 'kernel_size': [3, 2], 'strides': 1, 'padding': 0}]), (8, 8, 3), 4, 'cpu', False, False)
    with pytest.raises(ValueError, match='does not fit'):
        DiscreteModel(_net(convs=[{'filters': 4, 'kernel_size': 9, 'strides': 1, 'padding': 0}]), (8, 8, 3), 4, 'cpu', False, False)


# ----------------------------------------------------------------------------------------------- every Atari / minigrid YAML, header-checked
_FRAME = 36          # the smallest frame the shipped conv stacks (8/4, 4/2, 3/1) accept: the arena and activations stay small on CPU
_REFUSED = {'atari/ppo_breakout_torch_impala.yaml': "network 'resnet_actor_critic'", 'atari/ppo_pong_envpool_resnet.yaml':
            "network 'resnet_actor_critic'", 'atari/ppo_space_invaders_resnet.yaml': "network 'resnet_actor_critic'",
            'atari/ppo_pacman_torch_rnn.yaml': "'rnn' networks are not supported by the discrete",
            # LSTM straight on the conv output, no MLP: the model checks the MLP before the rnn
            'minigrid/lava_rnn_img.yaml': 'empty MLP', 'minigrid/minigrid_rnn_img.yaml': 'empty MLP'}


class _ImageEnv:
    def __init__(self, N, shape, K):
        self.N, self.shape, self.K = N, shape, K

    def reset(self):
        return torch.zeros((self.N,) + self.shape, dtype=torch.uint8)

    def step(self, actions):
        z8 = torch.zeros(self.N, dtype=torch.uint8)
        return self.reset(), torch.zeros(self.N), z8, {'time_outs': z8}

    def get_env_info(self):
        import gymnasium as gym
        return {'observation_space': gym.spaces.Box(0, 255, self.shape, np.uint8), 'action_space': gym.spaces.Discrete(self.K)}


def _image_yamls():
    if RR.REF is None:
        return []
    base = os.path.join(RR.REF, 'rl_games', 'configs')
    return sorted(os.path.join(d, f) for d in ('atari', 'minigrid') for f in os.listdir(os.path.join(base, d)) if f.endswith('.yaml'))


@needs_ref
@pytest.mark.parametrize('rel', _image_yamls())
def test_every_atari_and_minigrid_yaml_trains_or_gives_its_reason(rel, monkeypatch, tmp_path):
    """each shipped image YAML, unchanged but for what a launcher injects (a uint8 frame env at 36 x 36, device, one epoch): the plain
    conv2d networks train one epoch of `runner.run` through the conv kernels (every call header-checked); the others raise their reason"""
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
    nhwc = (net.get('cnn') or {}).get('permute_input', True)
    shape = (_FRAME, _FRAME, 4) if nhwc else (4, _FRAME, _FRAME)
    N = c['num_actors']
    env = _ImageEnv(N, shape, 6)
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
        with pytest.raises(NotImplementedError, match=_REFUSED[rel]):
            runner.run({'train': True, 'play': False, 'checkpoint': None, 'sigma': None})
        return
    runner.run({'train': True, 'play': False, 'checkpoint': None, 'sigma': None})
    agent, = made
    assert type(agent) is agent_discrete.DiscreteA2CAgent and agent.epoch_num == 1 and agent.obses.dtype == torch.uint8
    n_conv = len(net['cnn']['convs'])
    n_upd = c['mini_epochs'] * (N * c['horizon_length'] // c['minibatch_size'])
    trunks = 2 if net.get('separate') else 1
    assert rec.calls['b200rl_conv2d_fwd_f32'] == trunks * n_conv * (c['horizon_length'] + 1 + n_upd)
    assert rec.calls['b200rl_conv2d_bwd_weight_f32'] == trunks * n_conv * n_upd
    assert rec.calls['b200rl_conv2d_bwd_data_f32'] == trunks * (n_conv - 1) * n_upd
    assert rec.calls.get('b200rl_moments_update_u8_f64', 0) == (n_upd if c.get('normalize_input') else 0)
    assert rec.calls.get('b200rl_moments_update_f64', 0) == 0
