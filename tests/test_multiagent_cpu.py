"""Multi-agent envs (env_info['agents'] = G > 1) on the continuous agent, without a GPU: the agent's host logic on torch stand-ins
(tests/_torch_ops.py plus tests/_torch_ops_ma.py) against golden runs of the reference (tests/golden/gen_golden_ma.py), per env step
(the indices handed to process_infos, the game meters) and per epoch (buffers, losses, weights, frames); the C-ABI prototype of the
multi-agent post-step; the configurations that stay refused, each with its reason."""
import ctypes
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_agent_host_cpu as H  # noqa: E402
import test_discrete_host_cpu as DH  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')


class _MAEnv(H._Env):
    def get_env_info(self):
        info = super().get_env_info()
        info['agents'] = self.g['G']
        return info


class _RecordingObserver:
    """DefaultAlgoObserver plus a record of what every env step hands to process_infos and the meters right after it"""

    def __init__(self):
        self.steps = []
        self.agent = None

    def before_init(self, base_name, config, experiment_name):
        pass

    def after_init(self, algo):
        self.agent = algo

    def process_infos(self, infos, done_indices):
        a = self.agent
        a._meter_cache = None
        self.steps.append({'done_indices': done_indices.clone(), 'game_rewards_mean': a.game_rewards.mean.clone(),
                           'game_shaped_rewards_mean': a.game_shaped_rewards.mean.clone(),
                           'game_lengths_mean': a.game_lengths.mean.clone(), 'game_size': a.game_rewards.current_size})

    def after_steps(self):
        pass

    def after_clear_stats(self):
        pass

    def after_print_stats(self, frame, epoch_num, total_time):
        pass


def _network(g):
    net = {'name': 'actor_critic', 'separate': False,
           'space': {'continuous': {'mu_activation': 'None', 'sigma_activation': 'None', 'mu_init': {'name': 'default'},
                                    'sigma_init': {'name': 'const_initializer', 'val': 0}, 'fixed_sigma': True}},
           'mlp': {'units': g['units'], 'activation': 'elu', 'initializer': {'name': 'default'}}}
    if g.get('rnn_units', 0):
        net['rnn'] = {'name': 'lstm', 'units': g['rnn_units'], 'layers': 1, 'before_mlp': True}
    return net


def _build(monkeypatch, tmp_path, g, over=None, network=None, env_info_over=None, algo='a2c_continuous', env_cls=None):
    import _torch_ops
    import _torch_ops_ma
    from rl_games_b200.runner import Runner
    _torch_ops.install_continuous(monkeypatch)
    _torch_ops_ma.install(monkeypatch)
    monkeypatch.setitem(_torch_ops._USE_HOST_SCHED, 'on', True)
    monkeypatch.setattr(torch.cuda, 'set_device', lambda d: None)
    monkeypatch.setattr(torch.cuda, 'Event', H._Event)
    monkeypatch.setattr(torch.cuda, 'current_stream', lambda *a: H._Stream())
    monkeypatch.setattr(torch.Tensor, 'pin_memory', lambda self: self)
    env = (env_cls or _MAEnv)(g)
    obs = _RecordingObserver()
    info = env.get_env_info()
    info.update(env_info_over or {})
    config = {k: v for k, v in g['config'].items() if k not in ('device', 'torch_compile')}
    config.update({'device': H._CudaLookingStr('cpu'), 'env_info': info, 'vec_env': env, 'reward_shaper': dict(g['reward_shaper']),
                   'mixed_precision': False, 'b200_cuda_graph': False, 'train_dir': str(tmp_path)})
    config.update(over or {})
    r = Runner(algo_observer=obs)
    r.load({'params': {'seed': 7, 'algo': {'name': algo}, 'model': {'name': 'continuous_a2c_logstd'},
                       'network': network or _network(g), 'config': config}})
    r.params['config']['vec_env'] = env
    agent = r.algo_factory.create(r.algo_name, base_name='ma', params=r.params)
    return agent, obs


@pytest.mark.parametrize('name', ['agent_ma.pt', 'agent_ma_lstm.pt'])
def test_multiagent_agent_host_logic_matches_reference_golden(name, monkeypatch, tmp_path):
    from oracle import ppo_oracle as O
    g = torch.load(os.path.join(GOLDEN, name), weights_only=False)
    agent, obs = _build(monkeypatch, tmp_path, g)
    G, N, Hn = g['G'], g['N'], g['H']
    assert agent.num_agents == G and agent.num_rows == N * G and agent.batch_size == Hn * N * G
    agent.model.load_state_dict(g['init_state'], strict=False)
    agent.init_tensors()
    agent.obs = agent.env_reset()
    fl = O.swap_and_flatten01
    lstm = g['rnn_units'] > 0
    for ep, ref in enumerate(g['epochs_out']):
        obs.steps.clear()
        agent.epoch_num += 1
        agent.train_epoch(noise=g['noise'][ep])
        assert len(obs.steps) == len(ref['steps']) == Hn
        for t, (mine, theirs) in enumerate(zip(obs.steps, ref['steps'])):
            assert torch.equal(mine['done_indices'], theirs['done_indices']), (ep, t)
            assert mine['game_size'] == theirs['game_size'], (ep, t)
            for k in ('game_rewards_mean', 'game_shaped_rewards_mean', 'game_lengths_mean'):
                torch.testing.assert_close(mine[k], theirs[k].reshape(-1), rtol=1e-4, atol=1e-5, msg=lambda m: f'{ep} {t} {k}: {m}')
        ds = ref['dataset']
        assert torch.equal(agent.dones_buf, ref['mb_dones'])
        torch.testing.assert_close(agent.rewards.unsqueeze(2), ref['mb_rewards'], rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(agent.values.unsqueeze(2), ref['mb_values'], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(fl(agent.advs_n), ds['advantages'], rtol=2e-4, atol=2e-5)
        torch.testing.assert_close(fl(agent.returns_n.unsqueeze(2)), ds['returns'], rtol=1e-4, atol=1e-5)
        st = agent.last_stats
        torch.testing.assert_close(st[:, 0], ref['a_losses'], rtol=2e-3, atol=2e-6)
        torch.testing.assert_close(st[:, 1], ref['c_losses'], rtol=2e-3, atol=2e-6)
        torch.testing.assert_close(st[:, 2], ref['entropies'], rtol=1e-4, atol=1e-6)
        assert agent.curr_frames == ref['curr_frames']
        sd = agent.model.state_dict()
        for k in O.param_names(len(g['units']), lstm=lstm):
            torch.testing.assert_close(sd[k], ref['state'][k], rtol=1e-3, atol=2e-5, msg=lambda m: k + ': ' + m)
        assert agent.game_rewards.current_size == ref['game_rewards_size']
        torch.testing.assert_close(agent.game_rewards.mean, ref['game_rewards_mean'].reshape(-1), rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(agent.game_lengths.mean, ref['game_lengths_mean'].reshape(-1), rtol=1e-4, atol=1e-5)


def test_train_loop_counts_frames_per_env_and_scales_the_rates_by_agents(monkeypatch, tmp_path, capsys):
    """a2c_common.py:1686-1705: frame += batch_size each epoch, summaries at frame // agents, rates over agents * time"""
    g = torch.load(os.path.join(GOLDEN, 'agent_ma.pt'), weights_only=False)
    agent, _ = _build(monkeypatch, tmp_path, g, over={'max_epochs': 2, 'print_stats': True})
    scalars = []
    agent.writer = type('W', (), {'add_scalar': lambda self, tag, v, step=None: scalars.append((tag, float(v), step)),
                                  'flush': lambda self: None, 'close': lambda self: None})()
    times = {'sum': 0.5, 'play': 0.25}
    orig = agent.train_epoch

    def epoch():
        res = list(orig(noise=g['noise'][agent.epoch_num - 1]))
        res[1], res[3] = times['play'], times['sum']
        return tuple(res)
    monkeypatch.setattr(agent, 'train_epoch', epoch)
    agent.train()
    G, B = g['G'], g['H'] * g['N'] * g['G']
    assert agent.frame == 2 * B
    fps = {tag: (v, step) for tag, v, step in scalars if tag.startswith('performance/step_inference')}
    assert fps['performance/step_inference_rl_update_fps'] == (pytest.approx(B / (G * times['sum'])), 2 * B // G)
    assert fps['performance/step_inference_fps'] == (pytest.approx(B / (G * times['play'])), 2 * B // G)
    assert f'frames: {2 * B // G}' in capsys.readouterr().out


def test_post_step_ma_matches_its_header_prototype(monkeypatch):
    import test_abi_calls_cpu as ABI
    from rl_games_b200 import ops, _lib
    assert [n for n, _ in _lib.lib.protos['b200rl_post_step_ma_f32']] == [
        'rewards', 'dones', 'dones_is_u8', 'time_outs', 'time_outs_kind', 'values_t', 'valid_t', 'rewards_out_t', 'dones_cur',
        'prev_dones_f32', 'ep_state', 'meter', 'games_to_track', 'scratch', 'tile_status', 'scratch_tiles', 'counters', 'sel_idx',
        'sel_count', 'N', 'agents', 'cfg_host', 'stream']
    rec = ABI._patch(monkeypatch)
    N, G = 3000, 4
    bufs = ops.post_step_ma_buffers(N, G, 'cpu')
    assert bufs[0].numel() == 3 * 4 and bufs[1].numel() == 3 and bufs[3].numel() == 750
    f = lambda *s: torch.zeros(*s)      # noqa: E731
    cfg = ops.ShaperCfg(1.0, 0.0, -1e30, 1e30, 0.99, 0, 1)
    ops.post_step_ma(f(N), torch.zeros(N, dtype=torch.uint8), torch.zeros(N, dtype=torch.uint8), f(N), None, f(N),
                     torch.zeros(N, dtype=torch.uint8), None, f(3, N), torch.zeros(8, dtype=torch.float64), 100, bufs, N, G, cfg)
    assert rec.calls == {'b200rl_post_step_ma_f32': 1}
    assert ctypes.sizeof(cfg) == 28


def test_next_step_autoreset_with_agents_raises_the_reference_error(monkeypatch, tmp_path):
    g = torch.load(os.path.join(GOLDEN, 'agent_ma.pt'), weights_only=False)
    with pytest.raises(ValueError, match='PPO next_step autoreset masking does not support multi-agent envs; '
                                         'wrap the env with a same_step autoreset adapter instead'):
        _build(monkeypatch, tmp_path, g, env_info_over={'autoreset_mode': 'next_step'})


def test_refused_configurations_name_their_reason(monkeypatch, tmp_path):
    """value_size > 1, a central value on the discrete agent and a recurrent critic stay refused, each naming its reason"""
    from rl_games_b200.common import Box, Discrete
    from rl_games_b200.agent_discrete import DiscreteA2CAgent
    g = torch.load(os.path.join(GOLDEN, 'agent_ma.pt'), weights_only=False)
    with pytest.raises(NotImplementedError, match='value_size > 1'):
        _build(monkeypatch, tmp_path, g, env_info_over={'value_size': 2, 'agents': 1})
    cv = {'minibatch_size': 16, 'mini_epochs': 1, 'learning_rate': 5e-4, 'clip_value': True, 'normalize_input': True,
          'network': {'name': 'actor_critic', 'central_value': True, 'mlp': {'units': [8], 'activation': 'elu'},
                      'rnn': {'name': 'lstm', 'units': 8, 'layers': 1}}}
    with pytest.raises(NotImplementedError, match='central value network: a plain MLP'):
        _build(monkeypatch, tmp_path, g, over={'central_value_config': cv})
    base = {'observation_space': Box(-1.0, 1.0, (4,)), 'action_space': Discrete(3), 'agents': 4}
    for extra, over, msg in (({'value_size': 2}, {}, r'^value_size > 1$'), ({}, {'central_value_config': cv}, r'^central_value_config$')):
        config = {'name': 'd', 'env_name': 'x', 'env_info': dict(base, **extra), 'num_actors': 4, 'horizon_length': 8,
                  'minibatch_size': 32, 'mini_epochs': 1, 'normalize_advantage': True, 'normalize_input': False, 'critic_coef': 1,
                  'grad_norm': 1, 'gamma': 0.99, 'tau': 0.95, 'e_clip': 0.2, 'clip_value': False, 'entropy_coef': 0.0,
                  'reward_shaper': {}, 'learning_rate': 1e-3, 'lr_schedule': None, 'device': H._CudaLookingStr('cpu'),
                  'train_dir': str(tmp_path), **over}
        with pytest.raises(NotImplementedError, match=msg):
            DiscreteA2CAgent('d', {'config': config, 'network': {}})


class _MACVEnv(_MAEnv):
    def _o(self, j):
        return {'obs': self.g['obs_tape'][j].clone(), 'states': self.g['state_tape'][j].clone()}

    def reset(self):
        self.i = 0
        return self._o(0)

    def step(self, actions):
        o, rew, done, info = super().step(actions)
        return self._o(self.i % self.g['obs_tape'].shape[0]), rew, done, info

    def get_env_info(self):
        from rl_games_b200.common import Box
        return dict(super().get_env_info(), state_space=Box(-float('inf'), float('inf'), (self.g['S'],)))


def test_central_value_with_agents_matches_reference_golden(monkeypatch, tmp_path):
    """continuous G = 3 with a central value whose critic reads one state row per env: rollout values are each env's critic value on its
    agent rows, the critic trains on agent 0's old values / returns (update_multiagent_tensors order) over envs x horizon rows"""
    from oracle import ppo_oracle as O
    from rl_games_b200.agent_cv import A2CAgentCV
    g = torch.load(os.path.join(GOLDEN, 'agent_ma_cv.pt'), weights_only=False)
    cv_cfg = dict(g['cv_config'])
    cv_cfg['network'] = {'name': 'actor_critic', 'central_value': True,
                         'mlp': {'units': [24, 12], 'activation': 'elu', 'initializer': {'name': 'default'}}}
    agent, obs = _build(monkeypatch, tmp_path, g, over={'central_value_config': cv_cfg}, env_cls=_MACVEnv)
    assert isinstance(agent, A2CAgentCV) and agent.num_agents == g['G']
    cv = agent.central_value_net
    assert cv.N == g['N'] and cv.batch_size == g['N'] * g['H']
    agent.model.load_state_dict(g['init_state'], strict=False)
    cv.load_state_dict(g['cv_init_state'])
    agent.init_tensors()
    agent.obs = agent.env_reset()
    fl = O.swap_and_flatten01
    for ep, ref in enumerate(g['epochs_out']):
        obs.steps.clear()
        agent.epoch_num += 1
        agent.train_epoch(noise=g['noise'][ep][:g['H']])
        for mine, theirs in zip(obs.steps, ref['steps']):
            assert torch.equal(mine['done_indices'], theirs['done_indices'])
            assert mine['game_size'] == theirs['game_size']
        ds, cds = ref['dataset'], ref['cv_dataset']
        torch.testing.assert_close(agent.values.unsqueeze(2), ref['mb_values'], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(fl(agent.advs_n), ds['advantages'], rtol=2e-4, atol=2e-5)
        torch.testing.assert_close(fl(cv.old_values_n).unsqueeze(1), cds['old_values'], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(fl(cv.returns_n).unsqueeze(1), cds['returns'], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(fl(cv.states), cds['obs'], rtol=0, atol=0)
        st = agent.last_stats
        torch.testing.assert_close(st[:, 0], ref['a_losses'], rtol=2e-3, atol=2e-6)
        torch.testing.assert_close(st[:, 1], ref['c_losses'], rtol=2e-3, atol=2e-6)
        sd, csd = agent.model.state_dict(), cv.state_dict()
        for k in O.param_names(len(g['units'])):
            torch.testing.assert_close(sd[k], ref['state'][k], rtol=1e-3, atol=2e-5, msg=lambda m: k + ': ' + m)
        for k in cv.param_names():
            torch.testing.assert_close(csd[k], ref['cv_state'][k], rtol=1e-3, atol=2e-5, msg=lambda m: 'cv ' + k + ': ' + m)
        assert int(csd['running_mean_std.count']) == int(ref['cv_state']['running_mean_std.count'])
        assert cv.lr == pytest.approx(ref['cv_lr'], rel=1e-12)
        torch.testing.assert_close(agent.game_rewards.mean, ref['game_rewards_mean'].reshape(-1), rtol=1e-4, atol=1e-5)


class _MADiscreteEnv(DH._Env):
    def get_env_info(self):
        return dict(super().get_env_info(), agents=self.g['G'])


def test_discrete_agent_with_agents_and_action_masks_matches_reference_golden(monkeypatch, tmp_path):
    """discrete, separate trunks, per-row action masks, G = 4 (the ppo_smac shape) against the reference's run, per step and per epoch"""
    import _torch_ops
    import _torch_ops_ma
    g = torch.load(os.path.join(GOLDEN, 'agent_ma_discrete.pt'), weights_only=False)
    assert g['separate'] and g['use_action_masks'] and g['G'] == 4
    monkeypatch.setattr(DH, '_Env', _MADiscreteEnv)
    obs = _RecordingObserver()
    from rl_games_b200 import runner as R
    orig_runner = R.Runner
    monkeypatch.setattr(R, 'Runner', lambda *a, **kw: orig_runner(algo_observer=obs))
    _torch_ops.install(monkeypatch)
    _torch_ops_ma.install(monkeypatch)
    agent = DH._build(monkeypatch, tmp_path, g, stand_ins=False)
    assert agent.num_agents == 4 and agent.num_rows == g['N'] * 4 and obs.agent is agent
    fl = lambda t: t.transpose(0, 1).reshape(-1, *t.shape[2:])    # noqa: E731
    H_ = g['H']
    for ep, ref in enumerate(g['epochs_out']):
        obs.steps.clear()
        agent.epoch_num += 1
        res = agent.train_epoch(u=g['u'][ep])
        assert len(obs.steps) == H_
        for t, (mine, theirs) in enumerate(zip(obs.steps, ref['steps'])):
            assert torch.equal(mine['done_indices'], theirs['done_indices']), (ep, t)
            assert mine['game_size'] == theirs['game_size'], (ep, t)
            for k in ('game_rewards_mean', 'game_shaped_rewards_mean', 'game_lengths_mean'):
                torch.testing.assert_close(mine[k].float(), theirs[k].reshape(-1).float(), rtol=1e-4, atol=1e-5)
        ds = ref['dataset']
        assert torch.equal(agent.actions, ref['mb_actions'])
        assert torch.equal(fl(agent.action_masks).bool(), ds['action_masks'])
        torch.testing.assert_close(agent.values.unsqueeze(2), ref['mb_values'], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(fl(agent.advs_n), ds['advantages'], rtol=2e-4, atol=2e-5)
        torch.testing.assert_close(torch.stack(res[4]), ref['a_losses'], rtol=2e-3, atol=2e-6)
        torch.testing.assert_close(torch.stack(res[5]), ref['c_losses'], rtol=2e-3, atol=2e-6)
        sd = agent.model.state_dict()
        for k in g['param_order']:
            torch.testing.assert_close(sd[k], ref['state'][k], rtol=1e-3, atol=2e-5, msg=lambda m: k + ': ' + m)
        assert agent.game_rewards.current_size == ref['game_rewards_size']
        torch.testing.assert_close(agent.game_rewards.mean, ref['game_rewards_mean'].reshape(-1), rtol=1e-4, atol=1e-5)
        assert agent.curr_frames == H_ * g['N'] * 4
