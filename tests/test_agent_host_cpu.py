"""Host logic of the validated continuous agent (rl_games_b200.agent.A2CAgent, fp32 path, eager) on CPU: every C-ABI op is replaced
by a torch stand-in that restates the kernel's contract (tests/_torch_ops.py) and the agent is run against the reference's golden
runs.  A GPU-less regression net for arena addressing, flat-parameter offsets, call order, the on-device scheduler protocol, meters and
checkpoints; it proves nothing about the kernels (the `-m gpu` suite does)."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')


class _CudaLookingStr(str):
    """'cpu' that answers startswith('cuda'): lets the agent's "CUDA only" guard pass in this one test without touching the product"""

    def __str__(self):
        return self

    def startswith(self, *a):
        return True


class _Event:
    def __init__(self, enable_timing=False):
        pass

    def record(self):
        pass

    def elapsed_time(self, other):
        return 1.0


class _Stream:
    cuda_stream = 0

    def synchronize(self):
        pass


class _Env:
    def __init__(self, g):
        self.g, self.i = g, 0

    def reset(self):
        self.i = 0
        return self.g['obs_tape'][0].clone()

    def step(self, actions):
        g = self.g
        rew = -(actions * actions).sum(-1) * 0.1
        self.i += 1
        j = self.i % g['obs_tape'].shape[0]
        return g['obs_tape'][j].clone(), rew, g['done_tape'][j].clone(), {'time_outs': g['timeout_tape'][j].clone()}

    def get_env_info(self):
        from rl_games_b200.common import Box
        lo, hi = self.g.get('act_bounds', (-1.0, 1.0))
        info = {'observation_space': Box(-np.inf, np.inf, (self.g['D'],)), 'action_space': Box(lo, hi, (self.g['A'],))}
        if self.g['autoreset'] != 'same_step':
            info['autoreset_mode'] = self.g['autoreset']
        return info

    def get_env_state(self):
        return None

    def set_env_state(self, s):
        pass


@pytest.mark.parametrize('name,tc', [('agent_base.pt', False), ('agent_masked.pt', False), ('agent_hardclip.pt', False), ('agent_rmsadv.pt', False),
                                     ('agent_tcshape.pt', False), ('agent_tcshape.pt', True), ('agent_tcshape.pt', 2), ('agent_lstm.pt', False),
                                     ('agent_lstm_after.pt', False), ('agent_sched_standard.pt', False), ('agent_misc.pt', False),
                                     ('agent_rescale.pt', False), ('agent_lstm_masked.pt', False), ('agent_lstm_after_masked.pt', False),
                                     ('agent_minsigma.pt', False), ('agent_separate.pt', False)])
def test_continuous_agent_host_logic_matches_reference_golden(name, tc, monkeypatch, tmp_path):
    """tc=True drives the HOST code of the tcgen05 path (mixed_precision: True: packed-weight bookkeeping, split-partial offsets and
    stride, fused reduce+Adam tail, per-minibatch obs moments merged by the optimiser tail) with fp32 stand-ins for its kernels"""
    import _torch_ops
    from oracle import ppo_oracle as O
    from rl_games_b200.runner import Runner
    if tc:          # tc == 2: the wide-observation edition of the tcgen05 path (scratch buffer for the rollout's layer-1 kernel, gated)
        _torch_ops.install_tc(monkeypatch, kind=int(tc))
    else:
        _torch_ops.install_continuous(monkeypatch)
    # the scheduler step inside the optimiser stand-in is the optimiser kernels' own function compiled for the host (csrc/adam.cu
    # lr_schedule_step: per-minibatch mode and the per-mini-epoch modes of schedule_type 'standard')
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
                   'reward_shaper': dict(g.get('reward_shaper') or {'scale_value': 1.0}), 'mixed_precision': bool(tc), 'b200_cuda_graph': False, 'train_dir': str(tmp_path), 'lr_schedule': cfgk.get('lr_schedule', None)})
    network = {'name': 'actor_critic', 'separate': False,
               'space': {'continuous': {'mu_activation': 'None', 'sigma_activation': 'None', 'mu_init': {'name': 'default'},
                                        'sigma_init': {'name': 'const_initializer', 'val': 0}, 'fixed_sigma': True}},
               'mlp': {'units': g['units'], 'activation': 'elu', 'initializer': {'name': 'default'}}}
    network['space']['continuous'].update(g.get('space_over') or {})          # min_sigma (agent_minsigma.pt)
    network.update(g.get('network_over') or {})                               # separate: True (agent_separate.pt)
    lstm = g.get('rnn_units', 0) > 0
    if lstm:
        network['rnn'] = {'name': 'lstm', 'units': g['rnn_units'], 'layers': 1, 'before_mlp': bool(g.get('rnn_before_mlp', True))}
    r = Runner()
    r.load({'params': {'seed': 7, 'algo': {'name': 'a2c_continuous'}, 'model': {'name': 'continuous_a2c_logstd'}, 'network': network,
                       'config': config}})
    r.params['config']['vec_env'] = env
    agent = r.algo_factory.create(r.algo_name, base_name='parity', params=r.params)
    assert agent.use_tc == bool(tc) and getattr(agent, 'tc_wide', False) == (tc == 2)
    assert agent.model.min_sigma == (g.get('space_over') or {}).get('min_sigma', 0.0)
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
        torch.testing.assert_close(agent.rewards.unsqueeze(2), ref['mb_rewards'], rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(agent.values.unsqueeze(2), ref['mb_values'], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(fl(agent.advs_n), ds['advantages'], rtol=2e-4, atol=2e-5)
        torch.testing.assert_close(fl(agent.returns_n.unsqueeze(2)), ds['returns'], rtol=1e-4, atol=1e-5)
        if ds.get('rnn_masks') is not None:
            assert torch.equal(fl(agent.valid), ds['rnn_masks'])
        st = agent.last_stats
        torch.testing.assert_close(st[:, 0], ref['a_losses'], rtol=2e-3, atol=2e-6)
        torch.testing.assert_close(st[:, 1], ref['c_losses'], rtol=2e-3, atol=2e-6)
        torch.testing.assert_close(st[:, 2], ref['entropies'], rtol=1e-4, atol=1e-6)
        assert agent.last_lr == pytest.approx(ref['last_lr'], rel=1e-12)
        sd = agent.model.state_dict()
        for k in O.param_names(len(g['units']), lstm=lstm, separate=bool((g.get('network_over') or {}).get('separate', False))):
            torch.testing.assert_close(sd[k], ref['state'][k], rtol=1e-3, atol=2e-5, msg=lambda m: k + ': ' + m)
        for pre, key in (('running_mean_std.', 'normalize_input'), ('value_mean_std.', 'normalize_value')):
            if cfgk.get(key, True):
                assert int(sd[pre + 'count']) == int(ref['state'][pre + 'count'])
            else:
                assert pre + 'count' not in sd and pre + 'count' not in ref['state']        # same state-dict key set as the reference
        assert agent.game_rewards.current_size == ref['game_rewards_size']
        torch.testing.assert_close(agent.game_rewards.mean, ref['game_rewards_mean'].reshape(-1), rtol=1e-4, atol=1e-5)
    ck = agent.get_full_state_weights()
    for i, mref in enumerate(g['epochs_out'][-1]['adam_exp_avg']):
        torch.testing.assert_close(ck['optimizer']['state'][i]['exp_avg'].reshape(mref.shape), mref, rtol=1e-3, atol=1e-7)


def _build(monkeypatch, tmp_path, g, env, tc=False, over=None):
    import _torch_ops
    from rl_games_b200.runner import Runner
    (_torch_ops.install_tc if tc else _torch_ops.install_continuous)(monkeypatch)
    monkeypatch.setattr(torch.cuda, 'set_device', lambda d: None)
    monkeypatch.setattr(torch.cuda, 'Event', _Event)
    monkeypatch.setattr(torch.cuda, 'current_stream', lambda *a: _Stream())
    monkeypatch.setattr(torch.Tensor, 'pin_memory', lambda self: self)
    cfgk = g['config']
    config = {k: v for k, v in cfgk.items() if k not in ('device', 'torch_compile')}
    config.update({'device': _CudaLookingStr('cpu'), 'env_info': env.get_env_info(), 'vec_env': env, 'reward_shaper': {'scale_value': 1.0},
                   'mixed_precision': tc, 'b200_cuda_graph': False, 'train_dir': str(tmp_path), 'lr_schedule': cfgk.get('lr_schedule', None)})
    config.update(over or {})
    network = {'name': 'actor_critic', 'separate': False,
               'space': {'continuous': {'mu_activation': 'None', 'sigma_activation': 'None', 'mu_init': {'name': 'default'},
                                        'sigma_init': {'name': 'const_initializer', 'val': 0}, 'fixed_sigma': True}},
               'mlp': {'units': g['units'], 'activation': 'elu', 'initializer': {'name': 'default'}}}
    network['space']['continuous'].update(g.get('space_over') or {})
    network.update(g.get('network_over') or {})
    r = Runner()
    r.load({'params': {'seed': 7, 'algo': {'name': 'a2c_continuous'}, 'model': {'name': 'continuous_a2c_logstd'}, 'network': network,
                       'config': config}})
    r.params['config']['vec_env'] = env
    agent = r.algo_factory.create(r.algo_name, base_name='parity', params=r.params)
    agent.model.load_state_dict(g['init_state'], strict=False)
    agent.init_tensors()
    agent._repack()
    agent.obs = agent.env_reset()
    return agent


class _NumpyEnv(_Env):
    """the same tapes through the HOST-env contract (numpy in / numpy out): exercises the pinned staging path of env_step"""

    def reset(self):
        return super().reset().numpy()

    def step(self, actions):
        assert isinstance(actions, np.ndarray)
        o, r, d, info = super().step(torch.from_numpy(actions))
        return o.numpy(), r.numpy(), d.numpy(), {'time_outs': info['time_outs'].numpy()}


class _NumpyEnv64(_NumpyEnv):
    """what gymnasium MuJoCo vector envs hand over: float64 observations and rewards, bool dones / time-outs (a2c_common.py cast_obs:
    float64 -> float32)"""

    def reset(self):
        return super().reset().astype(np.float64)

    def step(self, actions):
        o, r, d, info = super().step(actions)
        return o.astype(np.float64), r.astype(np.float64), d.astype(bool), {'time_outs': info['time_outs'].astype(bool)}


def test_host_env_path_gives_the_same_epoch_as_the_tensor_env(monkeypatch, tmp_path):
    g = torch.load(os.path.join(GOLDEN, 'agent_masked.pt'), weights_only=False)
    out = []
    for env_cls in (_Env, _NumpyEnv, _NumpyEnv64):
        a = _build(monkeypatch, tmp_path, g, env_cls(g))
        a.epoch_num += 1
        a.train_epoch(noise=g['noise'][0])
        out.append((a.model.flat.clone(), a.rewards.clone(), a.dones_buf.clone(), a.valid.clone()))
        assert a.is_tensor_obses == (env_cls is _Env)
    for other in out[1:]:
        for x, y in zip(out[0], other):
            assert torch.equal(x, y)


def test_reference_style_per_minibatch_api_and_checkpoint_roundtrip(monkeypatch, tmp_path):
    """play_steps -> prepare_dataset -> train_actor_critic(dataset[i]) (the call sequence of the reference's own tests,
    tests/test_ppo_masking.py:92-107) gives the same weights as train_epoch; save / restore round-trips weights, Adam state, lr, epoch"""
    g = torch.load(os.path.join(GOLDEN, 'agent_base.pt'), weights_only=False)
    a = _build(monkeypatch, tmp_path, g, _Env(g))
    b = _build(monkeypatch, tmp_path, g, _Env(g))
    a.epoch_num += 1
    a.train_epoch(noise=g['noise'][0])
    b.epoch_num += 1
    batch = b.play_steps(noise=g['noise'][0])
    assert batch['obses'].shape == (g['N'] * g['H'], g['D']) and batch['played_frames'] == g['N'] * g['H']
    b.set_train()
    b.prepare_dataset(batch)
    for _ in range(b.mini_epochs_num):
        for i in range(len(b.dataset)):
            res = b.train_actor_critic(b.dataset[i])
            assert len(res) == 9
    torch.testing.assert_close(b.model.flat, a.model.flat, rtol=1e-6, atol=1e-7)
    fn = str(tmp_path / 'ck')
    a.save(fn)
    c = _build(monkeypatch, tmp_path, g, _Env(g))
    c.restore(fn + '.pth')
    assert torch.equal(c.model.flat, a.model.flat) and torch.equal(c.model.exp_avg, a.model.exp_avg)
    # like the reference (a2c_common.py:852-866): the optimizer comes back with its lr, the agent's own last_lr is not part of a restore
    assert c.epoch_num == a.epoch_num and c._resume_opt_lr == a.last_lr and c.last_lr == g['config']['learning_rate']
    assert c.get_full_state_weights()['optimizer']['param_groups'][0]['lr'] == a.last_lr
    assert int(c.model.running_mean_std.count) == int(a.model.running_mean_std.count)


def test_train_loop_runs_to_max_epochs_and_saves(monkeypatch, tmp_path):
    """A2CBase.train mirror (a2c_common.py:1662-1782): epoch loop, stats/writer hooks, checkpointing (save_frequency, last checkpoint),
    return value -- on CPU with the kernel stand-ins (noise comes from the mocked Philox-free path: a fixed tape per step)"""
    import _torch_ops
    g = torch.load(os.path.join(GOLDEN, 'agent_base.pt'), weights_only=False)
    a = _build(monkeypatch, tmp_path, g, _Env(g), over={'max_epochs': 3, 'save_frequency': 2, 'save_best_after': 1, 'print_stats': True,
                                                        'name': 'loop'})
    tape = g['noise'][0]
    orig = _torch_ops.policy_head_sample

    def sample_with_tape(*args, **kw):          # train() passes no noise tape: feed one so that the stand-in needs no RNG of its own
        args = list(args)
        if args[7] is None:
            args[7] = tape[int(args[10]) % tape.shape[0]]
        return orig(*args, **kw)
    from rl_games_b200 import ops
    monkeypatch.setattr(ops, 'policy_head_sample', sample_with_tape)
    last_mean, epochs = a.train()
    assert epochs == 3 and a.frame == 3 * g['N'] * g['H']
    assert torch.isfinite(a.model.flat).all()
    files = sorted(os.listdir(a.nn_dir))
    assert any(f.endswith('.pth') for f in files), files


class _TapeManagerEnv:
    """the golden tapes behind mjlab's manager-based API (obs groups, terminated / truncated, an extras dict with a per-burst 'log')"""

    def __init__(self, g):
        self.g, self.i = g, 0
        self.action_space = type('S', (), {'shape': (g['N'], g['A'])})()
        self.extras = {}

    def reset(self):
        self.i = 0
        return {'actor': self.g['obs_tape'][0].clone()}, self.extras

    def step(self, actions):
        g = self.g
        self.i += 1
        j = self.i % g['obs_tape'].shape[0]
        done, trunc = g['done_tape'][j].bool(), g['timeout_tape'][j].bool()
        self.extras['log'] = {'ep_len': done.nonzero().reshape(-1).float()} if bool(done.any()) else {}
        return {'actor': g['obs_tape'][j].clone()}, -(actions * actions).sum(-1) * 0.1, done & ~trunc, trunc, self.extras


def test_manager_based_adapter_and_isaac_observer_in_the_training_loop(monkeypatch, tmp_path):
    """SURVEY 8f rank 4: the adapter's bool dones / time-outs are ingested as they are, the observer sees every step's infos without
    asking for done indices (no per-step sync), and neither changes the epoch"""
    from rl_games_b200.env_adapters import ManagerBasedEnvAdapter
    from rl_games_b200.common import IsaacAlgoObserver
    g = dict(torch.load(os.path.join(GOLDEN, 'agent_masked.pt'), weights_only=False))
    g['done_tape'] = ((g['done_tape'] > 0) | (g['timeout_tape'] > 0)).to(g['done_tape'].dtype)      # truncated implies done in this API
    a = _build(monkeypatch, tmp_path, g, _Env(g))
    env = ManagerBasedEnvAdapter(_TapeManagerEnv(g))
    env.get_env_info = lambda base=env.get_env_info: {**base(), 'autoreset_mode': g['autoreset']}
    b = _build(monkeypatch, tmp_path, g, env, over={'algo_observer': 'isaac'})
    assert isinstance(b.algo_observer, IsaacAlgoObserver) and not b._whole_epoch_graph_ok()
    rows = []
    b.algo_observer.writer = type('W', (), {'add_scalar': lambda self, *r: rows.append(r)})()
    for ag in (a, b):
        ag.epoch_num += 1
        ag.train_epoch(noise=g['noise'][0])
    for x, y in ((a.model.flat, b.model.flat), (a.rewards, b.rewards), (a.dones_buf, b.dones_buf), (a.valid, b.valid)):
        assert torch.equal(x, y)
    H = a.horizon_length
    want = torch.cat([g['done_tape'][j % g['obs_tape'].shape[0]].nonzero().reshape(-1).float() for j in range(1, H + 1)])
    b.algo_observer.after_print_stats(123, 1, 0.5)
    assert rows == [('Episode/ep_len', pytest.approx(want.mean().item(), rel=1e-6), 1)]


def test_mixed_precision_auto_resolves_by_geometry_and_explicit_true_never_downgrades(monkeypatch, tmp_path, capsys):
    """key absent = the reference's 'auto' (a2c_common.py:427-429): tcgen05 path where this build has kernels for the geometry, fp32
    otherwise (with a note); an explicit True on a geometry without fused kernels runs layer by layer on the tensor cores"""
    g = dict(torch.load(os.path.join(GOLDEN, 'agent_base.pt'), weights_only=False))
    a = _build(monkeypatch, tmp_path, g, _Env(g), over={'mixed_precision': None})      # MLP (16, 8): no tcgen05 kernel
    assert a.use_tc is False and a.mixed_precision is False
    assert 'mixed_precision not set -> fp32 kernels' in capsys.readouterr().out
    # an explicit True on a geometry without FUSED kernels is served layer by layer on the tensor cores (gemm_tc), never by fp32 kernels
    c = _build(monkeypatch, tmp_path, g, _Env(g), tc=False, over={'mixed_precision': True})
    assert c.mixed_precision is True and c.use_tc is False and c.gemm_tc is True
    from rl_games_b200 import ops
    c.init_tensors()
    k = c.kernels
    assert k.bwd_weight is ops.linear_bwd_weight_tc and k.fwd.func is ops.linear_fwd_tc and k.bwd_data.func is ops.linear_bwd_data_tc
    # forward and data gradient read their weight operands from the bf16 twin of the parameter arena
    for f in (k.fwd, k.bwd_data):
        assert f.keywords['bf16_arena'][0] is c.model.flat and f.keywords['bf16_arena'][1] is c.wbf
    assert c.wbf.dtype == torch.bfloat16
    g2 = dict(torch.load(os.path.join(GOLDEN, 'agent_tcshape.pt'), weights_only=False))
    import _torch_ops
    _torch_ops.install_tc(monkeypatch)          # its tc_supported stand-in accepts the fixture's small three-layer geometry
    b = _build(monkeypatch, tmp_path, g2, _Env(g2), tc=True, over={'mixed_precision': None})
    assert b.use_tc is True and b.mixed_precision is True
    # a sigma floor is applied on the log-std vector handed to the kernels; the fused kernels read the raw parameter from the packed arena,
    # so a floored policy on a fused geometry is served layer by layer (mixed_precision: True) / by the fp32 kernels (absent key)
    g3 = dict(g2, space_over={'min_sigma': 0.15})
    d = _build(monkeypatch, tmp_path, g3, _Env(g3), tc=True, over={'mixed_precision': True})
    assert d.model.min_sigma == 0.15 and d.use_tc is False and d.gemm_tc is True
    e = _build(monkeypatch, tmp_path, g3, _Env(g3), tc=True, over={'mixed_precision': None})
    assert e.use_tc is False and e.gemm_tc is False and e.mixed_precision is False


@pytest.mark.parametrize('name', ['agent_trainloop.pt', 'agent_trainloop_adaptive.pt'])
def test_train_loop_matches_the_reference_outer_loop(name, monkeypatch, tmp_path):
    """agent.train() against the reference's own train() (a2c_common.py:1662-1782) on the same tapes: frame / epoch accounting, the
    linear schedule driven by FRAMES (max_epochs -1) / the adaptive one, stop on max_frames / max_epochs, periodic / best / final
    checkpoint names, every summary scalar (info/last_lr = the lr of the epoch's LAST minibatch), return value"""
    from oracle import ppo_oracle as O
    g = torch.load(os.path.join(GOLDEN, name), weights_only=False)
    cfgk, ref = g['config'], g['train_loop']
    agent = _build(monkeypatch, tmp_path, g, _Env(g), over={k: cfgk[k] for k in ('max_frames', 'max_epochs', 'save_frequency', 'save_best_after',
                                                                                 'games_to_track') if k in cfgk})
    assert (agent.max_epochs, agent.max_frames) == ((-1, 192) if name == 'agent_trainloop.pt' else (2, -1))
    orig, seen = agent.train_epoch, []

    def with_noise():
        e = agent.epoch_num - 1
        seen.append((agent.frame, agent.epoch_num))
        return orig(noise=g['noise'][e])
    agent.train_epoch = with_noise
    scalars = []
    agent.writer = type('W', (), {'add_scalar': lambda self, tag, v, step=None: scalars.append((tag, float(v), step))})()
    agent.algo_observer.writer = agent.writer
    ret = agent.train()
    # the same summary scalars as the reference, tag for tag and step for step (dashboards keep working); values of everything that is not a
    # wall-clock measurement agree
    assert [(t, s_) for t, _, s_ in scalars if not t.endswith('/time')] == [(t, s_) for t, _, s_ in ref['scalars'] if not t.endswith('/time')]
    assert [t for t, _, _ in scalars] == [t for t, _, _ in ref['scalars']]
    for (t, v, _), (_, rv, _) in zip(scalars, ref['scalars']):
        if not t.startswith('performance/'):
            assert v == pytest.approx(rv, rel=2e-3, abs=2e-6), t
    assert (float(ret[0]), int(ret[1])) == pytest.approx(ref['return'], rel=1e-5)
    assert agent.frame == ref['frame'] and agent.epoch_num == ref['epoch_num']
    assert seen == [(e['frame_before'], e['epoch_num']) for e in g['epochs_out']]
    assert agent.last_lr == pytest.approx(g['epochs_out'][-1]['last_lr'], rel=1e-12)
    assert float(agent.last_mean_rewards) == pytest.approx(ref['last_mean_rewards'], rel=1e-5)
    sd = agent.model.state_dict()
    for k in O.param_names(len(g['units'])):
        torch.testing.assert_close(sd[k], g['epochs_out'][-1]['state'][k], rtol=1e-3, atol=2e-5, msg=lambda m: k + ': ' + m)
    # same files, same name FORMAT (numpy float32 repr of the mean reward); the value itself is a float32 running mean, compared to 1e-5
    import re
    num = re.compile(r'_rew__?(-?[0-9.]+)')
    got, want = sorted(os.listdir(agent.nn_dir)), sorted(n.replace('golden', agent.config['name']) for n in ref['saved'])
    assert [num.sub('_rew_#', n) for n in got] == [num.sub('_rew_#', n) for n in want] and len(got) == len(ref['saved'])
    for a, b in zip(got, want):
        ma, mb_ = num.search(a), num.search(b)
        assert (ma is None) == (mb_ is None)
        if ma:
            assert float(ma.group(1).rstrip('.')) == pytest.approx(float(mb_.group(1).rstrip('.')), rel=1e-5)
            assert len(ma.group(1)) <= len(mb_.group(1)) + 1          # float32 repr, not a 17-digit double


def test_resume_from_a_reference_checkpoint_continues_like_the_reference(monkeypatch, tmp_path):
    """tests/golden/gen_golden.py resume: a checkpoint written by the reference after one epoch, loaded into a FRESH trainer that then
    runs one more epoch.  The product (set_full_state_weights on a fresh agent, env reset, train_epoch) must land where the reference's
    own fresh agent landed: weights, Adam moments and step count, adaptive LR carried over, normaliser statistics, epoch / frame."""
    from oracle import ppo_oracle as O
    g = torch.load(os.path.join(GOLDEN, 'agent_resume.pt'), weights_only=False)
    ref, ck = g['resumed_epoch'], g['checkpoint']
    agent = _build(monkeypatch, tmp_path, g, _Env(g), over={'weight_decay': g['config']['weight_decay']})
    agent.set_full_state_weights(ck)
    # the reference restores the optimizer (lr included) but not its own last_lr: one step on the checkpoint's lr, then the scheduler
    # continues from the configured learning rate (a2c_common.py:852-866)
    assert agent.epoch_num == ck['epoch'] and agent.frame == ck['frame']
    assert agent._resume_opt_lr == g['lr_at_checkpoint'] and agent.last_lr == g['config']['learning_rate']
    agent.obs = agent.env_reset()
    agent.epoch_num += 1
    agent.train_epoch(noise=g['noise'][1])
    assert agent.epoch_num == ref['epoch_num'] and agent.frame == ref['frame']
    assert agent.last_lr == pytest.approx(ref['last_lr'], rel=1e-12)
    torch.testing.assert_close(agent.values.unsqueeze(2), ref['mb_values'], rtol=1e-4, atol=1e-5)
    st = agent.last_stats
    torch.testing.assert_close(st[:, 0], ref['a_losses'], rtol=2e-3, atol=2e-6)
    torch.testing.assert_close(st[:, 1], ref['c_losses'], rtol=2e-3, atol=2e-6)
    sd = agent.model.state_dict()
    for k in O.param_names(len(g['units'])):
        torch.testing.assert_close(sd[k], ref['state'][k], rtol=1e-3, atol=2e-5, msg=lambda m: k + ': ' + m)
    for pre in ('running_mean_std.', 'value_mean_std.'):
        assert int(sd[pre + 'count']) == int(ref['state'][pre + 'count'])
        torch.testing.assert_close(sd[pre + 'running_mean'], ref['state'][pre + 'running_mean'].reshape(-1), rtol=1e-6, atol=1e-7)
    out = agent.get_full_state_weights()
    assert float(out['optimizer']['state'][0]['step']) == ref['adam_step']
    for i, mref in enumerate(ref['adam_exp_avg']):
        torch.testing.assert_close(out['optimizer']['state'][i]['exp_avg'].reshape(mref.shape), mref, rtol=1e-3, atol=1e-7)


def test_poison_flow_of_the_reference_masking_test_runs_through_the_public_api(monkeypatch, tmp_path):
    """call sequence of tests/test_ppo_masking.py:153-175 (play_steps -> edit returns / values of the filler rows -> prepare_dataset ->
    train_actor_critic per minibatch) through the host code: the edited tensors are scattered back into the arena, the masked moments are
    recomputed, and with the stand-ins' exact arithmetic the weights are bit-identical.  The kernels' own claim is the GPU twin
    (tests/test_agent_gpu.py::test_masked_rows_contribute_zero_gradient)."""
    g = torch.load(os.path.join(GOLDEN, 'agent_masked.pt'), weights_only=False)
    results = []
    for poison in (False, True):
        agent = _build(monkeypatch, tmp_path, g, _Env(g))
        agent.play_steps(noise=g['noise'][0])
        batch = agent.play_steps(noise=g['noise'][1])
        garbage = batch['rnn_masks'] == 0.0
        assert 0 < int(garbage.sum()) < garbage.numel()
        if poison:
            batch['returns'] = batch['returns'].clone()
            batch['values'] = batch['values'].clone()
            batch['returns'][garbage] = 1e6
            batch['values'][garbage] = -1e6
        agent.set_train()
        agent.prepare_dataset(batch)
        if poison:
            assert float(agent.returns.max()) == 1e6          # the edit reached the arena
        for _ in range(agent.mini_epochs_num):
            for i in range(len(agent.dataset)):
                agent.train_actor_critic(agent.dataset[i])
        results.append({k: v.clone() for k, v in agent.model.state_dict().items()})
    for k in results[0]:
        assert torch.equal(results[0][k], results[1][k]), k


@pytest.mark.parametrize('activation', ['relu', 'tanh'])
def test_tcgen05_path_takes_relu_and_tanh_networks(activation, monkeypatch, tmp_path):
    """the tcgen05 kernels take the MLP activation as a launch argument (elu / relu / tanh): a relu / tanh network of a supported geometry
    is routed there with mixed_precision: True (or an absent key), the activation id reaches every tcgen05 call, and the host logic
    around the kernels gives the same epoch as the fp32-kernel route (both computed by fp32 torch stand-ins here)"""
    import _torch_ops
    from rl_games_b200 import ops
    from rl_games_b200.runner import Runner
    g = dict(torch.load(os.path.join(GOLDEN, 'agent_tcshape.pt'), weights_only=False))
    seen = []

    def build(mp):
        (_torch_ops.install_tc if mp is not False else _torch_ops.install_continuous)(monkeypatch)
        if mp is not False:
            for name in ('tc_mlp_fwd_train', 'tc_mlp_fwd_rollout', 'tc_mlp_bwd'):
                inner = getattr(ops, name)

                def spy(*a, _inner=inner, _name=name, **k):
                    seen.append((_name, k.get('activation')))
                    return _inner(*a, **k)
                monkeypatch.setattr(ops, name, spy)
        monkeypatch.setattr(torch.cuda, 'set_device', lambda d: None)
        monkeypatch.setattr(torch.cuda, 'Event', _Event)
        monkeypatch.setattr(torch.cuda, 'current_stream', lambda *a: _Stream())
        monkeypatch.setattr(torch.Tensor, 'pin_memory', lambda self: self)
        env = _Env(g)
        config = {k: v for k, v in g['config'].items() if k not in ('device', 'torch_compile')}
        config.update({'device': _CudaLookingStr('cpu'), 'env_info': env.get_env_info(), 'vec_env': env, 'reward_shaper': {'scale_value': 1.0},
                       'mixed_precision': mp, 'b200_cuda_graph': False, 'train_dir': str(tmp_path)})
        network = {'name': 'actor_critic', 'separate': False,
                   'space': {'continuous': {'mu_activation': 'None', 'sigma_activation': 'None', 'mu_init': {'name': 'default'},
                                            'sigma_init': {'name': 'const_initializer', 'val': 0}, 'fixed_sigma': True}},
                   'mlp': {'units': g['units'], 'activation': activation, 'initializer': {'name': 'default'}}}
        r = Runner()
        r.load({'params': {'seed': 7, 'algo': {'name': 'a2c_continuous'}, 'model': {'name': 'continuous_a2c_logstd'}, 'network': network,
                           'config': config}})
        r.params['config']['vec_env'] = env
        a = r.algo_factory.create(r.algo_name, base_name='x', params=r.params)
        a.model.load_state_dict(g['init_state'], strict=False)
        a.init_tensors()
        a._repack()
        a.obs = a.env_reset()
        return a
    assert build(None).use_tc is True
    t = build(True)
    assert t.use_tc is True and t.model.activation == activation
    t.epoch_num += 1
    t.train_epoch(noise=g['noise'][0])
    assert seen and all(act == ops.ACT[activation] for _, act in seen) and {n for n, _ in seen} == {'tc_mlp_fwd_train', 'tc_mlp_fwd_rollout', 'tc_mlp_bwd'}
    f = build(False)
    f.epoch_num += 1
    f.train_epoch(noise=g['noise'][0])
    torch.testing.assert_close(t.model.flat, f.model.flat, rtol=1e-4, atol=2e-6)


class _StridedF64Env(_Env):
    """a tensor env that hands out what torch ops accept but raw-pointer kernels do not: float64 observations that are a strided view
    of a wider buffer, float64 rewards (ADVICE round 1: cast_obs passed such tensors to the kernels by data_ptr)"""

    def _wrap(self, o):
        wide = torch.zeros(o.shape[0], o.shape[1] + 3, dtype=torch.float64)
        wide[:, :o.shape[1]] = o.double()
        return wide[:, :o.shape[1]]

    def reset(self):
        return self._wrap(super().reset())

    def step(self, actions):
        o, r, d, info = super().step(actions)
        return self._wrap(o), r.double(), d, info


def test_tensor_env_with_strided_float64_tensors_is_normalised_once(monkeypatch, tmp_path):
    g = torch.load(os.path.join(GOLDEN, 'agent_base.pt'), weights_only=False)
    out = []
    for env_cls in (_Env, _StridedF64Env):
        a = _build(monkeypatch, tmp_path, g, env_cls(g))
        assert a.obs['obs'].dtype == torch.float32 and a.obs['obs'].is_contiguous()
        a.epoch_num += 1
        a.train_epoch(noise=g['noise'][0])
        out.append((a.model.flat.clone(), a.rewards.clone(), a.obses.clone()))
    for x, y in zip(*out):
        assert torch.equal(x, y)


def test_set_param_reaches_the_device_copies_the_kernels_read(monkeypatch, tmp_path):
    """PBT-style mutations (a2c_common.py set_param): entropy_coef is read by the kernels from device memory, so it must follow under
    lr_schedule 'adaptive' too; mini_epochs_num resizes everything that is sized by the number of updates per epoch"""
    g = torch.load(os.path.join(GOLDEN, 'agent_base.pt'), weights_only=False)
    a = _build(monkeypatch, tmp_path, g, _Env(g))
    assert a.is_adaptive_lr
    a.epoch_num += 1
    a.train_epoch(noise=g['noise'][0])
    a.set_param('entropy_coef', 0.0123)
    assert float(a.entropy_coef_dev) == pytest.approx(0.0123) and float(a.ent_next_dev) == pytest.approx(0.0123)
    assert a.get_param('entropy_coef') == 0.0123
    n0 = a.n_updates
    a.set_param('mini_epochs_num', a.mini_epochs_num + 1)
    assert a.n_updates == n0 + a.num_minibatches and a.stats.shape[0] == a.n_updates and a.host_stats.shape[0] == a.n_updates
    a.epoch_num += 1
    res = a.train_epoch(noise=g['noise'][1])
    assert len(res[4]) == a.n_updates and len(res[8]) == a.mini_epochs_num          # a_losses per update, kls per mini-epoch
    a.set_param('mini_epochs_num', 1)
    a.epoch_num += 1
    res = a.train_epoch(noise=g['noise'][0])
    assert len(res[4]) == a.num_minibatches and a.last_stats.shape[0] == a.num_minibatches


def test_separate_trunks_are_one_block_structured_mlp_whose_zeros_never_move(monkeypatch, tmp_path):
    """separate: True (network_builder.py:494-512) = one MLP of twice the width with block-structured weights (model.py).  After two epochs
    with weight decay, a global-norm clip and an entropy bonus: every structural zero of weights, gradients and both Adam moments is
    still EXACTLY zero (masked gradient -> fixed point of Adam and of weight decay), the state dict has the reference's keys / shapes /
    order, a reference state dict loads into the blocks, and the policy is never routed to the fused kernels (their optimiser tail has no
    place for the mask)."""
    from oracle import ppo_oracle as O
    g = dict(torch.load(os.path.join(GOLDEN, 'agent_separate.pt'), weights_only=False))
    a = _build(monkeypatch, tmp_path, g, _Env(g))
    m = a.model
    assert m.separate and m.trunk_units == g['units'] and m.units == [2 * u for u in g['units']] and not a.use_tc and not a.gemm_tc
    structural = m.grad_mask == 0
    assert int((~structural).sum()) == sum(g['init_state'][k].numel() for k in g['param_order'])
    for ep in range(2):
        a.epoch_num += 1
        a.train_epoch(noise=g['noise'][ep])
    assert float(m.exp_avg.abs().sum()) > 0
    for arena in (m.flat, m.grad, m.exp_avg, m.exp_avg_sq):
        assert float(arena[structural].abs().max()) == 0.0
    sd = m.state_dict()
    assert [k for k in sd if k.startswith('a2c_network')] == O.param_names(len(g['units']), separate=True) == g['param_order']
    ref = g['epochs_out'][-1]['state']
    for k in g['param_order']:
        assert sd[k].shape == ref[k].shape
    m.load_state_dict(ref)                       # a reference checkpoint's model goes into the blocks ...
    for k in g['param_order']:
        assert torch.equal(m.state_dict()[k], ref[k])
    assert float(m.flat[structural].abs().max()) == 0.0          # ... and nowhere else
    # tensor cores: layer by layer (the fused kernels' optimiser tail reduces and steps in one launch: no place for the mask)
    g2 = dict(torch.load(os.path.join(GOLDEN, 'agent_tcshape.pt'), weights_only=False), network_over={'separate': True})
    import _torch_ops
    b = _build(monkeypatch, tmp_path, dict(g2, init_state={}), _Env(g2), tc=True, over={'mixed_precision': True})
    assert b.model.separate and b.use_tc is False and b.gemm_tc is True
