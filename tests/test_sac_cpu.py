"""SAC host logic without a GPU: the B200 SACAgent on torch stand-ins of its ops (tests/_torch_ops_sac.py) replays the reference's golden
runs (tests/golden/gen_golden_sac.py); state-dict / optimiser layouts and checkpoints interoperate with the reference SACAgent in both
directions; refusals name their reasons; every shipped SAC YAML goes through the reference's own Runner with `register_sac`."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _sac_golden as SG  # noqa: E402
import test_abi_calls_cpu as ABI  # noqa: E402
import test_agent_host_cpu as H  # noqa: E402

ROOT = os.path.dirname(HERE)
REF = os.path.join(ROOT, 'oracle', '_ref')
HAVE_REF = os.path.isdir(os.path.join(REF, 'rl_games'))
needs_ref = pytest.mark.skipif(not HAVE_REF, reason='reference rl_games not present (oracle/_ref)')


def _cpu(monkeypatch):
    import _torch_ops_sac as TS
    TS.install(monkeypatch)
    monkeypatch.setattr(torch.cuda, 'set_device', lambda d: None)


@pytest.mark.parametrize('fixture', SG.FIXTURES)
def test_host_logic_reproduces_the_reference_golden_run(fixture, monkeypatch, tmp_path):
    _cpu(monkeypatch)
    g = SG.load(fixture)
    a = SG.make_agent(g, H._CudaLookingStr('cpu'), tmp_path, over={'mixed_precision': False})
    rows = SG.run(a, g)
    SG.compare(a, g, rows, rtol=1e-4, atol=1e-5)


def _ref_agent(g, tmp_path):
    from oracle import ref_arm
    ref_arm.import_reference()
    import gen_golden_sac as GS
    from rl_games.torch_runner import Runner
    env = GS.make_env(g['case'])
    r = Runner()
    r.load({'params': GS.params_for(g['case'], env, str(tmp_path))})
    r.params['config']['vec_env'] = env
    return r.algo_factory.create('sac', base_name='ref', params=r.params)


@needs_ref
@pytest.mark.parametrize('fixture', SG.FIXTURES)
def test_state_dict_and_optimiser_layout_match_the_reference(fixture, monkeypatch, tmp_path):
    _cpu(monkeypatch)
    g = SG.load(fixture)
    ref = _ref_agent(g, tmp_path / 'r')
    a = SG.make_agent(g, H._CudaLookingStr('cpu'), tmp_path / 'b')
    rs, ms = ref.model.state_dict(), a.model.state_dict()
    assert list(rs) == list(ms)
    for k in rs:
        assert tuple(rs[k].shape) == tuple(ms[k].shape), k
    m = a.model
    for opt, part in (('actor_optimizer', m.actor), ('critic_optimizer', m.critic)):
        ref_params = list((ref.model.sac_network.actor if part is m.actor else ref.model.sac_network.critic).parameters())
        assert [tuple(p.shape) for p in ref_params] == [tuple(v.shape) for v in part.views()], opt
    assert len(ref.log_alpha_optimizer.param_groups[0]['params']) == 1


@needs_ref
def test_initialisation_mirrors_sacbuilder_under_the_same_seed(monkeypatch):
    """same global torch seed -> the same Linear draws in the same construction order -> the same weights"""
    _cpu(monkeypatch)
    from oracle import ref_arm
    ref_arm.import_reference()
    from rl_games.algos_torch.network_builder import SACBuilder
    from rl_games_b200.model_sac import SACModel
    net = {'name': 'soft_actor_critic', 'separate': True, 'space': {'continuous': {}}, 'log_std_bounds': [-5, 2],
           'mlp': {'units': [32, 16], 'activation': 'relu', 'initializer': {'name': 'default'}}}
    b = SACBuilder()
    b.load(net)
    torch.manual_seed(5)
    ref = b.build('sac', obs_dim=7, action_dim=3, actions_num=3, input_shape=(7,), normalize_input=False)
    torch.manual_seed(5)
    m = SACModel(net, 7, 3, 'cpu', False, 1.0)
    sd = m.state_dict()
    for k, v in ref.state_dict().items():
        assert torch.equal(sd['sac_network.' + k], v), k


@needs_ref
@pytest.mark.parametrize('fixture', SG.FIXTURES)
def test_checkpoints_round_trip_through_the_reference_agent(fixture, monkeypatch, tmp_path):
    _cpu(monkeypatch)
    g = SG.load(fixture)
    # reference -> here: the golden run's final checkpoint (what SACAgent.save writes) restores and re-exports unchanged
    torch.save(g['state'], tmp_path / 'ref.pth')
    a = SG.make_agent(g, H._CudaLookingStr('cpu'), tmp_path / 'b')
    a.restore(str(tmp_path / 'ref.pth'))
    mine = a.get_full_state_weights()
    for part in ('actor', 'critic', 'critic_target'):
        for k, v in g['state'][part].items():
            assert torch.equal(mine[part][k], v), k
    assert mine['epoch'] == g['state']['epoch'] and mine['frame'] == g['state']['frame']
    assert torch.equal(mine['log_alpha'], g['state']['log_alpha'])
    for k in ('obses', 'actions', 'rewards', 'next_obses', 'dones', 'truncated', 'idx', 'full'):
        v = g['state']['replay_buffer'][k]
        assert (torch.equal(mine['replay_buffer'][k], v) if torch.is_tensor(v) else mine['replay_buffer'][k] == v), k
    for opt in ('actor_optimizer', 'critic_optimizer', 'log_alpha_optimizer'):
        for i, st in g['state'][opt]['state'].items():
            assert float(mine[opt]['state'][i]['step']) == float(st['step'])
            assert torch.equal(mine[opt]['state'][i]['exp_avg'].reshape(st['exp_avg'].shape), st['exp_avg'])
    # here -> reference: the reference SACAgent.restore accepts what this agent writes
    a.save(str(tmp_path / 'mine'))
    ref = _ref_agent(g, tmp_path / 'r')
    ref.restore(str(tmp_path / 'mine.pth'))
    assert ref.epoch_num == g['state']['epoch'] and ref.frame == g['state']['frame']
    assert torch.equal(ref.log_alpha.detach(), g['state']['log_alpha'])
    for k, v in ref.model.sac_network.critic_target.state_dict().items():
        assert torch.equal(v, g['state']['critic_target'][k]), k
    assert ref.replay_buffer.idx == g['state']['replay_buffer']['idx']
    for i, st in g['state']['critic_optimizer']['state'].items():
        assert torch.equal(ref.critic_optimizer.state_dict()['state'][i]['exp_avg_sq'], st['exp_avg_sq'])


_REFUSALS = {
    'discrete action space': ({'action_space': 'discrete'}, 'discrete action spaces are not supported'),
    'dict observations': ({'observation_space': 'dict'}, 'CNN / dict observations'),
    'multi-agent env': ({'agents': 2}, 'multi-agent SAC'),
    'multi_gpu': ({'multi_gpu': True}, 'multi_gpu'),
    'unknown key': ({'some_unbuilt_option': 1}, 'some_unbuilt_option'),
    'cnn network': ({'cnn': {}}, "'cnn' networks"),
}


@pytest.mark.parametrize('case', list(_REFUSALS))
def test_refusals_name_their_reason(case, monkeypatch, tmp_path):
    _cpu(monkeypatch)
    import gymnasium as gym  # noqa: F401  (the stubs, via tests/golden/_stubs on the path of gen_golden_sac)
    g = SG.load(SG.FIXTURES[0])
    what, msg = _REFUSALS[case]
    over, info, net = {}, None, None
    import copy
    from gen_golden_sac import SACTapeEnv
    e = g['env']
    env = SACTapeEnv(e['obs'], e['rew'], e['done'], e['tout'], g['low'], g['high'], g['autoreset'], e['final'])
    info = env.get_env_info()
    if 'action_space' in what:
        info['action_space'] = gym.spaces.Discrete(4)
    elif 'observation_space' in what:
        info['observation_space'] = {'obs': info['observation_space']}
    elif 'agents' in what:
        info['agents'] = 2
    elif 'cnn' in what:
        net = copy.deepcopy(g['network'])
        net['cnn'] = {}
    else:
        over = dict(what)
    over['env_info'] = info
    with pytest.raises(NotImplementedError, match=msg):
        if net is not None:
            g = dict(g, network=net)
        SG.make_agent(g, H._CudaLookingStr('cpu'), tmp_path, over=over)


def test_register_sac_and_the_runner_hook():
    import rl_games_b200
    from rl_games_b200.common import ObjectFactory
    from rl_games_b200.runner import Runner

    class _R:
        algo_factory = ObjectFactory()
    r = _R()
    assert rl_games_b200.register_sac(r) is r
    assert 'sac' in r.algo_factory._builders
    rr = Runner()
    assert 'sac' not in rr.algo_factory._builders          # register() stays PPO-only; load_config adds `sac` for a SAC config
    rl_games_b200.register(rr)
    assert 'sac' not in rr.algo_factory._builders


# ------------------------------------------------------------------------------------------ every shipped SAC YAML
_SAC_DIMS = {'sac_ant': (105, 8), 'sac_halfcheetah': (17, 6), 'sac_humanoid': (348, 17), 'sac_pendulum': (3, 1)}
_SAC_REFUSED = {'mujoco/sac_ant_tuned.yaml': 'normalization: layer_norm'}      # LayerNorm inside the MLPs: not built


def _shipped_sac_yamls():
    if not HAVE_REF:
        return []
    import yaml
    out = []
    base = os.path.join(REF, 'rl_games', 'configs')
    for d in (base, os.path.join(base, 'mujoco')):
        for f in sorted(os.listdir(d)):
            if f.endswith('.yaml'):
                try:
                    if yaml.safe_load(open(os.path.join(d, f)))['params']['algo']['name'] == 'sac':
                        out.append(os.path.relpath(os.path.join(d, f), base))
                except Exception:
                    continue
    return out


class _SACGymEnv:
    def __init__(self, N, D, A):
        self.N, self.D, self.A = N, D, A

    def reset(self):
        return torch.zeros(self.N, self.D)

    def step(self, actions):
        assert tuple(actions.shape) == (self.N, self.A)
        z8 = torch.zeros(self.N, dtype=torch.uint8)
        return torch.zeros(self.N, self.D), torch.zeros(self.N), z8, {'time_outs': z8}

    def get_env_info(self):
        import gymnasium as gym
        import numpy as np
        return {'observation_space': gym.spaces.Box(-np.inf, np.inf, (self.D,), np.float32),
                'action_space': gym.spaces.Box(-1.0, 1.0, (self.A,), np.float32)}

    def set_train_info(self, *a, **kw):
        pass

    def get_env_state(self):
        return None

    def set_env_state(self, s):
        pass


@pytest.mark.parametrize('rel', _shipped_sac_yamls())
def test_every_shipped_sac_yaml_runs_through_the_reference_runner(rel, monkeypatch, tmp_path):
    """`rl_games_b200.register_sac(runner)` into the reference's own Runner, then each SAC YAML unchanged except for what a launcher
    injects (env, device, train_dir, a short run): one epoch past warmup, every C-ABI call header-checked"""
    import yaml
    for p in (os.path.join(HERE, 'golden', '_stubs'), REF):
        if p not in sys.path:
            sys.path.insert(0, p)
    from rl_games.torch_runner import Runner
    import rl_games_b200
    from rl_games_b200.agent_sac import SACAgent

    rec = ABI._patch(monkeypatch)
    cfg = yaml.safe_load(open(os.path.join(REF, 'rl_games', 'configs', rel)))
    c = cfg['params']['config']
    N = c.get('num_actors', 1)
    D, A = _SAC_DIMS.get(os.path.basename(rel).split('.')[0].replace('_envpool', '').replace('_tuned', ''), (11, 3))
    env = _SACGymEnv(N, D, A)
    c.update({'env_info': env.get_env_info(), 'vec_env': env, 'device': H._CudaLookingStr('cpu'), 'train_dir': str(tmp_path),
              'b200_cuda_graph': False, 'replay_buffer_size': max(N, min(c['replay_buffer_size'], 4096)), 'num_warmup_steps': 1,
              'max_epochs': 2})
    c.pop('num_warmup_frames', None)
    c.pop('max_frames', None)
    runner = Runner()
    assert rl_games_b200.register_sac(runner) is runner
    runner.load(cfg)
    runner.params['config']['vec_env'] = env
    made = []
    orig = runner.algo_factory.create
    monkeypatch.setattr(runner.algo_factory, 'create', lambda name, **kw: (made.append(orig(name, **kw)), made[-1])[1])
    if rel in _SAC_REFUSED:
        with pytest.raises(NotImplementedError, match=_SAC_REFUSED[rel]):
            runner.run({'train': True, 'play': False, 'checkpoint': None, 'sigma': None})
        return
    runner.run({'train': True, 'play': False, 'checkpoint': None, 'sigma': None})
    agent, = made
    assert type(agent) is SACAgent and agent.epoch_num == 2
    n_upd = agent.num_updates_per_step * agent.num_steps_per_episode
    assert rec.calls['b200rl_sac_critic_loss_f32'] == n_upd and rec.calls['b200rl_sac_replay_insert_f32'] == 2 * agent.num_steps_per_episode
    assert rec.calls['b200rl_sac_polyak_f32'] == n_upd
    assert rec.calls.get('b200rl_sac_actor_loss_f32', 0) == n_upd // agent.policy_frequency


class _NumpyEnv:
    """the golden tape env as a numpy env (gym through RayVecEnv, envpool): numpy observations, rewards, dones, infos"""

    def __init__(self, env):
        self.env = env
        self.actions = []

    def __getattr__(self, name):
        return getattr(self.env, name)

    def reset(self):
        return self.env.reset().numpy()

    def step(self, actions):
        import numpy as np
        assert isinstance(actions, np.ndarray)
        self.actions.append(actions.copy())
        o, r, d, info = self.env.step(torch.from_numpy(actions))
        return o.numpy(), r.numpy(), d.numpy(), {k: v.numpy() for k, v in info.items()}


@pytest.mark.parametrize('fixture', SG.FIXTURES)
def test_numpy_env_trains_and_reproduces_the_golden_run(fixture, monkeypatch, tmp_path):
    _cpu(monkeypatch)
    g = SG.load(fixture)
    a = SG.make_agent(g, H._CudaLookingStr('cpu'), tmp_path, over={'mixed_precision': False})
    a.vec_env = _NumpyEnv(a.vec_env)
    rows = SG.run(a, g)
    assert not a._tensor_env and len(a.vec_env.actions) == g['epochs'] * a.num_steps_per_episode
    SG.compare(a, g, rows, rtol=1e-4, atol=1e-5)


def test_next_step_done_indices_are_the_live_done_rows(monkeypatch, tmp_path):
    """sac_agent.py _store_transitions: under next_step, process_infos sees (dones & live).nonzero() -- a row that reports done on the
    step after its episode ended is the reset step's filler and is not reported"""
    _cpu(monkeypatch)
    g = SG.load('sac_fixed_alpha_next_step')
    a = SG.make_agent(g, H._CudaLookingStr('cpu'), tmp_path)
    seen = []
    a.algo_observer.process_infos = lambda infos, idx: seen.append(idx.reshape(-1).tolist())
    done = g['env']['done'].bool()
    done[1] = done[1] | done[0]                    # every row done at step 0 reports done again at step 1
    a.vec_env.done = done.to(torch.uint8)
    SG.run(a, g)
    prev = torch.zeros(done.shape[1], dtype=torch.bool)
    for t, got in enumerate(seen):
        assert got == (done[t] & ~prev).nonzero().reshape(-1).tolist(), t
        prev = done[t]
    assert any(bool((done[t] & done[t - 1]).any()) for t in range(1, len(seen)))
