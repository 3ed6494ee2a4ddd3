"""Host logic of the CUDA players (rl_games_b200.players) on the CPU: the run() loop against the reference's BasePlayer.run on the same
tape env, the actions each player computes from the agents' forward code on the torch stand-ins, the recurrent-state zeroing of finished
rows, the refusals, every C-ABI call against the header, and the play route of both runners.  The kernels themselves are checked on the
GPU (tests/test_players_gpu.py)."""
import contextlib
import io
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _torch_ops_player as P  # noqa: E402
import test_abi_calls_cpu as ABI  # noqa: E402
import test_reference_runner_cpu as RR  # noqa: E402


# ---------------------------------------------------------------------------------------------------------------- the run() loop
class _TapeEnv:
    """rewards and dones from a fixed tape; obs = the step index (batched: [rows, D]; unbatched: [D])"""

    def __init__(self, rows, D, batched, seed=0, steps=40, info=None):
        g = torch.Generator().manual_seed(seed)
        self.rows, self.D, self.batched, self.info = rows, D, batched, info or {}
        self.rew = torch.randint(-3, 4, (steps, rows), generator=g).float()
        self.done = (torch.rand(steps, rows, generator=g) < 0.2).to(torch.uint8)
        self.i = 0

    def reset(self):
        return np.zeros((self.rows, self.D) if self.batched else (self.D,), np.float32)

    def step(self, actions):
        i = self.i % self.rew.shape[0]
        self.i += 1
        obs = np.full((self.rows, self.D) if self.batched else (self.D,), float(self.i), np.float32)
        if not self.batched:
            return obs, float(self.rew[i, 0]), bool(self.done[i, 0]), dict(self.info)
        return obs, self.rew[i].numpy(), self.done[i].numpy(), dict(self.info)


def _loop_attrs(p, env, obs_shape, agents, pc):
    p.env, p.obs_shape, p.num_agents, p.value_size = env, obs_shape, agents, 1
    p.render_env, p.is_deterministic, p.is_rnn, p.is_tensor_obses = False, True, False, False
    p.games_num, p.n_game_life = pc.get('games_num', 5), pc.get('n_game_life', 1)
    p.print_stats, p.balance_env_rewards = pc.get('print_stats', True), pc.get('balance_env_rewards', False)
    p.max_steps, p.batch_size, p.has_batch_dimension = 108000 // 4, 1, False
    p.evaluation, p.dir_to_monitor, p.update_checkpoint_freq = False, None, 100
    p.device = torch.device('cpu')
    p.get_action = lambda obs, det=False: torch.zeros(1)
    return p


def _printed(fn):
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        fn()
    return buf.getvalue()


LOOPS = [dict(rows=1, batched=False), dict(rows=4, batched=True), dict(rows=4, batched=True, agents=2),
         dict(rows=4, batched=True, pc={'balance_env_rewards': True}), dict(rows=3, batched=True, pc={'n_game_life': 2, 'games_num': 7}),
         dict(rows=4, batched=True, info={'battle_won': 1.0}), dict(rows=2, batched=True, info={'scores': 0.25}, pc={'balance_env_rewards': True}),
         dict(rows=1, batched=False, pc={'print_stats': False, 'games_num': 3})]


@pytest.mark.skipif(RR.REF is None, reason='reference rl_games not present (oracle/_ref)')
@pytest.mark.parametrize('case', range(len(LOOPS)))
def test_run_loop_prints_what_the_reference_prints(case):
    for p in (os.path.join(HERE, 'golden', '_stubs'), RR.REF):
        if p not in sys.path:
            sys.path.insert(0, p)
    from rl_games.common.player import BasePlayer as RefPlayer
    from rl_games_b200.players import BasePlayer
    c = LOOPS[case]
    agents, pc = c.get('agents', 1), c.get('pc', {})
    outs = []
    for cls in (RefPlayer, BasePlayer):
        env = _TapeEnv(c['rows'], 3, c['batched'], seed=case, info=c.get('info'))
        p = _loop_attrs(cls.__new__(cls), env, (3,), agents, pc)
        outs.append((_printed(p.run), env.i))
    assert outs[0] == outs[1]
    assert 'av reward:' in outs[1][0]


# ---------------------------------------------------------------------------------------------------------------- players on stand-ins
class _Env:
    def __init__(self, N, D, space, batched=True, obs_space=None, masks=None, seed=0):
        from rl_games_b200.common import Box
        self.N, self.D, self.batched = N, D, batched
        self.space, self.obs_space = space, obs_space or Box(-np.inf, np.inf, (D,))
        self.masks, self.g, self.i = masks, torch.Generator().manual_seed(seed), 0
        self.dones = []

    def _obs(self):
        shp = (self.N,) + tuple(self.obs_space.shape) if self.batched else tuple(self.obs_space.shape)
        if np.dtype(getattr(self.obs_space, 'dtype', np.float32)) == np.uint8:
            return torch.randint(0, 256, shp, generator=self.g, dtype=torch.uint8)
        return torch.randn(shp, generator=self.g)

    def reset(self):
        return self._obs()

    def step(self, actions):
        self.i += 1
        d = (torch.arange(self.N) + self.i) % 3 == 0
        self.dones.append(d)
        return self._obs(), torch.ones(self.N), d.to(torch.uint8), {}

    def has_action_mask(self):
        return self.masks is not None

    def get_action_mask(self):
        return self.masks

    def get_env_info(self):
        return {'observation_space': self.obs_space, 'action_space': self.space}


def _params(algo, env, network, over=None, player=None):
    config = {'env_name': 'tape', 'env_info': env.get_env_info(), 'vec_env': env, 'device_name': 'cpu', 'normalize_input': True,
              'normalize_value': True, 'b200_cuda_graph': False, 'player': {'games_num': 2, 'print_stats': False, **(player or {})}}
    config.update(over or {})
    return {'seed': 3, 'algo': {'name': algo}, 'model': {'name': {'a2c_continuous': 'continuous_a2c_logstd', 'a2c_discrete': 'discrete_a2c',
                                                                  'sac': 'soc'}[algo]},
            'network': network, 'config': config}


@pytest.fixture
def stand_ins(monkeypatch):
    from rl_games_b200 import players
    P.install(monkeypatch)
    monkeypatch.setattr(players.BasePlayer, '_require_cuda', lambda self: None)


def _randomise(model, seed=0):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        model.flat.copy_(torch.randn(model.flat.shape, generator=g) * 0.5)


MLP = {'name': 'actor_critic', 'separate': False, 'space': {'continuous': {'mu_activation': 'None', 'sigma_activation': 'None',
       'mu_init': {'name': 'default'}, 'sigma_init': {'name': 'const_initializer', 'val': 0}, 'fixed_sigma': True}},
       'mlp': {'units': [16, 8], 'activation': 'elu', 'initializer': {'name': 'default'}}}


def _mlp_ref(model, x, units):
    """the trunk's output with the stand-ins' arithmetic: elu MLP on clamp((x - mean) / std, -5, 5)"""
    m = model
    r = m.running_mean_std
    h = torch.clamp((x - r.mean_f32) / r.std_f32, -5.0, 5.0)
    for W, b in zip(m.W, m.b):
        h = torch.nn.functional.elu(h @ W.t() + b)
    return h


def test_continuous_deterministic_action_is_the_rescaled_clamped_mu(stand_ins):
    from rl_games_b200.common import Box
    from rl_games_b200.players import PpoPlayerContinuous
    env = _Env(5, 4, Box(np.array([-2.0, 0.0]), np.array([2.0, 1.0]), (2,)))
    p = PpoPlayerContinuous(_params('a2c_continuous', env, MLP))
    _randomise(p.model)
    p._weights_loaded()
    obs = env.reset()
    p.get_batch_size(obs, 1)
    a = p.get_action(obs, is_deterministic=True)
    mu = (_mlp_ref(p.model, obs, [16, 8]) @ p.model.W_head.t() + p.model.b_head)[:, 1:]
    want = torch.clamp(mu, -1, 1) * (p.actions_high - p.actions_low) / 2 + (p.actions_high + p.actions_low) / 2
    torch.testing.assert_close(a, want, rtol=1e-6, atol=1e-6)
    # sampled: mu + sigma * eps from the noise tape
    p.noise = torch.randn(5, 2)
    p.clip_actions = False
    a = p.get_action(obs, is_deterministic=False)
    torch.testing.assert_close(a, mu + torch.exp(p.model.sigma) * p.noise, rtol=1e-6, atol=1e-6)
    # one unbatched observation: the action comes back squeezed, as the reference's
    env1 = _Env(1, 4, Box(np.array([-2.0, 0.0]), np.array([2.0, 1.0]), (2,)), batched=False)
    p1 = PpoPlayerContinuous(_params('a2c_continuous', env1, MLP))
    o = env1.reset()
    p1.get_batch_size(o, 1)
    assert tuple(p1.get_action(o, True).shape) == (2,)


@pytest.mark.parametrize('before_mlp', [True, False])
def test_lstm_states_of_finished_rows_restart_from_zero(stand_ins, before_mlp):
    from rl_games_b200.common import Box
    from rl_games_b200.players import PpoPlayerContinuous
    net = dict(MLP, rnn={'name': 'lstm', 'units': 8, 'layers': 1, 'before_mlp': before_mlp})
    env = _Env(6, 4, Box(-np.ones(2), np.ones(2), (2,)))
    p = PpoPlayerContinuous(_params('a2c_continuous', env, net, player={'games_num': 12}))
    _randomise(p.model, 1)
    p._weights_loaded()
    ins, outs = [], []
    orig = p._policy_step

    def step(obs, t, noise=None):
        ins.append((p.rnn_h.clone(), p.rnn_c.clone()))      # the state the LSTM step reads: the previous step's, finished rows zeroed
        orig(obs, t, noise)
        outs.append((p.rnn_h.clone(), p.rnn_c.clone()))
    p._policy_step = step
    p.run()
    assert len(outs) >= 4 and any(bool(d.any()) for d in env.dones)
    assert all(float(s.abs().sum()) == 0.0 for s in ins[0])
    for k in range(1, len(outs)):
        keep = 1.0 - env.dones[k - 1].float().unsqueeze(1)
        for s_in, s_out in zip(ins[k], outs[k - 1]):
            assert torch.equal(s_in, s_out * keep)
        assert float(outs[k - 1][0].abs().sum()) > 0


DISCRETE = {'name': 'actor_critic', 'separate': False, 'space': {'discrete': None},
            'mlp': {'units': [16, 8], 'activation': 'relu', 'initializer': {'name': 'default'}}}


@pytest.mark.parametrize('multi', [False, True])
def test_discrete_deterministic_action_is_the_masked_argmax(stand_ins, multi):
    from rl_games_b200.common import Discrete, Tuple
    from rl_games_b200.players import PpoPlayerDiscrete
    sizes = [3, 4] if multi else [5]
    space = Tuple([Discrete(k) for k in sizes]) if multi else Discrete(5)
    K = sum(sizes)
    masks = (torch.rand(6, K, generator=torch.Generator().manual_seed(2)) < 0.6).to(torch.uint8)
    masks[0] = 0                         # an all-masked row plays action 0 in every head
    env = _Env(6, 4, space, masks=masks.numpy())
    net = dict(DISCRETE, space={'multi_discrete' if multi else 'discrete': None})
    params = _params('a2c_discrete', env, net)
    params['model']['name'] = 'multi_discrete_a2c' if multi else 'discrete_a2c'
    p = PpoPlayerDiscrete(params)
    _randomise(p.model, 3)
    obs = env.reset()
    p.get_batch_size(obs, 1)
    a = p.get_masked_action(obs, masks.numpy(), True)
    z = p.r_a[-1][:, 1:]
    want, off = [], 0
    for k in sizes:
        zj = torch.where(masks[:, off:off + k].bool(), z[:, off:off + k], torch.tensor(-1e8))
        want.append((zj - zj.logsumexp(-1, keepdim=True)).argmax(-1))
        off += k
    want = torch.stack(want, -1) if multi else want[0]
    assert torch.equal(a, want)
    assert torch.all(want[0] == 0)


def test_discrete_plays_uint8_frames_through_the_conv_trunk(stand_ins):
    from rl_games_b200.common import Box, Discrete
    from rl_games_b200.players import PpoPlayerDiscrete
    obs_space = Box(0, 255, (12, 12, 4), np.uint8)      # HWC frames, permuted to NCHW by the trunk
    net = dict(DISCRETE, cnn={'type': 'conv2d', 'activation': 'relu', 'initializer': {'name': 'default'},
                              'convs': [{'filters': 4, 'kernel_size': 3, 'strides': 2, 'padding': 0}]})
    env = _Env(3, 0, Discrete(4), obs_space=obs_space)
    p = PpoPlayerDiscrete(_params('a2c_discrete', env, net, over={'normalize_input': False}))
    _randomise(p.model, 4)
    obs = env.reset()
    p.get_batch_size(obs, 1)
    a = p.get_action(obs, True)
    assert p.obs_buf.dtype == torch.uint8
    lay = p.model.actor_conv[0]
    h = torch.relu(torch.nn.functional.conv2d(obs.permute(0, 3, 1, 2).float() / 255.0, lay.W, lay.b, stride=2)).reshape(3, -1)
    for W, b in zip([l.W for l in p.model.actor_mlp[:-1]], [l.b for l in p.model.actor_mlp[:-1]]):
        h = torch.relu(h @ W.t() + b)
    head = p.model.actor_mlp[-1]
    assert torch.equal(a, (h @ head.W.t() + head.b)[:, 1:].argmax(-1))


SAC_NET = {'name': 'soft_actor_critic', 'separate': True, 'space': {'continuous': None},
           'mlp': {'units': [16, 8], 'activation': 'relu', 'initializer': {'name': 'default'}}, 'log_std_bounds': [-5, 2]}


def test_sac_deterministic_action_is_the_rescaled_tanh_mu(stand_ins):
    from rl_games_b200.common import Box
    from rl_games_b200.players import SACPlayer
    env = _Env(4, 3, Box(np.array([-2.0, 0.0]), np.array([2.0, 1.0]), (2,)))
    p = SACPlayer(_params('sac', env, SAC_NET, over={'normalize_input': False}))
    with torch.no_grad():
        p.model.actor.flat.copy_(torch.randn(p.model.actor.flat.shape, generator=torch.Generator().manual_seed(5)))
    obs = env.reset()
    p.get_batch_size(obs, 1)
    a = p.get_action(obs, True)
    h = obs
    for lay in p.model.actor_mlp[:-1]:
        h = torch.relu(h @ lay.W.t() + lay.b)
    mu = (h @ p.model.actor_mlp[-1].W.t() + p.model.actor_mlp[-1].b)[:, :2]
    torch.testing.assert_close(a, (torch.tanh(mu) * p.action_scale + p.action_bias).clamp(p.action_low, p.action_high))


# ---------------------------------------------------------------------------------------------------------------- refusals
@pytest.mark.parametrize('what', ['evaluation', 'dict', 'value_size', 'discrete_rnn', 'model'])
def test_refusals_name_the_key(stand_ins, what):
    from rl_games_b200.common import Box, Discrete
    from rl_games_b200.players import PpoPlayerContinuous, PpoPlayerDiscrete
    env = _Env(2, 4, Box(-np.ones(2), np.ones(2), (2,)))
    params, cls, msg = _params('a2c_continuous', env, MLP), PpoPlayerContinuous, None
    if what == 'evaluation':
        params['config']['player'].update(evaluation=True, dir_to_monitor='/nonexistent')
        msg = 'dir_to_monitor'
    elif what == 'dict':
        info = env.get_env_info()
        info['observation_space'] = type('Dict', (), {'spaces': {}, 'shape': None})()
        params['config']['env_info'] = info
        msg = 'Dict observation'
    elif what == 'value_size':
        params['config']['env_info'] = dict(env.get_env_info(), value_size=2)
        msg = 'value_size'
    elif what == 'discrete_rnn':
        denv = _Env(2, 4, Discrete(3))
        params = _params('a2c_discrete', denv, dict(DISCRETE, rnn={'name': 'lstm', 'units': 8}))
        cls, msg = PpoPlayerDiscrete, "'rnn'"
    else:
        params['model']['name'] = 'continuous_a2c'
        msg = 'continuous_a2c'
    with pytest.raises(NotImplementedError, match=msg):
        cls(params)


# ---------------------------------------------------------------------------------------------------------------- C ABI
def test_player_calls_match_the_header(monkeypatch):
    from rl_games_b200 import players
    from rl_games_b200.common import Box, Discrete
    rec = ABI._patch(monkeypatch)
    monkeypatch.setattr(players.BasePlayer, '_require_cuda', lambda self: None)
    cont = _Env(3, 4, Box(-np.ones(2), np.ones(2), (2,)))
    mlp3 = dict(MLP, mlp={'units': [32, 16, 8], 'activation': 'elu', 'initializer': {'name': 'default'}})     # the fused kernels' geometry
    for net, over in ((mlp3, {}), (mlp3, {'b200_rollout_fp32': True}), (MLP, {'mixed_precision': False}),
                      (dict(MLP, rnn={'name': 'lstm', 'units': 8, 'layers': 1, 'layer_norm': True}), {'mixed_precision': True})):
        p = players.PpoPlayerContinuous(_params('a2c_continuous', cont, net, over))
        o = cont.reset()
        p.get_batch_size(o, 1)
        p.init_rnn()
        p.get_action(o, True)
        p.get_action(o, False)
    disc = _Env(3, 4, Discrete(5), masks=np.ones((3, 5), np.uint8))
    for over in ({}, {'mixed_precision': True}):
        p = players.PpoPlayerDiscrete(_params('a2c_discrete', disc, DISCRETE, over))
        o = disc.reset()
        p.get_batch_size(o, 1)
        p.get_masked_action(o, disc.masks, True)
        p.get_action(o, False)
    p = players.SACPlayer(_params('sac', cont, SAC_NET, {'normalize_input': True}))
    o = cont.reset()
    p.get_batch_size(o, 1)
    p.get_action(o, True)
    for name in ('b200rl_categorical_argmax_f32', 'b200rl_categorical_sample_f32', 'b200rl_tc_mlp_fwd_rollout', 'b200rl_policy_head_sample_f32',
                 'b200rl_rnn_mask_rows_f32', 'b200rl_lstm_cell_ln_fwd_f32', 'b200rl_sac_squash_fwd_f32', 'b200rl_linear_fwd_tc'):
        assert rec.calls.get(name, 0) > 0, name


# ---------------------------------------------------------------------------------------------------------------- play routes
def test_runner_plays_a_checkpoint_this_trainer_wrote(stand_ins, monkeypatch, tmp_path):
    import test_discrete_host_cpu as DH
    from rl_games_b200.runner import Runner
    g = torch.load(os.path.join(HERE, 'golden', 'agent_discrete_masked.pt'), weights_only=False)
    agent = DH._build(monkeypatch, tmp_path, g)
    agent.train_epoch()
    agent.save(str(tmp_path / 'ck'))
    env = DH._Env(g)
    env.has_action_mask = lambda: True
    env.get_action_mask = lambda: env.get_action_masks().numpy()
    net = {'name': 'actor_critic', 'separate': g['separate'], 'space': {'discrete': None},
           'mlp': {'units': g['units'], 'activation': 'relu', 'initializer': {'name': 'default'}}}
    config = {'env_name': 'tape', 'env_info': env.get_env_info(), 'vec_env': env, 'device_name': 'cpu', 'reward_shaper': {},
              'normalize_input': g['config'].get('normalize_input', False), 'normalize_value': g['config'].get('normalize_value', False),
              'b200_cuda_graph': False, 'player': {'games_num': 3}}
    r = Runner()
    r.load({'params': {'seed': 1, 'algo': {'name': 'a2c_discrete'}, 'model': {'name': 'discrete_a2c'}, 'network': net, 'config': config}})
    r.params['config']['vec_env'] = env
    player = r.create_player()
    from rl_games_b200 import runner as runner_mod
    runner_mod._restore(player, {'checkpoint': str(tmp_path / 'ck.pth')})
    for k, v in agent.model.state_dict().items():
        torch.testing.assert_close(player.model.state_dict()[k], v)
    out = _printed(lambda: r.run({'train': False, 'play': True, 'checkpoint': str(tmp_path / 'ck.pth')}))
    assert out.count('reward:') >= 2 and 'av reward:' in out


class _GymEnv:
    """an injected env for the shipped YAMLs: gymnasium-stub spaces (what a reference user passes), every row done every other step"""

    def __init__(self, obs_space, act_space, rows):
        self.obs_space, self.act_space, self.rows, self.i, self.actions = obs_space, act_space, rows, 0, []

    def _obs(self):
        shp = (self.rows,) + tuple(self.obs_space.shape)
        if np.dtype(self.obs_space.dtype) == np.uint8:
            return torch.randint(0, 256, shp, dtype=torch.uint8)
        return torch.randn(shp)

    def reset(self):
        return self._obs()

    def step(self, actions):
        self.actions.append(actions.clone())
        self.i += 1
        return self._obs(), torch.ones(self.rows), torch.full((self.rows,), self.i % 2, dtype=torch.uint8), {}

    def render(self, mode='human'):
        pass

    def get_env_info(self):
        return {'observation_space': self.obs_space, 'action_space': self.act_space}


@pytest.mark.skipif(RR.REF is None, reason='reference rl_games not present (oracle/_ref)')
@pytest.mark.parametrize('rel', ['ppo_cartpole.yaml', 'atari/ppo_pong.yaml', 'sac_pendulum.yaml'])
def test_shipped_yamls_play_through_the_reference_runner(rel, stand_ins, monkeypatch):
    """register_players inside the reference's own Runner, a shipped YAML unchanged but for the injected env and device"""
    import yaml
    for p in (os.path.join(HERE, 'golden', '_stubs'), RR.REF):
        if p not in sys.path:
            sys.path.insert(0, p)
    import gymnasium as gym
    from rl_games.torch_runner import Runner as RefRunner
    import rl_games_b200
    from rl_games_b200 import players
    cfg = yaml.safe_load(open(os.path.join(RR.REF, 'rl_games', 'configs', rel)))
    spaces = {'ppo_cartpole.yaml': (gym.spaces.Box(-np.inf, np.inf, (4,), np.float32), gym.spaces.Discrete(2)),
              'atari/ppo_pong.yaml': (gym.spaces.Box(0, 255, (4, 84, 84), np.uint8), gym.spaces.Discrete(6)),
              'sac_pendulum.yaml': (gym.spaces.Box(-np.inf, np.inf, (3,), np.float32),
                                    gym.spaces.Box(np.array([-2.0], np.float32), np.array([2.0], np.float32), (1,), np.float32))}[rel]
    env = _GymEnv(*spaces, rows=3)
    c = cfg['params']['config']
    c.update({'env_info': env.get_env_info(), 'vec_env': env, 'device_name': 'cpu', 'b200_cuda_graph': False})
    c.setdefault('player', {})['games_num'] = 4
    runner = RefRunner()
    rl_games_b200.register_players(runner)
    runner.load(cfg)
    runner.params['config']['vec_env'] = env
    made = []
    monkeypatch.setattr(players.BasePlayer, 'run', (lambda run: lambda self: (made.append(type(self).__name__), run(self)))(players.BasePlayer.run))
    out = _printed(lambda: runner.run({'train': False, 'play': True, 'checkpoint': None, 'sigma': None}))
    assert made == [{'ppo_cartpole.yaml': 'PpoPlayerDiscrete', 'atari/ppo_pong.yaml': 'PpoPlayerDiscrete',
                     'sac_pendulum.yaml': 'SACPlayer'}[rel]]
    assert 'av reward:' in out and len(env.actions) >= 2


@pytest.mark.skipif(RR.REF is None, reason='reference rl_games not present (oracle/_ref)')
def test_register_players_puts_the_players_into_the_reference_runner():
    for p in (os.path.join(HERE, 'golden', '_stubs'), RR.REF):
        if p not in sys.path:
            sys.path.insert(0, p)
    from rl_games.torch_runner import Runner as RefRunner
    import rl_games_b200
    from rl_games_b200 import players
    r = rl_games_b200.register_players(RefRunner())
    for name, cls in (('a2c_continuous', players.PpoPlayerContinuous), ('a2c_discrete', players.PpoPlayerDiscrete),
                      ('sac', players.SACPlayer)):
        assert r.player_factory._builders[name].__code__.co_names[-1] == cls.__name__
