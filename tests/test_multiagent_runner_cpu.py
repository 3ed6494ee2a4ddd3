"""The reference's multi-agent PPO YAMLs through its own Runner with `rl_games_b200.register(runner)`, UNCHANGED except for what a launcher
injects (`env_info` / `vec_env` with `agents`, `device`, `max_epochs`, `train_dir`): `ppo_smac.yaml` and every `smac/v1` config train one
epoch (every C-ABI call header-checked, the multi-agent post-step called once per env step) or raise NotImplementedError with the listed
reason.  Skipped when no reference checkout was vendored into oracle/_ref/."""
import math
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import test_abi_calls_cpu as ABI  # noqa: E402
import test_agent_host_cpu as H  # noqa: E402
import test_reference_runner_cpu as RR  # noqa: E402

REF = RR.REF
pytestmark = pytest.mark.skipif(REF is None, reason='reference rl_games not present (oracle/_ref)')
_AGENTS = 2          # per YAML: see the test
# ppo_multiwalker.yaml sets `use_experimental_cv: False` (an actor without a value loss), which the central-value agent does not build for
# any number of agents
_REFUSED_TOP = {'ppo_multiwalker.yaml': 'use_experimental_cv: False'}


def _refusal(rel, c, net):
    """what a YAML needs that is not built, as the reasons the agents give (None: it trains)"""
    if rel in _REFUSED_TOP:
        return _REFUSED_TOP[rel]
    why = []
    if 'cnn' in net:
        why.append("'cnn' networks")
    if 'rnn' in net:
        why.append("'rnn' networks are not supported by the discrete")
    if c.get('central_value_config'):
        why.append('^central_value_config$')
    if net.get('normalization'):
        why.append('normalization:')
    if net.get('mlp', {}).get('initializer', {}).get('name', 'default') != 'default':
        why.append("only the 'default' mlp initializer")
    return '|'.join(why) or None


def _yamls():
    if REF is None:
        return []
    d = os.path.join(REF, 'rl_games', 'configs', 'smac', 'v1')
    return ['ppo_smac.yaml', 'ppo_multiwalker.yaml'] + sorted(os.path.join('smac', 'v1', f) for f in os.listdir(d) if f.endswith('.yaml'))


class _MAEnv(RR._GymEnv):
    def get_env_info(self):
        return dict(super().get_env_info(), agents=_AGENTS)


class _MADiscreteEnv(RR._GymEnvDiscrete):
    def get_action_masks(self):
        return torch.ones(self.N, self.K, dtype=torch.uint8)

    def get_env_info(self):
        return dict(super().get_env_info(), agents=_AGENTS)


class _MACVEnv(RR._GymEnvCV):
    """agent rows of observations, one state row per env"""

    def _o(self):
        return {'obs': torch.zeros(self.N, self.D), 'states': torch.zeros(self.N // _AGENTS, self.S)}

    def get_env_info(self):
        return dict(super().get_env_info(), agents=_AGENTS)


@pytest.mark.parametrize('rel', _yamls())
def test_multiagent_yaml_runs_through_the_reference_runner(rel, monkeypatch, tmp_path):
    import yaml
    for p in (os.path.join(HERE, 'golden', '_stubs'), REF):
        if p not in sys.path:
            sys.path.insert(0, p)
    from rl_games.torch_runner import Runner
    import rl_games_b200
    from rl_games_b200 import agent_discrete
    rec = ABI._patch(monkeypatch)
    monkeypatch.setattr(agent_discrete.DiscreteA2CAgent, '_require_cuda', lambda self: None)
    monkeypatch.setattr(agent_discrete.DiscreteA2CAgent, '_sync', staticmethod(lambda: None))
    cfg = yaml.safe_load(open(os.path.join(REF, 'rl_games', 'configs', rel)))
    c, net = cfg['params']['config'], cfg['params']['network']
    discrete = cfg['params']['algo']['name'] == 'a2c_discrete'
    N, Hn = c['num_actors'], c['horizon_length']
    mb = c.get('minibatch_size') or N * c['minibatch_size_per_env']
    # the fewest agents (at least 2) that make the batch a whole number of minibatches, as the env of each YAML would
    G = mb // math.gcd(Hn * N, mb)
    G = G * (-(-2 // G))
    rows = N * G
    monkeypatch.setattr(sys.modules[__name__], '_AGENTS', G)
    if discrete:
        env = _MADiscreteEnv(rows, 12, 4)
    elif c.get('central_value_config'):
        env = _MACVEnv(rows, 24, 30, 6)
    else:
        env = _MAEnv(rows, 24, 6)
    c.update({'env_info': env.get_env_info(), 'vec_env': env, 'device': 'cpu' if discrete else H._CudaLookingStr('cpu'), 'max_epochs': 1,
              'train_dir': str(tmp_path), 'b200_cuda_graph': False, 'multi_gpu': False})
    c.pop('max_frames', None)
    runner = Runner()
    rl_games_b200.register(runner)
    runner.load(cfg)
    runner.params['config']['vec_env'] = env
    made = []
    orig_create = runner.algo_factory.create
    monkeypatch.setattr(runner.algo_factory, 'create', lambda name, **kw: (made.append(orig_create(name, **kw)), made[-1])[1])
    reason = _refusal(rel, c, net)
    if reason is not None:
        with pytest.raises(NotImplementedError, match=reason):
            runner.run({'train': True, 'play': False, 'checkpoint': None, 'sigma': None})
        return
    runner.run({'train': True, 'play': False, 'checkpoint': None, 'sigma': None})
    agent, = made
    assert agent.num_agents == G and agent.num_rows == rows
    assert agent.epoch_num == 1 and agent.frame == Hn * rows
    assert rec.calls['b200rl_post_step_ma_f32'] == Hn and 'b200rl_post_step_f32' not in rec.calls
    if discrete:
        assert type(agent) is agent_discrete.DiscreteA2CAgent and rec.calls['b200rl_categorical_loss_f32'] > 0
