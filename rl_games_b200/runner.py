"""Runner: mirror of rl_games.torch_runner.Runner (torch_runner.py:98-354) for the PPO hot path.

Same surface -- ``Runner(algo_observer=None)``, ``.algo_factory`` / ``.player_factory`` (ObjectFactory),
``.load(yaml_config)`` / ``.load_config(params)`` (seeding, rank discovery, reward shaper + observer
injection), ``.run(args)`` / ``.run_train(args)`` (create -> restore -> override sigma -> train) -- so an
rl_games YAML (``params: {seed, algo, model, network, config}``) runs unchanged with the B200 agent
registered under the reference's algo name ``a2c_continuous``.

When rl_games itself is importable, register the agents into ITS runner instead (INTEGRATION.md):
    rl_games_b200.register(runner)      # = runner.algo_factory.register_builder('a2c_continuous' / 'a2c_discrete', ...)
"""
import os
import random
import time
from copy import deepcopy

import numpy as np
import torch

from .agent import A2CAgent
from .common import ObjectFactory, DefaultAlgoObserver, IsaacAlgoObserver, DefaultRewardsShaper, configurations, register_env
from . import envs  # noqa: F401  (registers the synthetic envs)
from . import env_adapters  # noqa: F401  (registers vecenv type MJLAB)


def _restore(agent, args):
    """torch_runner.py:43-50"""
    if args.get('checkpoint'):
        if args.get('train', True) and args.get('load_critic_only', False):
            if not getattr(agent, 'has_central_value', False):
                raise ValueError('Loading critic only works only for asymmetric actor critic')
            agent.restore_central_value_function(args['checkpoint'])
            return
        agent.restore(args['checkpoint'])


def _override_sigma(agent, args):
    """torch_runner.py:52-60"""
    if args.get('sigma') is not None:
        net = agent.model.a2c_network
        if hasattr(net, 'sigma') and hasattr(net, 'fixed_sigma'):
            if net.fixed_sigma:
                with torch.no_grad():
                    net.sigma.fill_(float(args['sigma']))
            else:
                print('Cannot set new sigma because fixed_sigma is False')


def continuous_agent(**kwargs):
    """Builder for the algo name `a2c_continuous` (a2c_continuous.py:18): `central_value_config` in the YAML selects the
    asymmetric-critic subclass (the reference's A2CAgent builds its CentralValueTrain itself, a2c_common.py:250-262); everything else
    is A2CAgent"""
    if kwargs.get('params', {}).get('config', {}).get('central_value_config') is not None:
        from .agent_cv import A2CAgentCV
        return A2CAgentCV(**kwargs)
    return A2CAgent(**kwargs)


def discrete_agent(**kwargs):
    """Builder for the algo name `a2c_discrete` (a2c_discrete.py:15)"""
    from .agent_discrete import DiscreteA2CAgent
    return DiscreteA2CAgent(**kwargs)


def sac_agent(**kwargs):
    """Builder for the algo name `sac` (sac_agent.py)"""
    from .agent_sac import SACAgent
    return SACAgent(**kwargs)


_continuous_agent, _discrete_agent = continuous_agent, discrete_agent


def register(runner):
    """Put the B200 agents behind the reference's algo names in ANY runner with an `algo_factory` ObjectFactory -- the reference's own
    `rl_games.torch_runner.Runner` (torch_runner.py:117-120) or this module's mirror -- so that stock YAMLs run unchanged."""
    runner.algo_factory.register_builder('a2c_continuous', lambda **kwargs: continuous_agent(**kwargs))
    runner.algo_factory.register_builder('a2c_discrete', lambda **kwargs: discrete_agent(**kwargs))
    return runner


def register_players(runner):
    """Put the CUDA players (rl_games_b200.players) behind the reference's algo names in any runner with a `player_factory`
    ObjectFactory -- the reference's own `rl_games.torch_runner.Runner` (torch_runner.py:122-126) or this module's mirror"""
    from .players import player_builders
    for name, builder in player_builders():
        runner.player_factory.register_builder(name, builder)
    return runner


def register_sac(runner):
    """Put the B200 SAC agent behind the reference's algo name `sac` in any runner with an `algo_factory` ObjectFactory"""
    runner.algo_factory.register_builder('sac', lambda **kwargs: sac_agent(**kwargs))
    return runner


class Runner:
    def __init__(self, algo_observer=None):
        self.algo_factory = ObjectFactory()
        register(self)
        self.player_factory = ObjectFactory()
        register_players(self)
        self._observer_was_injected = algo_observer is not None
        self.algo_observer = algo_observer if algo_observer else DefaultAlgoObserver()

    def reset(self):
        pass

    def load_config(self, params):
        """torch_runner.py:143-226"""
        config = params.get('config', {})
        for module in config.get('import_modules', []):
            __import__(module)
        vecenv_type = config.get('vecenv_type')
        if vecenv_type is not None and config.get('env_name') and config['env_name'] not in configurations:
            register_env(config['env_name'], {'vecenv_type': vecenv_type})
        observer_name = config.get('algo_observer')     # config-driven observer selection; an injected object still wins
        if observer_name and not self._observer_was_injected:
            self.algo_observer = {'default': DefaultAlgoObserver, 'isaac': IsaacAlgoObserver}[observer_name]()
        self.seed = params.get('seed', None)
        if self.seed is None:
            self.seed = int(time.time())
        self.local_rank = self.global_rank = 0
        self.world_size = 1
        if params['config'].get('multi_gpu', False):
            self.local_rank = int(os.getenv('LOCAL_RANK', '0'))
            self.global_rank = int(os.getenv('RANK', '0'))
            self.world_size = int(os.getenv('WORLD_SIZE', '1'))
            self.seed += self.global_rank
            print(f'global_rank = {self.global_rank} local_rank = {self.local_rank} world_size = {self.world_size}')
        print(f'self.seed = {self.seed}')
        self.algo_params = params['algo']
        self.algo_name = self.algo_params['name']
        if self.algo_name == 'sac':
            register_sac(self)
        self.exp_config = None
        if self.seed:
            torch.manual_seed(self.seed)
            if torch.cuda.is_available():
                torch.cuda.manual_seed_all(self.seed)
            np.random.seed(self.seed)
            random.seed(self.seed)
            if 'env_config' in params['config']:
                if 'seed' not in params['config']['env_config']:
                    params['config']['env_config']['seed'] = self.seed
                elif params['config'].get('multi_gpu', False):
                    params['config']['env_config']['seed'] += self.seed
        config = params['config']
        if isinstance(config['reward_shaper'], dict):
            config['reward_shaper'] = DefaultRewardsShaper(**config['reward_shaper'])
        config.setdefault('features', {})
        config['features']['observer'] = self.algo_observer
        params['seed'] = self.seed
        self.params = params

    def load(self, yaml_config):
        config = deepcopy(yaml_config)
        self.default_config = deepcopy(config['params'])
        self.load_config(params=self.default_config)

    def run_train(self, args):
        """torch_runner.py:233-321 minus torch.compile (the hand-written kernels subsume its fusions)."""
        print('Started to train')
        agent = self.algo_factory.create(self.algo_name, base_name='run', params=self.params)
        _restore(agent, args)
        _override_sigma(agent, args)
        return agent.train()

    def run_play(self, args):
        """torch_runner.py:323-334"""
        print('Started to play')
        player = self.create_player()
        _restore(player, args)
        _override_sigma(player, args)
        player.run()

    def create_player(self):
        return self.player_factory.create(self.algo_name, params=self.params)

    def run(self, args):
        if args.get('train', True):
            return self.run_train(args)
        elif args.get('play', False):
            return self.run_play(args)
        return self.run_train(args)
