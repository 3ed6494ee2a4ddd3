"""rl_games_b200 -- the PPO rollout -> GAE -> minibatch-update hot path of Denys88/rl_games as
hand-written sm_90a CUDA behind the reference's plugin surface (Runner / A2CAgent / compute_gae)."""
__version__ = '0.1.0'


def register(runner):
    """rl_games_b200.runner.register: the B200 agents behind `a2c_continuous` / `a2c_discrete` in the given runner's algo_factory
    (imported lazily: the package itself stays importable without torch / the built library)"""
    from .runner import register as _register
    return _register(runner)


def register_sac(runner):
    """rl_games_b200.runner.register_sac: the B200 SAC agent behind `sac` in the given runner's algo_factory"""
    from .runner import register_sac as _register_sac
    return _register_sac(runner)


def register_players(runner):
    """rl_games_b200.runner.register_players: the CUDA players behind `a2c_continuous` / `a2c_discrete` / `sac` in the given runner's
    player_factory"""
    from .runner import register_players as _register_players
    return _register_players(runner)
