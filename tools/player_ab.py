"""Per-step act latency of the players: this package eager, this package graph-replayed (b200_cuda_graph), and the reference's player
(rl_games/algos_torch/players.py from oracle/_ref, on the same GPU), alternating arm by arm within each round.

    python tools/player_ab.py [--rounds 5] [--steps 200] [--out results.json]

Shapes: a batch-1 host env (one unbatched numpy observation per step, the action read back to the host: what `run()` does with a single
gym env) and a 4096-row tensor env (observations already on the GPU, the step ends in a device synchronise).  Policies: MLP
[256, 128, 64] (continuous, 8 actions, obs 60), LSTM 256 in front of MLP [256, 128, 64] (continuous), and the Nature CNN + [512] on
4 x 84 x 84 uint8 frames (discrete, 6 actions).  Deterministic actions, mixed_precision as each YAML family sets it (False: fp32 kernels;
the fused MLP kernels under the absent key's auto rule).  Reports the median and [min, max] per step over the rounds, with the GPU name
and power limit read in the same call.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONT = {'mu_activation': 'None', 'sigma_activation': 'None', 'mu_init': {'name': 'default'},
        'sigma_init': {'name': 'const_initializer', 'val': 0}, 'fixed_sigma': True}
MLP = {'units': [256, 128, 64], 'activation': 'elu', 'initializer': {'name': 'default'}}
NATURE = [{'filters': 32, 'kernel_size': 8, 'strides': 4, 'padding': 0}, {'filters': 64, 'kernel_size': 4, 'strides': 2, 'padding': 0},
          {'filters': 64, 'kernel_size': 3, 'strides': 1, 'padding': 0}]
POLICIES = {
    'mlp': dict(algo='a2c_continuous', model='continuous_a2c_logstd', obs=(60,), net={'space': {'continuous': CONT}, 'mlp': MLP}),
    'lstm': dict(algo='a2c_continuous', model='continuous_a2c_logstd', obs=(60,),
                 net={'space': {'continuous': CONT}, 'mlp': MLP, 'rnn': {'name': 'lstm', 'units': 256, 'layers': 1, 'before_mlp': True}}),
    'cnn': dict(algo='a2c_discrete', model='discrete_a2c', obs=(4, 84, 84), frames=True,
                net={'space': {'discrete': None}, 'mlp': {'units': [512], 'activation': 'relu', 'initializer': {'name': 'default'}},
                     'cnn': {'type': 'conv2d', 'permute_input': False, 'activation': 'relu', 'initializer': {'name': 'default'},
                             'convs': NATURE}}),
}


def _spaces(pol, gym):
    if pol.get('frames'):
        obs = gym.spaces.Box(0, 255, pol['obs'], np.uint8)
    else:
        obs = gym.spaces.Box(-np.inf, np.inf, pol['obs'], np.float32)
    act = gym.spaces.Discrete(6) if pol['algo'] == 'a2c_discrete' else gym.spaces.Box(-np.ones(8, np.float32), np.ones(8, np.float32),
                                                                                       (8,), np.float32)
    return obs, act


def _params(pol, spaces, over):
    net = {'name': 'actor_critic', 'separate': False}
    net.update(pol['net'])
    config = {'env_name': 'bench', 'env_info': {'observation_space': spaces[0], 'action_space': spaces[1]}, 'vec_env': None,
              'device_name': 'cuda:0', 'normalize_input': not pol.get('frames'), 'normalize_value': True}
    config.update(over)
    return {'seed': 1, 'algo': {'name': pol['algo']}, 'model': {'name': pol['model']}, 'network': net, 'config': config}


def _make(arm, pol):
    import gymnasium as gym
    spaces = _spaces(pol, gym)
    if arm == 'reference':
        from rl_games.algos_torch.players import PpoPlayerContinuous, PpoPlayerDiscrete
        cls = PpoPlayerDiscrete if pol['algo'] == 'a2c_discrete' else PpoPlayerContinuous
        return cls(_params(pol, spaces, {}))
    from rl_games_b200.players import PpoPlayerContinuous, PpoPlayerDiscrete
    cls = PpoPlayerDiscrete if pol['algo'] == 'a2c_discrete' else PpoPlayerContinuous
    return cls(_params(pol, spaces, {'b200_cuda_graph': arm == 'graph'}))


def _obs(pol, rows, host, g):
    shp = ((rows,) if rows > 1 else ()) + pol['obs']
    if pol.get('frames'):
        o = torch.randint(0, 256, shp, generator=g, dtype=torch.uint8)
    else:
        o = torch.randn(shp, generator=g)
    return o.numpy() if host else o.cuda()


def _time(p, arm, obs_list, host):
    """seconds per step over the list: host obs go through the player's own cast (H2D), the action comes back to the host"""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for o in obs_list:
        x = p.cast_obs(o) if host else o
        with torch.no_grad():
            a = p.get_action(x, True)
        if host:
            a.cpu()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / len(obs_list)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--out', default=None, help='also write the results as JSON here')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'player_ab measures on the GPU'
    from oracle import ref_arm
    ref_arm.import_reference()
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip()
    g = torch.Generator().manual_seed(0)
    results = {'gpu': gpu, 'rounds': a.rounds, 'steps': a.steps, 'unit': 'us per step', 'cases': {}}
    for pname, pol in POLICIES.items():
        for shape, rows, host in (('host_batch1', 1, True), ('tensor_4096', 4096, False)):
            arms = {arm: _make(arm, pol) for arm in ('eager', 'graph', 'reference')}
            obs_list = [_obs(pol, rows, host, g) for _ in range(min(a.steps, 50))]
            for arm, p in arms.items():         # batch detection, RNN states, warm-up (kernel loads, graph capture)
                x = p.cast_obs(obs_list[0]) if host else obs_list[0]
                p.get_batch_size(x, 1)
                if p.is_rnn:
                    p.init_rnn()
                _time(p, arm, obs_list[:5], host)
            steps = (obs_list * (a.steps // len(obs_list) + 1))[:a.steps]
            t = {arm: [] for arm in arms}
            for _ in range(a.rounds):
                for arm, p in arms.items():
                    t[arm].append(_time(p, arm, steps, host) * 1e6)
            case = {arm: {'median': statistics.median(v), 'min': min(v), 'max': max(v)} for arm, v in t.items()}
            results['cases'][f'{pname}/{shape}'] = case
            print(pname, shape, {arm: '%.1f [%.1f, %.1f]' % (c['median'], c['min'], c['max']) for arm, c in case.items()}, flush=True)
    results['gpu_after'] = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                                          text=True).stdout.strip()
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(results, f, indent=1)
    print(json.dumps(results))


if __name__ == '__main__':
    main()
