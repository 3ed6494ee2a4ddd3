"""Golden plays of the REAL reference players (rl_games/algos_torch/players.py: PpoPlayerContinuous, PpoPlayerDiscrete, SACPlayer) on the
CPU:

    python tests/golden/gen_golden_players.py

writes tests/golden/players_<case>.pt (committed).  The reference comes unmodified from oracle/_ref (vendored by
__graft_entry__.build()).  Each case builds the reference player for a network, perturbs its weights and the input normaliser's statistics
away from their initial values, and plays a recorded observation tape (and mask tape) deterministically, T steps of N rows, zeroing the
recurrent states of the rows each step's done tape finishes as BasePlayer.run() does.  A fixture holds the network / config, the model's
state dict (or the SAC checkpoint parts), the tapes, and per step the player's actions, mu / sigma or the masked normalised logits, the
recurrent states after the step, and for discrete heads a `clear` flag per row and head: the top-two masked logit margin exceeds
CLEAR_MARGIN, so the argmax cannot flip under bf16 arithmetic.  tests/test_players_gpu.py replays the tapes through this package's
players.  The printed summary of BasePlayer.run() is checked separately (tests/test_players_cpu.py, against the reference's own run()).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

T, N, D = 6, 8, 10
CLEAR_MARGIN = 0.05          # > the bf16 error of the tensor-core arms on these logits (a few bf16 ulps of O(1) values)
CONT = {'mu_activation': 'None', 'sigma_activation': 'None', 'mu_init': {'name': 'default'},
        'sigma_init': {'name': 'const_initializer', 'val': 0}, 'fixed_sigma': True}
MLP3 = {'units': [64, 32, 16], 'activation': 'elu', 'initializer': {'name': 'default'}}
CONVS = [{'filters': 8, 'kernel_size': 3, 'strides': 2, 'padding': 0}, {'filters': 8, 'kernel_size': 3, 'strides': 1, 'padding': 0}]

CASES = {
    'cont_mlp': dict(algo='a2c_continuous', net={'space': {'continuous': CONT}, 'mlp': MLP3}),
    'cont_lstm_before': dict(algo='a2c_continuous', net={'space': {'continuous': CONT}, 'mlp': MLP3,
                                                         'rnn': {'name': 'lstm', 'units': 32, 'layers': 1, 'before_mlp': True}}),
    'cont_lstm_after': dict(algo='a2c_continuous', net={'space': {'continuous': CONT}, 'mlp': MLP3,
                                                        'rnn': {'name': 'lstm', 'units': 32, 'layers': 1, 'before_mlp': False}}),
    'cont_lstm_ln': dict(algo='a2c_continuous', net={'space': {'continuous': CONT}, 'mlp': MLP3,
                                                     'rnn': {'name': 'lstm', 'units': 32, 'layers': 1, 'before_mlp': True, 'layer_norm': True}}),
    'cont_sdsigma': dict(algo='a2c_continuous', net={'space': {'continuous': dict(CONT, fixed_sigma=False)}, 'mlp': MLP3}),
    'cont_separate': dict(algo='a2c_continuous', net={'separate': True, 'space': {'continuous': CONT}, 'mlp': MLP3}),
    'disc_mlp': dict(algo='a2c_discrete', K=6, net={'space': {'discrete': None}, 'mlp': dict(MLP3, activation='relu')}),
    'disc_masked': dict(algo='a2c_discrete', K=6, masked=True, net={'space': {'discrete': None}, 'mlp': dict(MLP3, activation='relu')}),
    'disc_multi': dict(algo='a2c_discrete', K=[3, 5, 4], masked=True, net={'space': {'multi_discrete': None},
                                                                          'mlp': dict(MLP3, activation='relu')}),
    'disc_cnn': dict(algo='a2c_discrete', K=5, frames=(12, 12, 4), net={
        'space': {'discrete': None}, 'mlp': {'units': [32], 'activation': 'elu', 'initializer': {'name': 'default'}},
        'cnn': {'type': 'conv2d', 'permute_input': True, 'activation': 'relu', 'initializer': {'name': 'default'}, 'convs': CONVS}}),
    'disc_agents2': dict(algo='a2c_discrete', K=6, agents=2, masked=True, net={'separate': True, 'space': {'discrete': None},
                                                                              'mlp': dict(MLP3, activation='relu')}),
    'sac': dict(algo='sac', net={'name': 'soft_actor_critic', 'separate': True, 'space': {'continuous': {}}, 'log_std_bounds': [-5, 2],
                                 'mlp': {'units': [64, 32], 'activation': 'relu', 'initializer': {'name': 'default'}}}),
}
LOW, HIGH = np.array([-2.0, 0.0, -1.0], np.float32), np.array([2.0, 1.0, 3.0], np.float32)


def spaces(c):
    import gymnasium as gym
    if c.get('frames'):
        obs = gym.spaces.Box(0, 255, c['frames'], np.uint8)
    else:
        obs = gym.spaces.Box(-np.inf, np.inf, (D,), np.float32)
    if c['algo'] == 'a2c_discrete':
        K = c['K']
        act = gym.spaces.Tuple([gym.spaces.Discrete(k) for k in K]) if isinstance(K, list) else gym.spaces.Discrete(K)
    else:
        act = gym.spaces.Box(LOW, HIGH, (3,), np.float32)
    return obs, act


def params_for(name, c, env_info):
    net = {'name': 'actor_critic', 'separate': False}
    net.update(c['net'])
    model = {'a2c_continuous': 'continuous_a2c_logstd', 'sac': 'soft_actor_critic',
             'a2c_discrete': 'multi_discrete_a2c' if isinstance(c.get('K'), list) else 'discrete_a2c'}[c['algo']]
    config = {'name': name, 'env_name': 'tape', 'env_info': env_info, 'vec_env': None, 'device_name': 'cpu', 'clip_actions': True,
              'normalize_input': not c.get('frames'), 'normalize_value': c['algo'] != 'sac', 'player': {'deterministic': True}}
    if c['algo'] == 'sac':
        config.update(init_alpha=1.0)
    return {'seed': 5, 'algo': {'name': c['algo']}, 'model': {'name': model}, 'network': net, 'config': config}


def gen(name, c):
    from rl_games.algos_torch.players import PpoPlayerContinuous, PpoPlayerDiscrete, SACPlayer
    torch.manual_seed(sum(map(ord, name)))          # the reference network's initial draws
    obs_space, act_space = spaces(c)
    rows = N
    env_info = {'observation_space': obs_space, 'action_space': act_space, 'agents': c.get('agents', 1), 'value_size': 1}
    params = params_for(name, c, env_info)
    cls = {'a2c_continuous': PpoPlayerContinuous, 'a2c_discrete': PpoPlayerDiscrete, 'sac': SACPlayer}[c['algo']]
    import copy
    p = cls(copy.deepcopy(params))
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():       # weights and normaliser statistics away from their initial values
        for k, v in p.model.state_dict().items():
            if v.dtype.is_floating_point and 'running_mean_std' not in k and 'value_mean_std' not in k:
                v.add_(torch.randn(v.shape, generator=g) * 0.2)
        for mod, size in ((getattr(p.model, 'running_mean_std', None), None), (getattr(p.model, 'value_mean_std', None), None)):
            if mod is not None and hasattr(mod, 'running_mean'):
                mod.running_mean.copy_(torch.randn(mod.running_mean.shape, generator=g) * 0.5)
                mod.running_var.copy_(torch.rand(mod.running_var.shape, generator=g) + 0.5)
    if c.get('frames'):
        obs = torch.randint(0, 256, (T, rows) + tuple(c['frames']), generator=g, dtype=torch.uint8)
    else:
        obs = torch.randn(T, rows, D, generator=g) * 1.5
    dones = (torch.rand(T, rows, generator=g) < 0.3).to(torch.uint8)
    K = sum(c['K']) if isinstance(c.get('K'), list) else c.get('K')
    masks = (torch.rand(T, rows, K, generator=g) < 0.7) if c.get('masked') else None
    if masks is not None:
        masks[:, 0] = False                                     # an all-masked row
    out = {'actions': [], 'mu': [], 'sigma': [], 'logits': [], 'clear': [], 'rnn_h': [], 'rnn_c': []}
    p.has_batch_dimension = False
    p.get_batch_size(obs[0], 1)
    if p.is_rnn:
        p.init_rnn()
    for t in range(T):
        o = obs[t]
        if c['algo'] == 'sac':
            a = p.get_action(o, True)
        else:
            with torch.no_grad():
                res = p.model({'is_train': False, 'prev_actions': None, 'obs': p._preproc_obs(o), 'rnn_states': p.states,
                               **({'action_masks': masks[t]} if masks is not None else {})})
            if c['algo'] == 'a2c_continuous':
                out['mu'].append(res['mus'])
                out['sigma'].append(res['sigmas'])
                a = p.get_action(o, True)
            else:
                lg = res['logits'] if isinstance(res['logits'], (list, tuple)) else [res['logits']]
                clear = []
                for z in lg:
                    top = z.topk(2, dim=-1).values if z.shape[-1] > 1 else torch.cat([z, z - 1.0], -1)
                    clear.append((top[:, 0] - top[:, 1]) > CLEAR_MARGIN)
                out['logits'].append(torch.cat(lg, -1))
                out['clear'].append(torch.stack(clear, -1))
                a = p.get_masked_action(o, masks[t], True) if masks is not None else p.get_action(o, True)
        out['actions'].append(a.detach().clone())
        if p.is_rnn:
            out['rnn_h'].append(p.states[0][0].clone())
            out['rnn_c'].append(p.states[1][0].clone())
            d = dones[t].nonzero(as_tuple=False)
            for s in p.states:
                s[:, d, :] = s[:, d, :] * 0.0
    if c['algo'] == 'sac':
        sn = p.model.sac_network
        state = {'actor': sn.actor.state_dict(), 'critic': sn.critic.state_dict(), 'critic_target': sn.critic_target.state_dict()}
        if p.normalize_input:
            state['running_mean_std'] = p.model.running_mean_std.state_dict()
    else:
        state = {'model': p.model.state_dict()}
    fx = {'algo': c['algo'], 'params': {k: v for k, v in params.items()}, 'state': state, 'obs': obs, 'dones': dones, 'masks': masks,
          'agents': c.get('agents', 1), 'K': c.get('K'), 'frames': c.get('frames'), 'low': LOW, 'high': HIGH}
    fx['params']['config'] = {k: v for k, v in params['config'].items() if k not in ('env_info', 'vec_env')}
    for k, v in out.items():
        fx[k] = torch.stack(v) if v else None
    torch.save(fx, os.path.join(HERE, f'players_{name}.pt'))
    print(name, {k: tuple(v.shape) for k, v in fx.items() if torch.is_tensor(v)})


if __name__ == '__main__':
    from oracle import ref_arm
    ref_arm.import_reference()
    for name, c in CASES.items():
        gen(name, c)
