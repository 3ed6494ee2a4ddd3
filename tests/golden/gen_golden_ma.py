"""Golden runs of the REAL reference on a multi-agent env (env_info['agents'] = G > 1; a2c_common.py:340, :393, :556, :1039-1051).
Same recipe as gen_golden.py (its TapeVecEnv and make_params), with tapes of envs * G rows:

    python tests/golden/gen_golden_ma.py

writes tests/golden/agent_ma.pt (MLP, G = 3), agent_ma_lstm.pt (LSTM before the MLP, G = 3), agent_ma_cv.pt (MLP, G = 3, a central
value reading 10-wide states of one row per env) and agent_ma_discrete.pt (discrete, separate trunks, action masks, G = 4) (committed).  Besides the usual per-epoch
losses, weights and buffers, every fixture records per env step the indices the reference hands to algo_observer.process_infos
(dones.nonzero()[::G]) and its game_rewards / game_shaped_rewards / game_lengths meters after the step.  The done tapes are random per
agent row, so the agents of one env finish on different steps and several envs finish on one step with different agent subsets; the
script asserts that [::G] differs from "the first done row of each env" on some step, which is the part worth testing."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import gen_golden  # noqa: E402


class MATapeVecEnv(gen_golden.TapeVecEnv):
    def get_env_info(self):
        info = super().get_env_info()
        info['agents'] = self.G
        return info


class MACVTapeVecEnv(gen_golden.CVTapeVecEnv):
    """observations of envs * G agent rows, critic states of one row per env"""

    def get_env_info(self):
        info = super().get_env_info()
        info['agents'] = self.G
        return info


_CV_CFG = {'minibatch_size': 16, 'mini_epochs': 3, 'learning_rate': 5e-4, 'clip_value': True, 'normalize_input': True,
           'truncate_grads': True, 'grad_norm': 1.0,
           'network': {'name': 'actor_critic', 'central_value': True,
                       'mlp': {'units': [24, 12], 'activation': 'elu', 'initializer': {'name': 'default'}}}}


def _tapes(T, rows, D, seed, p_done=0.25, p_timeout=0.1):
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(T, rows, D, generator=g) * 1.5 + 0.3
    done = torch.rand(T, rows, generator=g) < p_done
    tout = (torch.rand(T, rows, generator=g) < p_timeout) & done
    return obs, done.to(torch.uint8), tout


def _differs_from_one_per_env(done_tape, G):
    for d in done_tape:
        idx = d.nonzero().reshape(-1)
        sel = idx[::G].tolist()
        first = sorted({int(r) // G: int(r) for r in reversed(idx.tolist())}.values())
        if sel != first:
            return True
    return False


def gen_agent_ma(name, N=4, G=3, H=8, D=6, A=3, units=(16, 8), mb=32, epochs=2, seed=41, rnn_units=0, overrides=None, S=0):
    """S > 0: with a central value whose critic reads S-wide states, one row per env"""
    from rl_games.torch_runner import Runner
    torch.manual_seed(seed)
    np.random.seed(seed)
    rows = N * G
    T = H * epochs + 1
    obs_tape, done_tape, tout_tape = _tapes(T, rows, D, seed)
    assert _differs_from_one_per_env(done_tape[1:], G), 'the tape does not separate [::G] from one row per env'
    state_tape = None
    if S:
        gs = torch.Generator().manual_seed(seed + 7)
        state_tape = torch.randn(T, N, S, generator=gs) * 1.3 - 0.2
        env = MACVTapeVecEnv(obs_tape, state_tape, done_tape, tout_tape)
        overrides = dict(overrides or {}, central_value_config=_CV_CFG)
    else:
        env = MATapeVecEnv(obs_tape, done_tape, tout_tape)
    env.A, env.G = A, G
    params = gen_golden.make_params(N, H, mb, units, overrides, rnn_units)
    params['config']['env_info'] = env.get_env_info()
    shaper_cfg = dict(params['config']['reward_shaper'])
    runner = Runner()
    runner.load({'params': params})
    runner.params['config']['vec_env'] = env
    agent = runner.algo_factory.create(runner.algo_name, base_name='golden', params=runner.params)
    assert agent.num_agents == G and agent.batch_size == H * rows
    g = torch.Generator().manual_seed(seed + 100)
    cvn = agent.central_value_net if S else None
    with torch.no_grad():
        for mdl in (agent.model,) + ((cvn.model,) if S else ()):
            for k, p in mdl.named_parameters():
                if k.endswith('bias') or k.endswith('sigma'):
                    p.add_(torch.randn(p.shape, generator=g) * 0.05)
    init_state = {k: v.clone() for k, v in agent.model.state_dict().items()}
    cv_init_state = {k: v.clone() for k, v in cvn.model.state_dict().items()} if S else None
    noise = torch.randn(epochs, H + 1, rows, A, generator=g)
    counter = {'k': 0}
    orig_normal = torch.normal

    def fake_normal(loc, scale, *a, **kw):
        k = counter['k']
        counter['k'] += 1
        e, n = divmod(k, H + (0 if S else 1))
        return loc + scale * noise[e, n]

    steps = []
    orig_process = agent.algo_observer.process_infos

    def process_infos(infos, done_indices):
        steps.append({'done_indices': done_indices.clone(), 'game_rewards_mean': agent.game_rewards.mean.clone(),
                      'game_shaped_rewards_mean': agent.game_shaped_rewards.mean.clone(),
                      'game_lengths_mean': agent.game_lengths.mean.clone(), 'game_size': agent.game_rewards.current_size})
        return orig_process(infos, done_indices)
    agent.algo_observer.process_infos = process_infos
    torch.normal = fake_normal
    try:
        agent.init_tensors()
        agent.obs = agent.env_reset()
        epochs_out = []
        for ep in range(epochs):
            agent.epoch_num += 1
            steps.clear()
            res = agent.train_epoch()
            step_time, play_time, update_time, total, a_losses, c_losses, b_losses, entropies, kls, last_lr, lr_mul = res
            ds = agent.dataset.values_dict
            epochs_out.append({
                'a_losses': torch.stack([x.detach() for x in a_losses]), 'c_losses': torch.stack([x.detach() for x in c_losses]),
                'entropies': torch.stack([x.detach() for x in entropies]), 'kls': torch.stack([x.detach() for x in kls]),
                'last_lr': agent.last_lr, 'state': {k: v.clone() for k, v in agent.model.state_dict().items()},
                'dataset': {k: (v.clone() if torch.is_tensor(v) else v) for k, v in ds.items() if k != 'rnn_states'},
                'mb_rewards': agent.experience_buffer.tensor_dict['rewards'].clone(),
                'mb_values': agent.experience_buffer.tensor_dict['values'].clone(),
                'mb_dones': agent.experience_buffer.tensor_dict['dones'].clone(),
                'game_rewards_mean': agent.game_rewards.mean.clone(), 'game_rewards_size': agent.game_rewards.current_size,
                'game_lengths_mean': agent.game_lengths.mean.clone(), 'curr_frames': agent.curr_frames,
                'adam_exp_avg': [agent.optimizer.state[p]['exp_avg'].clone() for p in agent.model.parameters()],
                'steps': list(steps),
            })
            if S:
                epochs_out[-1].update({'cv_state': {k: v.clone() for k, v in cvn.model.state_dict().items()}, 'cv_lr': cvn.lr,
                                       'cv_dataset': {k: v.clone() for k, v in cvn.dataset.values_dict.items()
                                                      if k in ('old_values', 'returns', 'obs')}})
            agent.dataset.update_values_dict(None)
        # get_values goes through the critic when there is a central value: no normal draw for it
        assert counter['k'] == epochs * (H + (0 if S else 1)), counter
    finally:
        torch.normal = orig_normal
    gen_golden.save(name, {'N': N, 'G': G, 'H': H, 'D': D, 'A': A, 'units': list(units), 'mb': mb, 'epochs': epochs,
                           'config': {k: v for k, v in params['config'].items() if isinstance(v, (int, float, str, bool, type(None)))},
                           'reward_shaper': shaper_cfg, 'autoreset': 'same_step', 'rnn_units': rnn_units, 'rnn_before_mlp': True,
                           'obs_tape': obs_tape, 'done_tape': done_tape, 'timeout_tape': tout_tape, 'noise': noise,
                           'init_state': init_state, 'epochs_out': epochs_out, 'S': S, 'state_tape': state_tape,
                           'cv_init_state': cv_init_state, 'cv_config': {k: v for k, v in _CV_CFG.items() if k != 'network'} if S else None,
                           'param_order': [k for k, _ in agent.model.named_parameters()]})


def gen_agent_discrete_ma(name, N=4, G=4, H=8, D=5, K=3, mb=64, seed=43):
    """discrete, separate trunks, action masks (the ppo_smac shape) on envs * G rows, through gen_golden.gen_agent_discrete; the
    reference's observer records every step's process_infos indices and meters"""
    from rl_games.common.algo_observer import DefaultAlgoObserver
    steps = []
    orig_info, orig_process = gen_golden.DiscreteTapeVecEnv.get_env_info, DefaultAlgoObserver.process_infos

    def get_env_info(self):
        return dict(orig_info(self), agents=G)

    def process_infos(self, infos, done_indices):
        a = self.algo
        steps.append({'done_indices': done_indices.clone(), 'game_rewards_mean': a.game_rewards.mean.clone(),
                      'game_shaped_rewards_mean': a.game_shaped_rewards.mean.clone(),
                      'game_lengths_mean': a.game_lengths.mean.clone(), 'game_size': a.game_rewards.current_size})
        return orig_process(self, infos, done_indices)
    import oracle.ppo_oracle as PO
    orig_make = PO.make_tapes
    PO.make_tapes = lambda T, rows, D_, seed=0: _tapes(T, rows, D_, seed)
    gen_golden.DiscreteTapeVecEnv.get_env_info = get_env_info
    DefaultAlgoObserver.process_infos = process_infos
    try:
        gen_golden.gen_agent_discrete(name, N=N * G, H=H, D=D, K=K, mb=mb, seed=seed, use_action_masks=True,
                                      overrides={'num_actors': N})
    finally:
        PO.make_tapes = orig_make
        gen_golden.DiscreteTapeVecEnv.get_env_info = orig_info
        DefaultAlgoObserver.process_infos = orig_process
    path = os.path.join(gen_golden.HERE, name)
    fx = torch.load(path, weights_only=False)
    assert _differs_from_one_per_env(fx['done_tape'][1:], G)
    assert len(steps) == fx['epochs'] * H
    fx['N'], fx['G'] = N, G
    for e, ep in enumerate(fx['epochs_out']):
        ep['steps'] = steps[e * H:(e + 1) * H]
    torch.save(fx, path)


def gen_ma():
    gen_agent_ma('agent_ma.pt')
    gen_agent_ma('agent_ma_lstm.pt', seed=42, rnn_units=8, mb=48, overrides={'seq_length': 4})
    gen_agent_ma('agent_ma_cv.pt', seed=44, S=10)
    gen_agent_discrete_ma('agent_ma_discrete.pt')


if __name__ == '__main__':
    gen_ma()
