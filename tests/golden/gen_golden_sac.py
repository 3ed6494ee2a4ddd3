"""Golden runs of the REAL reference SACAgent (rl_games/algos_torch/sac_agent.py) on the CPU against a tape env:

    python tests/golden/gen_golden_sac.py

writes tests/golden/sac_*.pt (committed).  The reference comes unmodified from oracle/_ref (vendored by __graft_entry__.build()); the
only things replaced are its random draws, which are taken from recorded tapes so that another implementation can replay them: the
replay indices (VectorizedReplayBuffer.sample), the rsample noise of the critic-target and actor passes, the rollout's sample() noise
and the warmup's torch.rand.  Each fixture holds the tapes, the initial weights, per-update losses (critic1 / critic2 / actor / alpha
loss, alpha, entropy) and the full checkpoint dict after the run (weights, target weights, the three Adam states, log_alpha, the
replay buffer)."""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)


class SACTapeEnv:
    """tensor env replaying obs / reward / done / time-out tapes; same_step envs report `final_observation`"""

    def __init__(self, obs, rew, done, tout, low, high, autoreset='same_step', final=None):
        self.obs, self.rew, self.done, self.tout, self.final = obs, rew, done, tout, final
        self.low, self.high, self.autoreset = np.asarray(low, np.float32), np.asarray(high, np.float32), autoreset
        self.t = 0

    def reset(self):
        self.t = 0
        return self.obs[0].clone()

    def step(self, actions):
        t = self.t
        self.t += 1
        infos = {'time_outs': self.tout[t].clone()}
        if self.final is not None:
            infos['final_observation'] = self.final[t].clone()
        return self.obs[t + 1].clone(), self.rew[t].clone(), self.done[t].clone(), infos

    def get_env_info(self):
        import gymnasium as gym
        D = self.obs.shape[2]
        info = {'observation_space': gym.spaces.Box(-np.inf, np.inf, (D,), np.float32),
                'action_space': gym.spaces.Box(self.low, self.high, (len(self.low),), np.float32)}
        if self.autoreset != 'same_step':
            info['autoreset_mode'] = self.autoreset
        return info

    def get_env_state(self):
        return None

    def set_env_state(self, s):
        pass

    def set_train_info(self, *a, **kw):
        pass


def make_tapes(T, N, D, seed, p_done=0.2, p_tout=0.4, final=False):
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(T + 1, N, D, generator=g) * 1.3 + 0.2
    rew = torch.randn(T, N, generator=g)
    done = torch.rand(T, N, generator=g) < p_done
    tout = (torch.rand(T, N, generator=g) < p_tout) & done
    fin = torch.randn(T, N, D, generator=g) if final else None
    return obs, rew, done.to(torch.uint8), tout.to(torch.uint8), fin


CASES = {
    # non-unit box, learnable temperature, policy_frequency 2, normalize_input, same_step autoreset with final_observation
    'sac_box_norm_same_step': dict(N=8, D=5, low=[-2.0, -1.0, 0.0], high=[2.0, 3.0, 0.5], units=[32, 16], act='relu', autoreset='same_step',
                                   final=True, cfg={'normalize_input': True, 'policy_frequency': 2, 'learnable_temperature': True,
                                                    'init_alpha': 0.5}),
    # fixed temperature, policy_frequency 1, next_step autoreset with time-outs, elu, replay ring that wraps
    'sac_fixed_alpha_next_step': dict(N=6, D=4, low=[-1.0, -1.0], high=[1.0, 1.0], units=[24, 24], act='elu', autoreset='next_step', final=False,
                                      cfg={'normalize_input': False, 'policy_frequency': 1, 'learnable_temperature': False, 'init_alpha': 0.2,
                                           'replay_buffer_size': 40, 'critic_grad_clip': 0.5}),
}
EPOCHS, WARMUP, STEPS, UPDATES, BATCH = 6, 2, 2, 2, 16


def params_for(case, env, train_dir):
    c = CASES[case]
    config = {'name': case, 'env_name': 'unused', 'reward_shaper': {'scale_value': 0.5, 'shift_value': 0.1}, 'device': 'cpu',
              'mixed_precision': False, 'gamma': 0.97, 'critic_tau': 0.05, 'batch_size': BATCH, 'replay_buffer_size': 1000,
              'num_warmup_steps': WARMUP, 'num_steps_per_episode': STEPS, 'num_updates_per_step': UPDATES, 'num_actors': c['N'],
              'actor_lr': 3e-3, 'critic_lr': 2e-3, 'alpha_lr': 5e-3, 'critic_grad_clip': 5.0, 'max_epochs': EPOCHS,
              'save_replay_buffer': True, 'print_stats': False, 'train_dir': train_dir, 'save_best_after': 10 ** 9,
              'env_info': env.get_env_info(), 'vec_env': env}
    config.update(c['cfg'])
    network = {'name': 'soft_actor_critic', 'separate': True, 'space': {'continuous': {}}, 'log_std_bounds': [-5, 2],
               'mlp': {'units': c['units'], 'activation': c['act'], 'initializer': {'name': 'default'}}}
    return {'seed': 11, 'algo': {'name': 'sac'}, 'model': {'name': 'soft_actor_critic'}, 'network': network, 'config': config}


def make_env(case):
    c = CASES[case]
    T = EPOCHS * STEPS
    obs, rew, done, tout, fin = make_tapes(T, c['N'], c['D'], seed=len(case) * 7, final=c['final'])
    return SACTapeEnv(obs, rew, done, tout, c['low'], c['high'], c['autoreset'], fin)


def run_reference(case):
    from oracle import ref_arm
    ref_arm.import_reference()
    import torch.distributions.normal as tdn
    from rl_games.torch_runner import Runner

    env = make_env(case)
    runner = Runner()
    runner.load({'params': params_for(case, env, tempfile.mkdtemp())})
    runner.params['config']['vec_env'] = env
    agent = runner.algo_factory.create('sac', base_name='golden', params=runner.params)
    init = {'actor': agent.model.sac_network.actor.state_dict(), 'critic': agent.model.sac_network.critic.state_dict(),
            'critic_target': agent.model.sac_network.critic_target.state_dict(), 'log_alpha': agent.log_alpha.detach().clone()}
    init = {k: ({n: v.clone() for n, v in d.items()} if isinstance(d, dict) else d) for k, d in init.items()}

    g = torch.Generator().manual_seed(1234)
    tapes = {'idx': [], 'noise_next': [], 'noise_actor': [], 'noise_roll': [], 'u': []}
    site = {'s': None}
    orig_std = tdn._standard_normal
    orig_sample = tdn.Normal.sample
    orig_rand = torch.rand

    def std_normal(shape, dtype, device):
        e = torch.randn(shape, generator=g, dtype=dtype)
        tapes[site['s']].append(e.clone())
        return e

    def normal_sample(self, sample_shape=torch.Size()):
        with torch.no_grad():
            e = torch.randn(self._extended_shape(sample_shape), generator=g)
            tapes['noise_roll'].append(e.clone())
            return self.loc + e * self.scale

    def rand(*shape, **kw):
        u = orig_rand(*shape, generator=g)
        tapes['u'].append(u.clone())
        return u

    rb = agent.replay_buffer

    def rb_sample(batch_size):
        idxs = torch.randint(0, rb.capacity if rb.full else rb.idx, (batch_size,), generator=g)
        tapes['idx'].append(idxs.clone())
        return rb.obses[idxs], rb.actions[idxs], rb.rewards[idxs], rb.next_obses[idxs], rb.dones[idxs], rb.truncated[idxs]

    rb.sample = rb_sample
    upd_c, upd_a = agent.update_critic, agent.update_actor_and_alpha

    def update_critic(*a, **k):
        site['s'] = 'noise_next'
        return upd_c(*a, **k)

    def update_actor_and_alpha(*a, **k):
        site['s'] = 'noise_actor'
        return upd_a(*a, **k)
    agent.update_critic, agent.update_actor_and_alpha = update_critic, update_actor_and_alpha
    losses = []
    upd = agent.update

    def update(step):
        info, c1, c2 = upd(step)
        row = {'c1': float(c1), 'c2': float(c2)}
        if info is not None:
            a_loss, ent, alpha, alpha_loss = info
            row.update(a_loss=float(a_loss), entropy=float(ent), alpha=float(alpha), alpha_loss=None if alpha_loss is None else float(alpha_loss))
        losses.append(row)
        return info, c1, c2
    agent.update = update

    tdn._standard_normal = std_normal
    tdn.Normal.sample = normal_sample
    torch.rand = rand
    try:
        agent.init_tensors()
        agent.obs = agent.env_reset()
        meters = []
        for _ in range(EPOCHS):
            agent.epoch_num += 1
            agent.train_epoch()
            meters.append((int(agent.game_rewards.current_size), float(agent.game_rewards.get_mean()) if agent.game_rewards.current_size else 0.0,
                           float(agent.game_lengths.get_mean()) if agent.game_lengths.current_size else 0.0))
        agent.frame = EPOCHS * agent.num_frames_per_epoch
        state = agent.get_full_state_weights()
    finally:
        tdn._standard_normal = orig_std
        tdn.Normal.sample = orig_sample
        torch.rand = orig_rand
    state.pop('env_state', None)
    c = CASES[case]
    return {'case': case, 'params': {k: v for k, v in params_for(case, env, '')['config'].items() if k not in ('env_info', 'vec_env')},
            'network': params_for(case, env, '')['network'], 'N': c['N'], 'D': c['D'], 'low': c['low'], 'high': c['high'],
            'autoreset': c['autoreset'], 'env': {'obs': env.obs, 'rew': env.rew, 'done': env.done, 'tout': env.tout, 'final': env.final},
            'init': init, 'tapes': tapes, 'losses': losses, 'meters': meters, 'state': state, 'epochs': EPOCHS}


if __name__ == '__main__':
    for case in CASES:
        out = run_reference(case)
        torch.save(out, os.path.join(HERE, case + '.pt'))
        print(case, len(out['losses']), 'updates;', {k: len(v) for k, v in out['tapes'].items()}, 'meters', out['meters'][-1])
