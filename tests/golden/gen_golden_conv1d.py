"""Generate the golden runs of the discrete agent with a conv1d trunk by running the REAL reference (see gen_golden.py) on a tape of
frame-stacked fp32 observations, the shape wrappers.BatchedFrameStack gives a smac env (``Box(frames, features)``):

    python tests/golden/gen_golden_conv1d.py

Writes tests/golden/agent_conv1d_separate.pt (separate trunks, action masks, 3 agents per env, the input normaliser, a "same" stack of
k3 s1 p1 convs, default init) and agent_conv1d_shared.pt (a shared trunk whose first conv is strided, k3 s2 p1, glorot init).  The
observations are 4 frames x 24 features; the action draws replay through the same inverse-CDF tape as gen_golden.gen_agent_discrete.

Also writes tests/golden/conv1d_player_disc.pt: the reference's PpoPlayerDiscrete with a separate conv1d trunk, action masks and the
input normaliser, playing a frame-stack tape deterministically, in gen_golden_players.py's fixture format (its observation space is
the rank-2 fp32 `Box(frames, features)`, which the players_*.pt fixtures do not describe, hence the name).
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import gen_golden as G  # noqa: E402  (puts the reference and the import stubs on sys.path)

import numpy as np  # noqa: E402
import torch  # noqa: E402

FRAMES, FEATURES = 4, 24
SAME = [{'filters': 16, 'kernel_size': 3, 'strides': 1, 'padding': 1}, {'filters': 16, 'kernel_size': 3, 'strides': 1, 'padding': 1}]
STRIDED = [{'filters': 8, 'kernel_size': 3, 'strides': 2, 'padding': 1}, {'filters': 16, 'kernel_size': 3, 'strides': 1, 'padding': 0}]


class StackTapeVecEnv(G.DiscreteTapeVecEnv):
    """DiscreteTapeVecEnv on frame stacks [T, rows, frames, features]: the reward is 1 when the action is the argmax of the newest
    frame's first K features; ``agents`` rows per env"""

    def __init__(self, obs_tape, done_tape, timeout_tape, K, mask_tape, agents):
        super().__init__(obs_tape, done_tape, timeout_tape, K, mask_tape)
        self.agents = agents

    def step(self, actions):
        j0 = self.i % self.obs_tape.shape[0]
        rew = (actions.long() == self.obs_tape[j0][:, -1, :self.K].argmax(dim=-1)).float()
        self.i += 1
        j = self.i % self.obs_tape.shape[0]
        return self.obs_tape[j].clone(), rew, self.done_tape[j].clone(), {'time_outs': self.timeout_tape[j].clone()}

    def get_env_info(self):
        import gymnasium as gym
        info = {'observation_space': gym.spaces.Box(-np.inf, np.inf, tuple(self.obs_tape.shape[2:]), np.float32),
                'action_space': gym.spaces.Discrete(self.K)}
        if self.agents > 1:
            info['agents'] = self.agents
        return info


def stack_tape(T, rows, seed):
    """[T, rows, FRAMES, FEATURES] fp32: each step shifts the stack by one frame, as BatchedFrameStack does"""
    g = torch.Generator().manual_seed(seed)
    frames = torch.randn(T + FRAMES - 1, rows, FEATURES, generator=g)
    return torch.stack([frames[t:t + FRAMES].transpose(0, 1) for t in range(T)]).contiguous()


def gen_agent_conv1d(name, convs, separate, agents, normalize_input, use_action_masks, initializer, N=4, H=8, K=5, units=(32,), mb=32,
                     epochs=2, seed=61):
    from rl_games.torch_runner import Runner
    from oracle.ppo_discrete_oracle import sample_inverse_cdf
    torch.manual_seed(seed)
    np.random.seed(seed)
    T, rows = H * epochs + 1, N * agents
    obs_tape = stack_tape(T, rows, seed)
    g = torch.Generator().manual_seed(seed + 100)
    done_tape = (torch.rand(T, rows, generator=g) < 0.1).to(torch.uint8)
    tout_tape = ((torch.rand(T, rows, generator=g) < 0.3) & done_tape.bool()).to(torch.uint8)
    mask_tape = None
    if use_action_masks:
        mask_tape = torch.rand(T, rows, K, generator=g) < 0.6
        mask_tape.scatter_(2, torch.randint(0, K, (T, rows, 1), generator=g), True)
    env = StackTapeVecEnv(obs_tape, done_tape, tout_tape, K, mask_tape, agents)
    network = {'name': 'actor_critic', 'separate': separate, 'space': {'discrete': None},
               'cnn': {'type': 'conv1d', 'activation': 'relu', 'initializer': dict(initializer), 'regularizer': {'name': 'None'},
                       'convs': convs},
               'mlp': {'units': list(units), 'activation': 'relu', 'initializer': dict(initializer), 'regularizer': {'name': 'None'}}}
    config = {'name': 'golden_conv1d', 'env_name': 'unused', 'reward_shaper': {'scale_value': 0.1}, 'normalize_advantage': True,
              'gamma': 0.99, 'tau': 0.95, 'learning_rate': 3e-4, 'grad_norm': 0.5, 'entropy_coef': 0.005, 'truncate_grads': True,
              'e_clip': 0.2, 'clip_value': True, 'num_actors': N, 'horizon_length': H, 'minibatch_size': mb, 'mini_epochs': 2,
              'critic_coef': 2, 'lr_schedule': None, 'kl_threshold': 0.05, 'normalize_input': normalize_input, 'normalize_value': False,
              'device': 'cpu', 'multi_gpu': False, 'mixed_precision': False, 'torch_compile': False, 'max_epochs': 100,
              'save_frequency': 0, 'save_best_after': 10_000, 'print_stats': False, 'train_dir': '/tmp/golden_runs',
              'use_action_masks': use_action_masks}
    params = {'seed': seed, 'algo': {'name': 'a2c_discrete'}, 'model': {'name': 'discrete_a2c'}, 'network': network, 'config': config}
    params['config']['env_info'] = env.get_env_info()
    runner = Runner()
    runner.load({'params': params})
    runner.params['config']['vec_env'] = env
    torch.manual_seed(seed)          # the network's draws from a known state: tests rebuild it from the same seed
    agent = runner.algo_factory.create(runner.algo_name, base_name='golden', params=runner.params)
    assert agent.num_agents == agents and agent.batch_size == H * rows
    seeded_state = {k: v.clone() for k, v in agent.model.state_dict().items()}
    with torch.no_grad():
        for k, p in agent.model.named_parameters():
            if k.endswith('bias'):
                p.add_(torch.randn(p.shape, generator=g) * 0.05)
    init_state = {k: v.clone() for k, v in agent.model.state_dict().items()}
    u = torch.rand(epochs, H + 1, rows, generator=g)
    counter = {'k': 0}
    orig_multinomial = torch.multinomial

    def fake_multinomial(probs_2d, num_samples, replacement=False, **kw):
        k = counter['k']
        counter['k'] += 1
        e, n = divmod(k, H + 1)
        return sample_inverse_cdf(probs_2d, u[e, n]).unsqueeze(-1)
    torch.multinomial = fake_multinomial
    try:
        agent.init_tensors()
        agent.obs = agent.env_reset()
        epochs_out = []
        for ep in range(epochs):
            agent.epoch_num += 1
            res = agent.train_epoch()
            _, _, _, _, a_losses, c_losses, entropies, kls, _, _ = res
            ds = agent.dataset.values_dict
            epochs_out.append({
                'a_losses': torch.stack([x.detach() for x in a_losses]), 'c_losses': torch.stack([x.detach() for x in c_losses]),
                'entropies': torch.stack([x.detach() for x in entropies]), 'kls': torch.stack([x.detach() for x in kls]),
                'last_lr': agent.last_lr, 'state': {k: v.clone() for k, v in agent.model.state_dict().items()},
                'advantages': ds['advantages'].clone(), 'returns': ds['returns'].clone(),
                'old_logp_actions': ds['old_logp_actions'].clone(),
                'mb_rewards': agent.experience_buffer.tensor_dict['rewards'].clone(),
                'mb_values': agent.experience_buffer.tensor_dict['values'].clone(),
                'mb_actions': agent.experience_buffer.tensor_dict['actions'].clone()})
            agent.dataset.update_values_dict(None)
        assert counter['k'] == epochs * (H + 1), counter
    finally:
        torch.multinomial = orig_multinomial
    params_only = lambda sd: {k: v for k, v in sd.items() if k.startswith('a2c_network.')}   # noqa: E731  (fresh normalisers)
    for ep in epochs_out:
        ep['state'] = {k: v.float() if k.startswith('running_mean_std.') and v.dtype == torch.float64 else v
                       for k, v in ep['state'].items()}
    G.save(name, {'N': N, 'agents': agents, 'rows': rows, 'H': H, 'K': K, 'units': list(units), 'mb': mb, 'epochs': epochs,
                  'separate': separate, 'seed': seed, 'network': network, 'use_action_masks': use_action_masks,
                  'config': {k: v for k, v in params['config'].items() if isinstance(v, (int, float, str, bool, type(None)))},
                  'T': T, 'obs_tape': obs_tape, 'done_tape': done_tape, 'timeout_tape': tout_tape, 'mask_tape': mask_tape, 'u': u,
                  'seeded_state': params_only(seeded_state), 'init_state': params_only(init_state), 'epochs_out': epochs_out,
                  'param_order': [k for k, _ in agent.model.named_parameters()]})


def gen_player_conv1d(name='conv1d_player_disc.pt', T=6, N=8, K=6, seed=71):
    """gen_golden_players.gen for a conv1d network on Box(FRAMES, FEATURES): the weights and the normaliser's statistics moved away
    from their initial values, T deterministic masked steps of N rows, the masked logits and a `clear` flag per row (top-two margin
    above gen_golden_players.CLEAR_MARGIN, so the argmax cannot flip under bf16 arithmetic)"""
    import copy
    import gymnasium as gym
    import gen_golden_players as GP
    from rl_games.algos_torch.players import PpoPlayerDiscrete
    torch.manual_seed(seed)
    obs_space = gym.spaces.Box(-np.inf, np.inf, (FRAMES, FEATURES), np.float32)
    env_info = {'observation_space': obs_space, 'action_space': gym.spaces.Discrete(K), 'agents': 1, 'value_size': 1}
    net = {'name': 'actor_critic', 'separate': True, 'space': {'discrete': None},
           'cnn': {'type': 'conv1d', 'activation': 'relu', 'initializer': {'name': 'default'}, 'convs': STRIDED},
           'mlp': {'units': [32], 'activation': 'relu', 'initializer': {'name': 'default'}}}
    config = {'name': 'conv1d_player', 'env_name': 'tape', 'env_info': env_info, 'vec_env': None, 'device_name': 'cpu',
              'clip_actions': True, 'normalize_input': True, 'normalize_value': True, 'player': {'deterministic': True}}
    params = {'seed': 5, 'algo': {'name': 'a2c_discrete'}, 'model': {'name': 'discrete_a2c'}, 'network': net, 'config': config}
    p = PpoPlayerDiscrete(copy.deepcopy(params))
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():
        for k, v in p.model.state_dict().items():
            if v.dtype.is_floating_point and 'running_mean_std' not in k and 'value_mean_std' not in k:
                v.add_(torch.randn(v.shape, generator=g) * 0.2)
        for mod in (p.model.running_mean_std, p.model.value_mean_std):
            mod.running_mean.copy_(torch.randn(mod.running_mean.shape, generator=g) * 0.5)
            mod.running_var.copy_(torch.rand(mod.running_var.shape, generator=g) + 0.5)
    obs = torch.randn(T, N, FRAMES, FEATURES, generator=g) * 1.5
    dones = (torch.rand(T, N, generator=g) < 0.3).to(torch.uint8)
    masks = torch.rand(T, N, K, generator=g) < 0.7
    masks[:, 0] = False                                         # an all-masked row
    out = {'actions': [], 'logits': [], 'clear': []}
    p.has_batch_dimension = False
    p.get_batch_size(obs[0], 1)
    assert p.has_batch_dimension and p.batch_size == N
    for t in range(T):
        with torch.no_grad():
            res = p.model({'is_train': False, 'prev_actions': None, 'obs': p._preproc_obs(obs[t]), 'rnn_states': p.states,
                           'action_masks': masks[t]})
        z = res['logits']
        top = z.topk(2, dim=-1).values
        out['logits'].append(z)
        out['clear'].append(((top[:, 0] - top[:, 1]) > GP.CLEAR_MARGIN).unsqueeze(-1))
        out['actions'].append(p.get_masked_action(obs[t], masks[t], True).detach().clone())
    assert p.model.running_mean_std.running_mean.shape == (FRAMES, FEATURES)
    fx = {'algo': 'a2c_discrete', 'params': {k: v for k, v in params.items()}, 'state': {'model': p.model.state_dict()}, 'obs': obs,
          'dones': dones, 'masks': masks, 'agents': 1, 'K': K, 'obs_shape': (FRAMES, FEATURES)}
    fx['params']['config'] = {k: v for k, v in config.items() if k not in ('env_info', 'vec_env')}
    fx.update({k: torch.stack(v) for k, v in out.items()})
    G.save(name, fx)


if __name__ == '__main__':
    gen_agent_conv1d('agent_conv1d_separate.pt', SAME, separate=True, agents=3, normalize_input=True, use_action_masks=True,
                     initializer={'name': 'default'})
    gen_agent_conv1d('agent_conv1d_shared.pt', STRIDED, separate=False, agents=1, normalize_input=False, use_action_masks=False,
                     initializer={'name': 'glorot_uniform_initializer', 'gain': 1.4241}, N=8, seed=62)
    gen_player_conv1d()
