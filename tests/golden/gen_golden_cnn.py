"""Generate the golden runs of the discrete agent with a conv2d trunk by running the REAL reference (see gen_golden.py) on a tape of
uint8 frames:

    python tests/golden/gen_golden_cnn.py

Writes tests/golden/agent_cnn_shared.pt and agent_cnn_separate.pt.  The frames are 4 x 36 x 36 (convs 8/4, 4/2, 3/1: the Nature-CNN
pattern at a size the CPU runs in seconds); the action draws replay through the same inverse-CDF tape as gen_golden.gen_agent_discrete.
The frames themselves are not stored: tests/_cnn_frames.py computes them from (T, N, frame shape, seed), which the fixtures record.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import gen_golden as G  # noqa: E402  (puts the reference and the import stubs on sys.path)

sys.path.insert(0, os.path.dirname(HERE))
from _cnn_frames import frame_tape  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402

CONVS = [{'filters': 8, 'kernel_size': 8, 'strides': 4, 'padding': 0}, {'filters': 8, 'kernel_size': 4, 'strides': 2, 'padding': 0},
         {'filters': 16, 'kernel_size': 3, 'strides': 1, 'padding': 0}]


class FrameTapeVecEnv(G.DiscreteTapeVecEnv):
    """DiscreteTapeVecEnv on uint8 frames [T, N, *frame]: the reward is 1 when the action is the argmax of the frame's first K bytes"""

    def step(self, actions):
        j0 = self.i % self.obs_tape.shape[0]
        target = self.obs_tape[j0].reshape(self.obs_tape.shape[1], -1)[:, :self.K].argmax(dim=-1)
        rew = (actions.long() == target).float()
        self.i += 1
        j = self.i % self.obs_tape.shape[0]
        return self.obs_tape[j].clone(), rew, self.done_tape[j].clone(), {'time_outs': self.timeout_tape[j].clone()}

    def get_env_info(self):
        import gymnasium as gym
        return {'observation_space': gym.spaces.Box(0, 255, tuple(self.obs_tape.shape[2:]), np.uint8),
                'action_space': gym.spaces.Discrete(self.K)}


def frame_tapes(T, N, shape, seed):
    """the computed uint8 frames (tests/_cnn_frames.py), and random done / time-out tapes"""
    g = torch.Generator().manual_seed(seed)
    frames = frame_tape(T, N, tuple(shape), seed)
    done = (torch.rand(T, N, generator=g) < 0.1).to(torch.uint8)
    tout = ((torch.rand(T, N, generator=g) < 0.3) & done.bool()).to(torch.uint8)
    return frames, done, tout


def gen_agent_cnn(name, frame_shape, nhwc, normalize_input, separate, use_action_masks, initializer, N=8, H=8, K=5, units=(32,), mb=32,
                  epochs=2, seed=21):
    from rl_games.torch_runner import Runner
    from oracle.ppo_discrete_oracle import sample_inverse_cdf
    torch.manual_seed(seed)
    np.random.seed(seed)
    T = H * epochs + 1
    obs_tape, done_tape, tout_tape = frame_tapes(T, N, frame_shape, seed)
    g = torch.Generator().manual_seed(seed + 100)
    mask_tape = None
    if use_action_masks:
        mask_tape = torch.rand(T, N, K, generator=g) < 0.6
        mask_tape.scatter_(2, torch.randint(0, K, (T, N, 1), generator=g), True)
    env = FrameTapeVecEnv(obs_tape, done_tape, tout_tape, K, mask_tape)
    network = {'name': 'actor_critic', 'separate': separate, 'space': {'discrete': None},
               'cnn': {'type': 'conv2d', 'permute_input': nhwc, 'activation': 'elu', 'initializer': dict(initializer), 'convs': CONVS},
               'mlp': {'units': list(units), 'activation': 'elu', 'initializer': dict(initializer), 'regularizer': {'name': 'None'}}}
    config = {'name': 'golden_cnn', 'env_name': 'unused', 'reward_shaper': {'scale_value': 0.1}, 'normalize_advantage': True,
              'gamma': 0.99, 'tau': 0.95, 'learning_rate': 3e-4, 'grad_norm': 1.0, 'entropy_coef': 0.01, 'truncate_grads': True,
              'e_clip': 0.2, 'clip_value': True, 'num_actors': N, 'horizon_length': H, 'minibatch_size': mb, 'mini_epochs': 2,
              'critic_coef': 1, 'lr_schedule': None, 'kl_threshold': 0.008, 'normalize_input': normalize_input, 'normalize_value': True,
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
    seeded_state = {k: v.clone() for k, v in agent.model.state_dict().items()}
    with torch.no_grad():
        for k, p in agent.model.named_parameters():
            if k.endswith('bias'):
                p.add_(torch.randn(p.shape, generator=g) * 0.05)
    init_state = {k: v.clone() for k, v in agent.model.state_dict().items()}
    u = torch.rand(epochs, H + 1, N, generator=g)
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
        assert agent.experience_buffer.tensor_dict['obses'].dtype == torch.uint8
    finally:
        torch.multinomial = orig_multinomial
    params_only = lambda sd: {k: v for k, v in sd.items() if k.startswith('a2c_network.')}   # noqa: E731  (fresh normalisers)
    for ep in epochs_out:            # the input normaliser's fp64 statistics as fp32: a fifth of the fixture otherwise, and fp32 holds
        ep['state'] = {k: v.float() if k.startswith('running_mean_std.') and v.dtype == torch.float64 else v   # what the tests compare
                       for k, v in ep['state'].items()}
    G.save(name, {'N': N, 'H': H, 'K': K, 'units': list(units), 'mb': mb, 'epochs': epochs, 'separate': separate, 'seed': seed,
                  'network': network, 'use_action_masks': use_action_masks,
                  'config': {k: v for k, v in params['config'].items() if isinstance(v, (int, float, str, bool, type(None)))},
                  'T': T, 'frame_shape': tuple(frame_shape), 'done_tape': done_tape, 'timeout_tape': tout_tape, 'mask_tape': mask_tape, 'u': u,
                  'seeded_state': params_only(seeded_state), 'init_state': params_only(init_state), 'epochs_out': epochs_out,
                  'param_order': [k for k, _ in agent.model.named_parameters()]})


if __name__ == '__main__':
    # shared trunk, NCHW frames (envpool's layout), no input normaliser, orthogonal init
    gen_agent_cnn('agent_cnn_shared.pt', (4, 36, 36), nhwc=False, normalize_input=False, separate=False, use_action_masks=False,
                  initializer={'name': 'orthogonal_initializer', 'gain': 1.41421356237})
    # separate trunks, NHWC frames (permute_input), the input normaliser on bytes, action masks, torch's default init
    gen_agent_cnn('agent_cnn_separate.pt', (36, 36, 4), nhwc=True, normalize_input=True, separate=True, use_action_masks=True,
                  initializer={'name': 'default'}, seed=22)
