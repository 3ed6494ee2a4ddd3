"""Measure the discrete agent's conv trunk on a Pong-shaped workload (configs/atari/ppo_pong.yaml's network and batch): 64 actors x 128
steps of 4x84x84 uint8 frames from a synthetic device env, 6 actions, Nature-CNN trunk (32@8/4, 64@4/2, 64@3/1, elu), MLP [512],
minibatch 2048 x 4 mini-epochs, input normaliser on.

Prints one JSON line:
- epoch_ms: one train_epoch (rollout + GAE + 16 minibatch updates), CUDA events, after a warm-up epoch (median of --epochs);
- mb_update_ms: one minibatch update of the agent (forward, loss, backward, Adam);
- ref_fp32_ms / ref_bf16_ms: the reference's ModelA2C network (oracle/_ref) on the same 2048 frames: forward, the same kind of loss,
  backward and torch Adam, in fp32 and under bf16 autocast (cuDNN);
- conv_share: the conv kernels' share of the GPU kernel time of one epoch, from a separate torch.profiler run;
- the card's name and power limit.
Usage: python tools/cnn_ab.py [--epochs 3]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

DEV = 'cuda:0'
N, H, K, MB, FRAME = 64, 128, 6, 2048, (4, 84, 84)
NETWORK = {'name': 'actor_critic', 'separate': False, 'space': {'discrete': None},
           'cnn': {'type': 'conv2d', 'permute_input': False, 'activation': 'elu', 'initializer': {'name': 'default'},
                   'convs': [{'filters': 32, 'kernel_size': 8, 'strides': 4, 'padding': 0},
                             {'filters': 64, 'kernel_size': 4, 'strides': 2, 'padding': 0},
                             {'filters': 64, 'kernel_size': 3, 'strides': 1, 'padding': 0}]},
           'mlp': {'units': [512], 'activation': 'elu', 'initializer': {'name': 'orthogonal_initializer', 'gain': 1.41421356237}}}


class FrameEnv:
    """random uint8 frames generated on the device; episodes end at random"""

    def __init__(self):
        self.g = torch.Generator(device=DEV).manual_seed(0)

    def _frames(self):
        return torch.randint(0, 256, (N,) + FRAME, generator=self.g, device=DEV, dtype=torch.uint8)

    def reset(self):
        return self._frames()

    def step(self, actions):
        r = torch.rand(N, generator=self.g, device=DEV)
        return self._frames(), r, (r < 0.01).to(torch.uint8), {}

    def get_env_info(self):
        from rl_games_b200.common import Box, Discrete
        return {'observation_space': Box(0, 255, FRAME, 'uint8'), 'action_space': Discrete(K)}


def make_agent():
    from rl_games_b200.runner import Runner
    env = FrameEnv()
    config = {'name': 'cnn_ab', 'env_name': 'unused', 'reward_shaper': {'min_val': -1, 'max_val': 1}, 'normalize_value': True,
              'normalize_input': True, 'normalize_advantage': True, 'gamma': 0.99, 'tau': 0.95, 'learning_rate': 3e-4, 'grad_norm': 1.0,
              'entropy_coef': 0.01, 'truncate_grads': True, 'e_clip': 0.2, 'clip_value': True, 'num_actors': N, 'horizon_length': H,
              'minibatch_size': MB, 'mini_epochs': 4, 'critic_coef': 1, 'lr_schedule': None, 'kl_threshold': 0.008, 'device': DEV,
              'mixed_precision': False, 'max_epochs': 1000, 'save_frequency': 0, 'print_stats': False,
              'train_dir': tempfile.mkdtemp(prefix='cnn_ab_'), 'env_info': env.get_env_info(), 'vec_env': env}
    r = Runner()
    r.load({'params': {'seed': 1, 'algo': {'name': 'a2c_discrete'}, 'model': {'name': 'discrete_a2c'}, 'network': NETWORK, 'config': config}})
    r.params['config']['vec_env'] = env
    agent = r.algo_factory.create(r.algo_name, base_name='cnn_ab', params=r.params)
    agent.init_tensors()
    agent.obs = agent.env_reset()
    return agent


def timed(fn, reps):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    t = sorted(a.elapsed_time(b) for a, b in ev)
    return t[len(t) // 2]


def reference_ms(frames, bf16, reps):
    for p in (os.path.join(ROOT, 'tests', 'golden', '_stubs'), os.path.join(ROOT, 'oracle', '_ref')):
        if p not in sys.path:
            sys.path.insert(0, p)
    from rl_games.algos_torch import model_builder
    model = model_builder.ModelBuilder().load({'model': {'name': 'discrete_a2c'}, 'network': NETWORK}).build(
        {'actions_num': K, 'input_shape': FRAME, 'num_seqs': N, 'value_size': 1, 'normalize_value': True, 'normalize_input': True})
    model = model.to(DEV).train()
    opt = torch.optim.Adam(model.parameters(), lr=3e-4)
    actions = torch.randint(0, K, (MB,), device=DEV)

    def step():
        with torch.autocast('cuda', dtype=torch.bfloat16, enabled=bf16):
            out = model({'is_train': True, 'obs': frames.float() / 255.0, 'prev_actions': actions})
            loss = out['prev_neglogp'].mean() + out['values'].float().pow(2).mean() - 0.01 * out['entropy'].mean()
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
    for _ in range(3):
        step()
    return timed(step, reps)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--epochs', type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'cnn_ab measures on a GPU'
    torch.cuda.set_device(0)
    agent = make_agent()
    agent.train_epoch()                                    # warm-up: every shape of the timed window
    epoch_ms = timed(agent.train_epoch, args.epochs)
    mb_ms = timed(lambda: agent._minibatch_update(0), 10)
    frames = agent.obses.view(H * N, -1)[:MB].view(MB, *FRAME)
    ref32, ref16 = reference_ms(frames, False, 10), reference_ms(frames, True, 10)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        agent.train_epoch()
        torch.cuda.synchronize()
    tot = conv = 0.0
    for e in prof.key_averages():
        t = getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0.0)
        if e.key.startswith(('cuda', 'Memcpy', 'Memset')) or t <= 0:
            continue
        tot += t
        conv += t if 'conv2d_' in e.key else 0.0
    print(json.dumps({'workload': 'pong-shaped: 64x128 uint8 4x84x84, nature-cnn + [512], mb 2048 x 4', 'epoch_ms': round(epoch_ms, 2),
                      'mb_update_ms': round(mb_ms, 3), 'ref_fp32_mb_ms': round(ref32, 3), 'ref_bf16_autocast_mb_ms': round(ref16, 3),
                      'conv_share_of_kernel_time': round(conv / max(tot, 1e-9), 3), 'card': card()}))


if __name__ == '__main__':
    main()
