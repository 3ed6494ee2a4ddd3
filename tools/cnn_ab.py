"""Measure the discrete agent's conv trunk on a Pong-shaped workload (configs/atari/ppo_pong.yaml's network and batch): 64 actors x 128
steps of 4x84x84 uint8 frames from a synthetic device env, 6 actions, Nature-CNN trunk (32@8/4, 64@4/2, 64@3/1, elu), MLP [512],
minibatch 2048 x 4 mini-epochs, input normaliser on.

Two arms in one process, alternated round by round: the fp32 agent (mixed_precision: False, conv.cu + mlp_simt.cu) and the
tensor-core agent (mixed_precision: True, conv_tc.cu + gemm_tc.cu).  Prints one JSON line:
- epoch_ms / mb_update_ms per arm: one train_epoch (rollout + GAE + 16 minibatch updates) and one minibatch update (forward, loss,
  backward, Adam), CUDA events, after a warm-up epoch: the median over --rounds rounds and the [min, max] spread;
- ref_fp32_ms / ref_bf16_ms: the reference's ModelA2C network (oracle/_ref) on the same 2048 frames: forward, the same kind of loss,
  backward and torch Adam, in fp32 and under bf16 autocast (cuDNN);
- conv_share per arm: the conv kernels' share of the GPU kernel time of one epoch, from a separate torch.profiler run;
- max_abs_diff: the largest difference in logits and in value between the arms on the same frames with the same weights;
- the card's name and power limit, read in the same call.
Usage: python tools/cnn_ab.py [--rounds 5]"""
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


def make_agent(mixed_precision):
    from rl_games_b200.runner import Runner
    env = FrameEnv()
    config = {'name': 'cnn_ab', 'env_name': 'unused', 'reward_shaper': {'min_val': -1, 'max_val': 1}, 'normalize_value': True,
              'normalize_input': True, 'normalize_advantage': True, 'gamma': 0.99, 'tau': 0.95, 'learning_rate': 3e-4, 'grad_norm': 1.0,
              'entropy_coef': 0.01, 'truncate_grads': True, 'e_clip': 0.2, 'clip_value': True, 'num_actors': N, 'horizon_length': H,
              'minibatch_size': MB, 'mini_epochs': 4, 'critic_coef': 1, 'lr_schedule': None, 'kl_threshold': 0.008, 'device': DEV,
              'mixed_precision': mixed_precision, 'max_epochs': 1000, 'save_frequency': 0, 'print_stats': False,
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


def conv_share(agent):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        agent.train_epoch()
        torch.cuda.synchronize()
    tot = conv = 0.0
    per = []
    for e in prof.key_averages():
        t = getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0.0)
        if e.key.startswith(('cuda', 'Memcpy', 'Memset')) or t <= 0:
            continue
        tot += t
        conv += t if ('conv2d_' in e.key or 'conv_tc_' in e.key) else 0.0
        per.append((t, e.key))
    top = [[k[:90], round(t / 1e3, 2)] for t, k in sorted(per, reverse=True)[:6]]       # ms per epoch
    return round(conv / max(tot, 1e-9), 3), top


def spread(ts):
    ts = sorted(ts)
    return round(ts[len(ts) // 2], 3), [round(ts[0], 3), round(ts[-1], 3)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'cnn_ab measures on a GPU'
    torch.cuda.set_device(0)
    arms = {'fp32': make_agent(False), 'tc': make_agent(True)}
    for a in arms.values():
        a.train_epoch()                                    # warm-up: every shape of the timed window
        a._minibatch_update(0)
    ep = {k: [] for k in arms}
    mb = {k: [] for k in arms}
    for _ in range(args.rounds):                           # the arms alternate: both see the same state of the shared machine
        for k, a in arms.items():
            ep[k].append(timed(a.train_epoch, 1))
            mb[k].append(timed(lambda: a._minibatch_update(0), 5))
    a32, atc = arms['fp32'], arms['tc']
    frames = a32.obses.view(H * N, -1)[:MB].view(MB, *FRAME)
    ref32, ref16 = reference_ms(frames, False, 10), reference_ms(frames, True, 10)
    share = {k: conv_share(a) for k, a in arms.items()}
    # the same weights and frames through both arms' rollout forward
    atc.set_weights(a32.get_weights())
    for a in arms.values():
        a._forward(a32.obs, a.r_a, a.r_c, N, conv=(a.r_ka, a.r_kc))
    torch.cuda.synchronize()
    d_logits = (a32.r_out[0] - atc.r_out[0]).abs().max().item()
    d_value = (a32.r_out[2][:, :1] - atc.r_out[2][:, :1]).abs().max().item()
    out = {'workload': 'pong-shaped: 64x128 uint8 4x84x84, nature-cnn + [512], mb 2048 x 4', 'rounds': args.rounds}
    for k in arms:
        (e, es), (m, ms) = spread(ep[k]), spread(mb[k])
        out[k] = {'epoch_ms': e, 'epoch_ms_spread': es, 'mb_update_ms': m, 'mb_update_ms_spread': ms,
                  'conv_share_of_kernel_time': share[k][0], 'top_kernels_ms_per_epoch': share[k][1]}
    out.update({'ref_fp32_mb_ms': round(ref32, 3), 'ref_bf16_autocast_mb_ms': round(ref16, 3),
                'max_abs_diff': {'logits': d_logits, 'value': d_value,
                                 'logits_scale': a32.r_out[0].abs().max().item(), 'value_scale': a32.r_out[2][:, :1].abs().max().item()},
                'card': card()})
    print(json.dumps(out))


if __name__ == '__main__':
    main()
