"""SAC throughput on one GPU: this package's SACAgent against the reference's SACAgent (sac_agent.py, unmodified, from oracle/_ref) on the
same device, same shapes, same config.

    python tools/sac_ab.py [--rounds 5] [--updates 200] [--steps 20] [--json out.json]

Two shapes:
  sac_ant : 32 actors, obs 105, 8 actions, MLP [256, 256] relu, batch 256, utd_ratio 1.0 (32 updates per env step), policy_frequency 2
  wide    : 4096 actors, obs 105, 8 actions, MLP [256, 256] relu, batch 4096, 32 updates per env step, policy_frequency 2
Arms: 'reference' (fp32, the reference's eager update), 'b200 fp32' and 'b200 mixed' (b200_cuda_graph on).  Per arm and shape:
  updates/s    : `--updates` consecutive agent.update() calls on a full replay buffer, CUDA events around a synchronised loop;
  env-steps/s  : `--steps` env steps of play_steps() (sampling, an on-device random env, the replay write, the updates of the step).
Rounds alternate the arms; the median round is reported, with min / max.  The SM clock and power (nvidia-smi, read-only queries) are
sampled before and after each shape.  Per-call kernel times of one b200 update (CUDA events around every C-ABI call) are printed too:
they are the per-launch numbers behind the twin-critic and Polyak layout choices (DESIGN.md SAC)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests', 'golden', '_stubs'))       # gymnasium spaces (descriptors only)

SHAPES = {
    'sac_ant': dict(N=32, D=105, A=8, units=[256, 256], B=256, cfg={'utd_ratio': 1.0}),
    'wide': dict(N=4096, D=105, A=8, units=[256, 256], B=4096, cfg={'num_updates_per_step': 32}),
}


class RandomGPUEnv:
    """obs ~ N(0, 1) on the device, reward -|a|^2, done with p = 0.01; time_outs on half of the dones"""

    def __init__(self, N, D, A, dev):
        self.N, self.D, self.A, self.dev = N, D, A, dev

    def reset(self):
        return torch.randn(self.N, self.D, device=self.dev)

    def step(self, actions):
        d = torch.rand(self.N, device=self.dev) < 0.01
        return (torch.randn(self.N, self.D, device=self.dev), -(actions * actions).sum(-1), d.to(torch.uint8),
                {'time_outs': (d & (torch.rand(self.N, device=self.dev) < 0.5)).to(torch.uint8)})

    def get_env_info(self):
        import gymnasium as gym
        import numpy as np
        return {'observation_space': gym.spaces.Box(-np.inf, np.inf, (self.D,), np.float32),
                'action_space': gym.spaces.Box(-1.0, 1.0, (self.A,), np.float32)}

    def get_env_state(self):
        return None

    def set_env_state(self, s):
        pass

    def set_train_info(self, *a, **kw):
        pass


def _params(shape, env, mixed, graph):
    s = SHAPES[shape]
    config = {'name': 'sac_ab_' + shape, 'env_name': 'unused', 'reward_shaper': {'scale_value': 1.0}, 'device': 'cuda:0',
              'mixed_precision': mixed, 'gamma': 0.99, 'critic_tau': 0.005, 'batch_size': s['B'], 'replay_buffer_size': 200000,
              'num_warmup_steps': 0, 'num_steps_per_episode': 1, 'num_actors': s['N'], 'actor_lr': 3e-4, 'critic_lr': 3e-4, 'alpha_lr': 3e-4,
              'init_alpha': 1.0, 'learnable_temperature': True, 'policy_frequency': 2, 'print_stats': False, 'save_best_after': 10 ** 9,
              'train_dir': tempfile.mkdtemp(), 'env_info': env.get_env_info(), 'vec_env': env}
    config.update(s['cfg'])
    if graph is not None:
        config['b200_cuda_graph'] = graph
    network = {'name': 'soft_actor_critic', 'separate': True, 'space': {'continuous': {}}, 'log_std_bounds': [-20, 2],
               'mlp': {'units': s['units'], 'activation': 'relu', 'initializer': {'name': 'default'}}}
    return {'seed': 42, 'algo': {'name': 'sac'}, 'model': {'name': 'soft_actor_critic'}, 'network': network, 'config': config}


def build(arm, shape):
    s = SHAPES[shape]
    dev = torch.device('cuda:0')
    env = RandomGPUEnv(s['N'], s['D'], s['A'], dev)
    if arm == 'reference':
        from oracle import ref_arm
        ref_arm.import_reference()
        from rl_games.torch_runner import Runner
        r = Runner()
        r.load({'params': _params(shape, env, False, None)})
        r.params['config']['vec_env'] = env
        a = r.algo_factory.create('sac', base_name='ab', params=r.params)
        rb = a.replay_buffer
        n = rb.capacity
        rb.add(torch.randn(n, s['D'], device=dev), torch.rand(n, s['A'], device=dev) * 2 - 1, torch.randn(n, 1, device=dev),
               torch.randn(n, s['D'], device=dev), torch.zeros(n, 1, dtype=torch.bool, device=dev))
        a.init_tensors()
        a.obs = a.env_reset()
        a.epoch_num = 1
        return a, (lambda: a.update(a.epoch_num)), (lambda: a.play_steps(False))
    from rl_games_b200.runner import Runner
    r = Runner()
    r.load({'params': _params(shape, env, arm == 'b200 mixed', True)})
    r.params['config']['vec_env'] = env
    a = r.algo_factory.create('sac', base_name='ab', params=r.params)
    n = a.replay_buffer_size
    a.rb['obs'].normal_()
    a.rb['next'].normal_()
    a.rb['act'].uniform_(-1, 1)
    a.rb['rew'].normal_()
    a.rb['state'].copy_(torch.tensor([0, n]))
    a.init_tensors()
    a.obs = a.env_reset()
    a.epoch_num = 1
    return a, (lambda: a.update(a.stats[0])), (lambda: a.play_steps(False))


def timed(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3


def gpu_state():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,clocks.sm,clocks.max.sm,power.draw,power.limit', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        return out
    except Exception as e:      # noqa: BLE001
        return f'unavailable ({e})'


def kernel_breakdown(agent, update):
    from rl_games_b200._lib import lib
    graph = agent.use_graph
    agent.use_graph = False          # per-call events need the eager launches
    update()
    lib.start_profile()
    for _ in range(2):               # one critic-only and one critic + actor update
        update()
    prof = lib.stop_profile()
    agent.use_graph = graph
    return {k: {'n': v['n'], 'us_per_call': round(1e3 * v['ms'] / v['n'], 2)} for k, v in sorted(prof.items(), key=lambda kv: -kv[1]['ms'])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--updates', type=int, default=200)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--shapes', default='sac_ant,wide')
    ap.add_argument('--arms', default='reference,b200 fp32,b200 mixed')
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    result = {}
    for shape in args.shapes.split(','):
        arms = args.arms.split(',')
        built = {arm: build(arm, shape) for arm in arms}
        for arm in arms:                     # warm-up: graph captures, allocator, autotuning
            _, upd, step = built[arm]
            timed(upd, 8)
            timed(step, 2)
        before = gpu_state()
        ups, sps = {arm: [] for arm in arms}, {arm: [] for arm in arms}
        for _ in range(args.rounds):
            for arm in arms:
                a, upd, step = built[arm]
                ups[arm].append(args.updates / timed(upd, args.updates))
                sps[arm].append(SHAPES[shape]['N'] * args.steps / timed(step, args.steps))
        after = gpu_state()
        res = {'gpu_before': before, 'gpu_after': after, 'updates_per_step': built[arms[-1]][0].num_updates_per_step}
        for arm in arms:
            res[arm] = {'updates_per_s': {'median': statistics.median(ups[arm]), 'min': min(ups[arm]), 'max': max(ups[arm])},
                        'env_steps_per_s': {'median': statistics.median(sps[arm]), 'min': min(sps[arm]), 'max': max(sps[arm])}}
        for arm in arms:
            if arm != 'reference':
                a, upd, _ = built[arm]
                res[arm]['kernels_per_update_pair'] = kernel_breakdown(a, upd)
        result[shape] = res
        print(json.dumps({shape: res}, indent=1))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
