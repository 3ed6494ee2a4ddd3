"""Developer tool: what a state-dependent sigma head costs on the c2 workload (16384 envs x horizon 16, obs 60, 8 actions, MLP
[256,128,64], minibatch 32768 x 4 mini-epochs), measured as whole `train_epoch` times (CUDA events, L2 flushed between epochs), the
arms alternating round by round in one process so that they share the card's state:

  fixed_fused    fixed exp log-std, mixed_precision: True -> the fused wgmma kernels (what bench.py measures)
  fixed_layer    fixed softplus sigma (min_sigma 0.2)     -> layer-wise wgmma GEMMs + fp32 head kernels
  sd_layer       state-dependent softplus head (wujihand) -> layer-wise wgmma GEMMs + the state-dependent fp32 head kernels
  sd_fp32        state-dependent softplus head, mixed_precision: False -> fp32 CUDA-core GEMMs

fixed_layer vs sd_layer isolates the head; fixed_fused vs sd_layer is what a user switching heads sees today.  Prints the card's name
and power limit next to the numbers, then one instrumented eager epoch per arm (per-call CUDA-event times).
Usage: python tools/sdsigma_ab.py [--rounds 5] [--steps 5] [--arms fixed_fused,fixed_layer,sd_layer,sd_fp32]"""
import argparse
import copy
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

SOFTPLUS_SD = {'fixed_sigma': False, 'sigma_parametrization': 'softplus', 'min_sigma': 0.2,
               'sigma_init': {'name': 'const_initializer', 'val': -1.05}}
ARMS = {'fixed_fused': ({}, True), 'fixed_layer': ({'sigma_parametrization': 'softplus', 'min_sigma': 0.2}, True),
        'sd_layer': (SOFTPLUS_SD, True), 'sd_fp32': (SOFTPLUS_SD, False)}


def build(space_over, mixed_precision, device):
    from rl_games_b200.runner import Runner
    w = bench.WORKLOADS['c2']
    params = bench.make_params(w, device, 'b200_synthetic', False, graph=True, mixed_precision=mixed_precision)
    params = copy.deepcopy(params)
    params['network']['space']['continuous'].update(space_over)
    r = Runner()
    r.load({'params': params})
    agent = r.algo_factory.create(r.algo_name, base_name='sdsigma_ab', params=r.params)
    agent.init_tensors()
    agent.obs = agent.env_reset()
    return agent


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:      # noqa: BLE001
        return f'unknown ({e})'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=5, help='epochs per arm per round')
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--arms', default=','.join(ARMS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    device = 'cuda:0'
    torch.cuda.set_device(0)
    names = args.arms.split(',')
    agents = {n: build(*ARMS[n], device) for n in names}
    for n, a in agents.items():
        print(f'{n:12s} use_tc={a.use_tc} gemm_tc={a.gemm_tc} fixed_sigma={a.model.fixed_sigma}')
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=device)
    for a in agents.values():
        bench.timed_epochs(a, args.warmup, flush, 1)
    times = {n: [] for n in names}
    for rd in range(args.rounds):
        order = names if rd % 2 == 0 else names[::-1]
        for n in order:
            ms = bench.timed_epochs(agents[n], args.steps, flush, 1)
            times[n].append(statistics.median(ms))
    print(f'card: {card()}')
    print(f'train_epoch, c2, median of {args.steps} epochs per round, {args.rounds} alternating rounds (ms):')
    base = statistics.mean(times[names[0]])
    for n in names:
        t = times[n]
        print(f'  {n:12s} mean {statistics.mean(t):8.3f}  min {min(t):8.3f}  max {max(t):8.3f}  '
              f'({statistics.mean(t) / base:5.2f}x {names[0]})  rounds: {" ".join(f"{x:.3f}" for x in t)}')
    print('per-call CUDA-event times of one instrumented eager epoch (ms per epoch):')
    for n in names:
        prof = bench.kernel_breakdown(agents[n])
        top = sorted(prof.items(), key=lambda kv: -kv[1]['ms'])[:8]
        print(f'  {n:12s} ' + ', '.join(f'{k} {v["ms"]:.3f} ({v["n"]})' for k, v in top))


if __name__ == '__main__':
    main()
