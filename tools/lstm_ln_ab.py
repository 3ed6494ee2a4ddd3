"""Developer tool: what `rnn.layer_norm: True` costs on the c4 workload (8192 envs x horizon 32, obs 348, 17 actions, LSTM 256 before the
MLP [512, 256, 128], seq_length 4, minibatch 32768 x 4 mini-epochs, layer-wise wgmma GEMMs, CUDA graphs), measured as whole `train_epoch`
times (CUDA events, L2 flushed between epochs).  The two arms -- layer_norm off (what bench.py --workload c4 measures) and on (the
LSTM-cell + LayerNorm kernels in the rollout step and the BPTT window) -- alternate round by round in one process so that they share the
card's state.  Prints the card's name and power limit next to the numbers, then the LayerNorm kernels' share of one instrumented eager
epoch of the `on` arm (per-call CUDA-event times).
Usage: python tools/lstm_ln_ab.py [--rounds 5] [--steps 3]"""
import argparse
import copy
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import bench  # noqa: E402
from sdsigma_ab import card  # noqa: E402


def build(layer_norm, device):
    from rl_games_b200.runner import Runner
    params = copy.deepcopy(bench.make_params(bench.WORKLOADS['c4'], device, 'b200_synthetic', False, graph=True, mixed_precision=True))
    params['network']['rnn']['layer_norm'] = layer_norm
    r = Runner()
    r.load({'params': params})
    agent = r.algo_factory.create(r.algo_name, base_name='lstm_ln_ab', params=r.params)
    agent.init_tensors()
    agent.obs = agent.env_reset()
    return agent


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=3, help='epochs per arm per round')
    ap.add_argument('--warmup', type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    device = 'cuda:0'
    torch.cuda.set_device(0)
    agents = {'off': build(False, device), 'on': build(True, device)}
    for n, a in agents.items():
        print(f'{n:4s} gemm_tc={a.gemm_tc} layer_norm={a.model.rnn_layer_norm}')
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=device)
    for a in agents.values():
        bench.timed_epochs(a, args.warmup, flush, 1)
    names = list(agents)
    times = {n: [] for n in names}
    for rd in range(args.rounds):
        for n in (names if rd % 2 == 0 else names[::-1]):
            times[n].append(statistics.median(bench.timed_epochs(agents[n], args.steps, flush, 1)))
    print(f'card: {card()}')
    print(f'train_epoch, c4, median of {args.steps} epochs per round, {args.rounds} alternating rounds (ms):')
    for n in names:
        t = times[n]
        print(f'  {n:4s} mean {statistics.mean(t):8.3f}  min {min(t):8.3f}  max {max(t):8.3f}  rounds: {" ".join(f"{x:.3f}" for x in t)}')
    d = [b - a for a, b in zip(times['off'], times['on'])]
    print(f'  on - off per round (ms): {" ".join(f"{x:+.3f}" for x in d)}  mean {statistics.mean(d):+.3f} '
          f'({100 * statistics.mean(d) / statistics.mean(times["off"]):+.1f} %)')
    prof = bench.kernel_breakdown(agents['on'])
    for k in ('lstm_cell_ln_fwd_f32', 'lstm_cell_ln_bwd_f32'):
        ev = prof.get(k, {'ms': float('nan'), 'n': 0})
        print(f'{k} in one instrumented eager epoch: {ev["ms"]:.3f} ms ({ev["n"]} launches)')


if __name__ == '__main__':
    main()
