"""Developer tool: what a multi-agent env costs on the c2 workload (16384 rows x horizon 16, obs 60, 8 actions, MLP [256, 128, 64],
minibatch 32768 x 4 mini-epochs, fused wgmma kernels, whole-epoch CUDA graphs), measured as whole `train_epoch` times (CUDA events, L2
flushed between epochs).  The two arms train the same rows: 16384 envs x 1 agent (the single-agent post-step) and 4096 envs x 4 agents
(the multi-agent post-step with its ordered done-row selection).  They alternate round by round in one process so that they share the
card's state.  Prints the card's name and power limit next to the numbers, then the post-step kernels' per-call time from one
instrumented eager epoch of each arm (per-call CUDA-event times, launch overhead included).
Usage: python tools/ma_ab.py [--rounds 6] [--steps 5]"""
import argparse
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import bench  # noqa: E402
from sdsigma_ab import card  # noqa: E402


def build(envs, agents, device):
    from rl_games_b200.runner import Runner
    w = dict(bench.WORKLOADS['c2'], num_actors=envs)
    params = bench.make_params(w, device, 'b200_synthetic', False, graph=True, mixed_precision=True)
    params['config']['env_config']['agents'] = agents
    r = Runner()
    r.load({'params': params})
    agent = r.algo_factory.create(r.algo_name, base_name='ma_ab', params=r.params)
    agent.init_tensors()
    agent.obs = agent.env_reset()
    return agent


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=6)
    ap.add_argument('--steps', type=int, default=5, help='epochs per arm per round')
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    device = 'cuda:0'
    torch.cuda.set_device(0)
    n = bench.WORKLOADS['c2']['num_actors']
    agents = {'G=1': build(n, 1, device), 'G=4': build(n // 4, 4, device)}
    for k, a in agents.items():
        print(f'{k}: envs {a.num_actors} x agents {a.num_agents} = {a.num_rows} rows, fused={a.use_tc}, '
              f'whole-epoch graph={a._whole_epoch_graph_ok()}')
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=device)
    for a in agents.values():
        bench.timed_epochs(a, args.warmup, flush, 1)
    names = list(agents)
    times = {k: [] for k in names}
    for rd in range(args.rounds):
        for k in (names if rd % 2 == 0 else names[::-1]):
            times[k].append(statistics.median(bench.timed_epochs(agents[k], args.steps, flush, 1)))
    print(f'card: {card()}')
    print(f'train_epoch, c2, median of {args.steps} epochs per round, {args.rounds} alternating rounds (ms):')
    for k in names:
        t = times[k]
        print(f'  {k} mean {statistics.mean(t):8.3f}  min {min(t):8.3f}  max {max(t):8.3f}  rounds: {" ".join(f"{x:.3f}" for x in t)}')
    d = [b - a for a, b in zip(times['G=1'], times['G=4'])]
    print(f'  G=4 - G=1 per round (ms): {" ".join(f"{x:+.3f}" for x in d)}  mean {statistics.mean(d):+.3f}')
    for k, key in (('G=1', 'post_step_f32'), ('G=4', 'post_step_ma_f32')):
        prof = bench.kernel_breakdown(agents[k])
        ev = prof.get(key, {'ms': float('nan'), 'n': 0})
        print(f'{k}: {key} in one instrumented eager epoch: {ev["ms"]:.3f} ms over {ev["n"]} launches = '
              f'{1e3 * ev["ms"] / max(ev["n"], 1):.2f} us per step')


if __name__ == '__main__':
    main()
