"""Measure the discrete agent's conv1d trunk on smac-shaped minibatch updates: separate actor / critic trunks, action masks, relu, MLP
[256, 128], 4 stacked frames of fp32 unit features from a synthetic device env.
- corridor: 156 features, convs 64@k3s2p1, 128@k3, 256@k3 (corridor_torch.yaml), minibatch 3072;
- 27m: 285 features, convs 256, 512, 1024 @k3s1p1 (27m_vs_30m_torch.yaml), minibatch 3456, 14 actions.
Per shape, the fp32 agent (conv.cu + mlp_simt.cu) and the tensor-core agent (mixed_precision: True, conv_tc.cu + gemm_tc.cu), alternated
round by round when both fit the device at once (else one after the other, reported as such): one minibatch update (forward, loss,
backward, reductions, Adam), CUDA events, median [min, max] over the rounds; the peak device memory of each arm
(torch.cuda.max_memory_allocated); the reference's network (oracle/_ref) on the same
observations: forward, a PPO-like loss, backward and torch Adam, fp32 and under bf16 autocast (cuDNN); the card's name and power limit.
Peak memory is each arm's own: the peak over building the agent (init_tensors), one epoch and its updates, less what was allocated
before it (the other arm's buffers when both are resident); beside it, what the agent counts before allocating (init_tensors_bytes
plus the model's 12 bytes per parameter), the number its out-of-memory refusal compares with the device's free memory.
Prints one JSON line.  Usage: python tools/conv1d_ab.py [--rounds 5] [--shapes corridor,27m]"""
import argparse
import gc
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

DEV = 'cuda:0'
SHAPES = {
    'corridor': dict(L=156, K=6, agents=6, mb=3072, convs=[(64, 2, 1), (128, 1, 0), (256, 1, 0)]),
    '27m': dict(L=285, K=14, agents=27, mb=3456, convs=[(256, 1, 1), (512, 1, 1), (1024, 1, 1)]),
}
ENVS, FRAMES = 8, 4


def network(sh):
    return {'name': 'actor_critic', 'separate': True, 'space': {'discrete': None},
            'cnn': {'type': 'conv1d', 'activation': 'relu', 'initializer': {'name': 'default'},
                    'convs': [{'filters': f, 'kernel_size': 3, 'strides': s, 'padding': p} for f, s, p in sh['convs']]},
            'mlp': {'units': [256, 128], 'activation': 'relu', 'initializer': {'name': 'default'}}}


class StackEnv:
    """random frame stacks and masks on the device; episodes end at random"""

    def __init__(self, rows, L, K, agents):
        self.rows, self.L, self.K, self.agents = rows, L, K, agents
        self.g = torch.Generator(device=DEV).manual_seed(0)

    def reset(self):
        return torch.rand(self.rows, FRAMES, self.L, generator=self.g, device=DEV)

    def step(self, actions):
        r = torch.rand(self.rows, generator=self.g, device=DEV)
        return self.reset(), r, (r < 0.01).to(torch.uint8), {}

    def get_action_masks(self):
        return torch.ones(self.rows, self.K, dtype=torch.uint8, device=DEV)

    def get_env_info(self):
        from rl_games_b200.common import Box, Discrete
        return {'observation_space': Box(0, 1, (FRAMES, self.L)), 'action_space': Discrete(self.K), 'agents': self.agents}


def make_agent(sh, mixed_precision):
    from rl_games_b200.runner import Runner
    rows = ENVS * sh['agents']
    env = StackEnv(rows, sh['L'], sh['K'], sh['agents'])
    config = {'name': 'conv1d_ab', 'env_name': 'unused', 'reward_shaper': {'scale_value': 1}, 'normalize_value': False,
              'normalize_input': True, 'normalize_advantage': True, 'gamma': 0.99, 'tau': 0.95, 'learning_rate': 1e-4, 'grad_norm': 0.5,
              'entropy_coef': 0.005, 'truncate_grads': True, 'e_clip': 0.2, 'clip_value': True, 'num_actors': ENVS,
              'horizon_length': sh['mb'] // rows, 'minibatch_size': sh['mb'], 'mini_epochs': 1, 'critic_coef': 2, 'lr_schedule': None,
              'kl_threshold': 0.05, 'device': DEV, 'mixed_precision': mixed_precision, 'use_action_masks': True, 'max_epochs': 1000,
              'save_frequency': 0, 'print_stats': False, 'train_dir': tempfile.mkdtemp(prefix='conv1d_ab_'),
              'env_info': env.get_env_info(), 'vec_env': env}
    r = Runner()
    r.load({'params': {'seed': 1, 'algo': {'name': 'a2c_discrete'}, 'model': {'name': 'discrete_a2c'}, 'network': network(sh),
                       'config': config}})
    r.params['config']['vec_env'] = env
    agent = r.algo_factory.create(r.algo_name, base_name='conv1d_ab', params=r.params)
    agent.init_tensors()
    agent.obs = agent.env_reset()
    agent.train_epoch()                 # fills the arena and the prepared batch; warms every shape of the timed window
    agent._minibatch_update(0)
    torch.cuda.synchronize()
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


def spread(ts):
    ts = sorted(ts)
    return round(ts[len(ts) // 2], 3), [round(ts[0], 3), round(ts[-1], 3)]


def reference_ms(sh, obs, bf16, rounds):
    for p in (os.path.join(ROOT, 'tests', 'golden', '_stubs'), os.path.join(ROOT, 'oracle', '_ref')):
        if p not in sys.path:
            sys.path.insert(0, p)
    from rl_games.algos_torch import model_builder
    model = model_builder.ModelBuilder().load({'model': {'name': 'discrete_a2c'}, 'network': network(sh)}).build(
        {'actions_num': sh['K'], 'input_shape': (FRAMES, sh['L']), 'num_seqs': 1, 'value_size': 1, 'normalize_value': False,
         'normalize_input': True})
    model = model.to(DEV).train()
    opt = torch.optim.Adam(model.parameters(), lr=1e-4)
    actions = torch.randint(0, sh['K'], (sh['mb'],), device=DEV)

    def step():
        with torch.autocast('cuda', dtype=torch.bfloat16, enabled=bf16):
            out = model({'is_train': True, 'obs': obs, 'prev_actions': actions})
            loss = out['prev_neglogp'].mean() + out['values'].float().pow(2).mean() - 0.005 * out['entropy'].mean()
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    for _ in range(2):
        step()
    ts = [timed(step, 3) for _ in range(rounds)]
    peak = torch.cuda.max_memory_allocated() - base
    del model, opt
    return ts, peak


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                       text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else torch.cuda.get_device_name(0)


def free():
    gc.collect()
    torch.cuda.empty_cache()


def measure(name, sh, rounds):
    out = {'features': sh['L'], 'minibatch': sh['mb'], 'convs': sh['convs'], 'actions': sh['K']}
    arms, peak, counted, ts = {}, {}, {}, {'fp32': [], 'tc': []}
    try:
        for k, mp in (('fp32', False), ('tc', True)):
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            arms[k] = make_agent(sh, mp)
            peak[k] = torch.cuda.max_memory_allocated() - base
            counted[k] = arms[k].init_tensors_bytes() + 12 * arms[k].model.num_params
        out['alternated'] = True
        for _ in range(rounds):                        # the arms alternate: both see the same state of the shared machine
            for k, a in arms.items():
                ts[k].append(timed(lambda: a._minibatch_update(0), 3))
    except torch.OutOfMemoryError:                     # both do not fit at once: one after the other
        arms.clear()
        free()
        out['alternated'] = False
        for k, mp in (('fp32', False), ('tc', True)):
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            a = make_agent(sh, mp)
            peak[k] = torch.cuda.max_memory_allocated() - base
            counted[k] = a.init_tensors_bytes() + 12 * a.model.num_params
            ts[k] = [timed(lambda: a._minibatch_update(0), 3) for _ in range(rounds)]
            arms[k] = a
            if k == 'fp32':
                obs = a.obses.view(-1, FRAMES, sh['L'])[:sh['mb']].clone()
                arms.clear()
                del a
                free()
    for k in ('fp32', 'tc'):
        m, s = spread(ts[k])
        out[k] = {'mb_update_ms': m, 'mb_update_ms_spread': s, 'peak_mem_bytes': peak[k], 'counted_bytes': counted[k]}
    if 'fp32' in arms:
        obs = arms['fp32'].obses.view(-1, FRAMES, sh['L'])[:sh['mb']].clone()
        out['num_params'] = arms['fp32'].model.num_params
    else:
        out['num_params'] = arms['tc'].model.num_params
    arms.clear()
    free()
    for k, bf16 in (('ref_fp32', False), ('ref_bf16_autocast', True)):
        t, p = reference_ms(sh, obs, bf16, rounds)
        m, s = spread(t)
        out[k] = {'mb_update_ms': m, 'mb_update_ms_spread': s, 'peak_mem_bytes': p}
        free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--shapes', default='corridor,27m')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'conv1d_ab measures on a GPU'
    torch.cuda.set_device(0)
    res = {'rounds': args.rounds, 'card': card()}
    for name in args.shapes.split(','):
        res[name] = measure(name, SHAPES[name], args.rounds)
        print(json.dumps({name: res[name]}), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
