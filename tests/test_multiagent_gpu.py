"""Multi-agent envs (env_info['agents'] = G > 1) on the GPU: the multi-agent post-step kernel against torch's dones.nonzero()[::G] from one
row to about 10^6 rows (none, some and all rows done; several steps in a row, so every launch re-arms its tile status), run twice for
determinism; the continuous agent against the reference's multi-agent golden runs, eager and with CUDA graphs; the layer-wise tensor-core
agent against the fp32 agent; the fused wgmma agent with G = 4 against the same rows trained as G = 1, and the whole-epoch CUDA graph
against eager epochs."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from oracle import ppo_oracle as O  # noqa: E402
from test_agent_gpu import DEV, TapeEnvGPU, _check_epoch, make_agent  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _shaper():
    from rl_games_b200 import ops
    return ops.ShaperCfg(1.0, 0.0, -float('inf'), float('inf'), 0.99, 0, 1)


def _ref_step(rew, done, tout, val, ep, meter, G, gtt):
    """a2c_common.py:1019-1051 in torch (fp64 meter means): returns shaped rewards, the selected indices; updates ep and meter"""
    sh = rew + 0.99 * val * tout.float()
    cr, cs, cl = ep[0] + rew, ep[1] + sh, ep[2] + 1.0
    sel = done.nonzero().reshape(-1)[::G]
    n = sel.numel()
    if n:
        size = min(n, gtt)
        old = min(gtt - size, meter[3])
        tot = old + size
        for s, x in ((0, cr), (1, cs), (2, cl)):
            meter[s] = (meter[s] * old + float(x[sel].double().mean()) * size) / tot
        meter[3] = tot
        meter[4] += n
    nd = 1.0 - done.float()
    ep.copy_(torch.stack([cr * nd, cs * nd, cl * nd]))
    return sh, sel


def _run_kernel(N, G, pattern, steps=3, seed=0):
    from rl_games_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(seed)
    ep = torch.zeros(3, N, device=DEV)
    meter = torch.zeros(8, dtype=torch.float64, device=DEV)
    bufs = ops.post_step_ma_buffers(N, G, DEV)
    dcur = torch.empty(N, dtype=torch.uint8, device=DEV)
    out = []
    for s in range(steps):
        rew = torch.randn(N, generator=g, device=DEV)
        val = torch.randn(N, generator=g, device=DEV)
        u = torch.rand(N, generator=g, device=DEV)
        done = {'none': u < -1, 'all': u >= 0, 'sparse': u < 0.01, 'dense': u < 0.4}[pattern].to(torch.uint8)
        tout = (torch.rand(N, generator=g, device=DEV) < 0.3).to(torch.uint8) & done
        rout = torch.empty(N, device=DEV)
        ops.post_step_ma(rew, done, tout, val, None, rout, dcur, None, ep, meter, 100, bufs, N, G, _shaper())
        n = int(bufs[4].item())
        out.append((rew, val, done, tout, rout.clone(), dcur.clone(), bufs[3][:n].clone(), ep.clone(), meter.clone()))
    return out


@pytest.mark.parametrize('N', [1, 7, 1023, 1024, 1025, 4099, 65537, 1_000_003])
@pytest.mark.parametrize('G', [2, 3, 4])
@pytest.mark.parametrize('pattern', ['none', 'sparse', 'dense', 'all'])
def test_post_step_ma_selects_every_gth_done_row_like_torch(N, G, pattern):
    runs = [_run_kernel(N, G, pattern), _run_kernel(N, G, pattern)]
    torch.cuda.synchronize()
    ep = torch.zeros(3, N, device=DEV, dtype=torch.float32)
    meter = [0.0] * 5
    for s, step in enumerate(runs[0]):
        rew, val, done, tout, rout, dcur, sel, ep_k, meter_k = step
        sh, sel_ref = _ref_step(rew, done, tout, val, ep, meter, G, 100)
        assert torch.equal(sel, sel_ref), (s, sel[:8], sel_ref[:8])
        assert torch.equal(dcur, done)
        torch.testing.assert_close(rout, sh, rtol=1e-6, atol=1e-6)
        torch.testing.assert_close(ep_k, ep, rtol=1e-6, atol=1e-5)
        torch.testing.assert_close(meter_k[:5].cpu(), torch.tensor(meter, dtype=torch.float64), rtol=1e-9, atol=1e-9)
        other = runs[1][s]
        assert torch.equal(other[6], sel) and torch.equal(other[7], ep_k)
        assert torch.equal(other[8], meter_k), 'the meter is not bit-reproducible'


@pytest.mark.parametrize('N,G', [(1, 2), (37, 3), (4096, 4), (250_000, 4)])
@pytest.mark.parametrize('normalize_value', [False, True])
def test_cv_value_broadcast_matches_torch_repeat(N, G, normalize_value):
    """central_value.py:224-226: value.repeat(1, G).view(N * G, -1) of the de-normalised critic values"""
    from rl_games_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(N + G)
    val = torch.randn(N, 1, generator=g, device=DEV) * 3
    mean, var = torch.tensor([0.7], dtype=torch.float64, device=DEV), torch.tensor([2.5], dtype=torch.float64, device=DEV)
    out = torch.full((N * G,), float('nan'), device=DEV)
    ops.cv_value_broadcast(val, mean, var, normalize_value, out, N, G)
    v = val
    if normalize_value:
        v = torch.sqrt(var.float() + 1e-5) * torch.clamp(val, -5.0, 5.0) + mean.float()
    assert torch.equal(out, v.repeat(1, G).view(N * G, -1).reshape(-1))


@pytest.mark.parametrize('H,N,G', [(1, 1, 2), (8, 37, 3), (16, 4096, 4), (32, 8192, 3)])
def test_cv_gather_agent0_matches_update_multiagent_tensors(H, N, G):
    """central_value.py:235-244 on the flat [env*G*H] batch: view (N, G, H), transpose (G, N, H), first N*H rows; against the kernel's
    [H, N] critic arena read back in the flat env*H + t order"""
    from rl_games_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(H * N * G)
    a, b = torch.randn(H, N * G, generator=g, device=DEV), torch.randn(H, N * G, generator=g, device=DEV)
    da, db = torch.full((H, N), float('nan'), device=DEV), torch.full((H, N), float('nan'), device=DEV)
    ops.cv_gather_agent0(a, b, da, db, H, N, G)
    fl = O.swap_and_flatten01
    for src, dst in ((a, da), (b, db)):
        ref = fl(src).view(N, G, H).transpose(0, 1).contiguous().view(N * G * H)[:N * H]
        assert torch.equal(fl(dst), ref)


class _CVEnvGPU(TapeEnvGPU):
    def __init__(self, g):
        super().__init__(g['obs_tape'], g['done_tape'], g['timeout_tape'], g['A'])
        self.state_tape, self.S, self.G = g['state_tape'].to(DEV), g['S'], g['G']

    def _o(self, j):
        return {'obs': self.obs_tape[j].clone(), 'states': self.state_tape[j].clone()}

    def reset(self):
        self.i = 0
        return self._o(0)

    def step(self, actions):
        o, rew, done, info = super().step(actions)
        return self._o(self.i % self.obs_tape.shape[0]), rew, done, info

    def get_env_info(self):
        from rl_games_b200.common import Box
        return dict(super().get_env_info(), agents=self.G, state_space=Box(-float('inf'), float('inf'), (self.S,)))


@pytest.mark.parametrize('graph', [False, True])
def test_central_value_agent_with_agents_matches_reference_golden(graph):
    from rl_games_b200.agent_cv import A2CAgentCV
    g = torch.load(os.path.join(GOLDEN, 'agent_ma_cv.pt'), weights_only=False)
    cv_cfg = dict(g['cv_config'])
    cv_cfg['network'] = {'name': 'actor_critic', 'central_value': True,
                         'mlp': {'units': [24, 12], 'activation': 'elu', 'initializer': {'name': 'default'}}}
    cfgk = g['config']
    cfg = {k: cfgk[k] for k in ('clip_value', 'use_smooth_clamp', 'bound_loss_type', 'bounds_loss_coef', 'entropy_coef', 'truncate_grads',
                                'value_bootstrap', 'mini_epochs', 'lr_schedule', 'critic_coef', 'learning_rate', 'kl_threshold',
                                'normalize_input', 'normalize_value', 'normalize_advantage', 'e_clip', 'tau', 'gamma') if k in cfgk}
    cfg.update({'b200_cuda_graph': graph, 'central_value_config': cv_cfg})
    env = _CVEnvGPU(g)
    agent = make_agent(cfg, g['N'], g['H'], g['D'], g['A'], g['units'], g['mb'], env, g['init_state'])
    assert isinstance(agent, A2CAgentCV)
    cv = agent.central_value_net
    cv.load_state_dict({k: v.to(DEV) for k, v in g['cv_init_state'].items()})
    agent.obs = agent.env_reset()
    fl = O.swap_and_flatten01
    for ep, ref in enumerate(g['epochs_out']):
        agent.epoch_num += 1
        agent.train_epoch(noise=g['noise'][ep][:g['H']].to(DEV))
        torch.testing.assert_close(agent.values.cpu().unsqueeze(2), ref['mb_values'], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(agent.rewards.cpu().unsqueeze(2), ref['mb_rewards'], rtol=1e-5, atol=1e-6)
        cds = ref['cv_dataset']
        torch.testing.assert_close(fl(cv.old_values_n).unsqueeze(1).cpu(), cds['old_values'], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(fl(cv.returns_n).unsqueeze(1).cpu(), cds['returns'], rtol=1e-4, atol=1e-5)
        st = agent.last_stats
        torch.testing.assert_close(st[:, 0].cpu(), ref['a_losses'], rtol=2e-3, atol=2e-6)
        torch.testing.assert_close(st[:, 1].cpu(), ref['c_losses'], rtol=2e-3, atol=2e-6)
        assert agent.last_lr == pytest.approx(ref['last_lr'], rel=1e-12) and cv.lr == pytest.approx(ref['cv_lr'], rel=1e-12)
        sd, csd = agent.model.state_dict(), cv.state_dict()
        for k in O.param_names(len(g['units'])):
            torch.testing.assert_close(sd[k].cpu(), ref['state'][k], rtol=1e-3, atol=2e-5, msg=lambda m: k + ': ' + m)
        for k in cv.param_names():
            torch.testing.assert_close(csd[k].cpu(), ref['cv_state'][k], rtol=1e-3, atol=2e-5, msg=lambda m: 'cv ' + k + ': ' + m)
        assert agent.game_rewards.current_size == ref['game_rewards_size']
        torch.testing.assert_close(agent.game_rewards.mean, ref['game_rewards_mean'].reshape(-1), rtol=1e-4, atol=1e-5)


def test_discrete_agent_with_agents_and_action_masks_matches_reference_golden():
    """discrete, separate trunks, action masks, G = 4 (the ppo_smac shape): two train_epoch()s against the reference's run"""
    from test_discrete_gpu import DiscreteTapeEnvGPU
    from rl_games_b200.runner import Runner
    g = torch.load(os.path.join(GOLDEN, 'agent_ma_discrete.pt'), weights_only=False)
    env = DiscreteTapeEnvGPU(g)
    base_info = env.get_env_info
    env.get_env_info = lambda: dict(base_info(), agents=g['G'])
    config = {k: v for k, v in g['config'].items() if k not in ('device', 'torch_compile')}
    config.update({'device': DEV, 'env_info': env.get_env_info(), 'vec_env': env, 'reward_shaper': {'scale_value': 0.1},
                   'train_dir': '/tmp/b200_parity_runs', 'lr_schedule': g['config'].get('lr_schedule', None)})
    network = {'name': 'actor_critic', 'separate': g['separate'], 'space': {'discrete': None},
               'mlp': {'units': g['units'], 'activation': 'relu', 'initializer': {'name': 'default'}}}
    r = Runner()
    r.load({'params': {'seed': 1, 'algo': {'name': 'a2c_discrete'}, 'model': {'name': 'discrete_a2c'}, 'network': network, 'config': config}})
    r.params['config']['vec_env'] = env
    agent = r.algo_factory.create(r.algo_name, base_name='parity', params=r.params)
    agent.model.load_state_dict({k: v.to(DEV) for k, v in g['init_state'].items()}, strict=False)
    agent.init_tensors()
    agent.obs = agent.env_reset()
    assert agent.num_rows == g['N'] * g['G']
    seen = []
    agent.algo_observer.wants_done_indices = True
    agent.algo_observer.process_infos = lambda infos, idx: seen.append(idx.cpu().clone())
    fl = lambda t: t.transpose(0, 1).reshape(-1, *t.shape[2:])    # noqa: E731
    for ep, ref in enumerate(g['epochs_out']):
        seen.clear()
        agent.epoch_num += 1
        res = agent.train_epoch(u=g['u'][ep].to(DEV))
        assert [s.tolist() for s in seen] == [st['done_indices'].tolist() for st in ref['steps']]
        assert (agent.actions.cpu() == ref['mb_actions']).all()
        torch.testing.assert_close(agent.values.cpu().unsqueeze(2), ref['mb_values'], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(fl(agent.advs_n).cpu(), ref['dataset']['advantages'], rtol=2e-4, atol=2e-5)
        torch.testing.assert_close(torch.stack(res[4]).cpu(), ref['a_losses'], rtol=2e-3, atol=2e-6)
        torch.testing.assert_close(torch.stack(res[5]).cpu(), ref['c_losses'], rtol=2e-3, atol=2e-6)
        sd = agent.model.state_dict()
        for k in g['param_order']:
            torch.testing.assert_close(sd[k].cpu(), ref['state'][k], rtol=1e-3, atol=2e-5, msg=lambda m: k + ': ' + m)
        assert agent.game_rewards.current_size == ref['game_rewards_size']
        torch.testing.assert_close(agent.game_rewards.mean, ref['game_rewards_mean'].reshape(-1), rtol=1e-4, atol=1e-5)


def _golden(name, graph, over=None):
    g = torch.load(os.path.join(GOLDEN, name), weights_only=False)
    cfgk = g['config']
    cfg = {k: cfgk[k] for k in ('clip_value', 'use_smooth_clamp', 'bound_loss_type', 'bounds_loss_coef', 'entropy_coef', 'truncate_grads',
                                'value_bootstrap', 'mini_epochs', 'lr_schedule', 'critic_coef', 'seq_length', 'learning_rate',
                                'kl_threshold', 'normalize_input', 'normalize_value', 'normalize_advantage', 'e_clip', 'tau',
                                'gamma') if k in cfgk}
    cfg['b200_cuda_graph'] = graph
    cfg.update(over or {})
    env = TapeEnvGPU(g['obs_tape'], g['done_tape'], g['timeout_tape'], g['A'])
    base_info = env.get_env_info
    env.get_env_info = lambda: {**base_info(), 'agents': g['G']}
    return g, make_agent(cfg, g['N'], g['H'], g['D'], g['A'], g['units'], g['mb'], env, g['init_state'], rnn_units=g['rnn_units'])


@pytest.mark.parametrize('name', ['agent_ma.pt', 'agent_ma_lstm.pt'])
@pytest.mark.parametrize('graph', [False, True])
def test_multiagent_agent_matches_reference_golden(name, graph):
    g, agent = _golden(name, graph)
    assert agent.num_rows == g['N'] * g['G'] and not agent.use_tc
    seen = []
    agent.algo_observer.wants_done_indices = True
    agent.algo_observer.process_infos = lambda infos, idx: seen.append(idx.cpu().clone())
    for ep, ref in enumerate(g['epochs_out']):
        seen.clear()
        agent.epoch_num += 1
        agent.train_epoch(noise=g['noise'][ep].to(DEV))
        assert [s.tolist() for s in seen] == [r['done_indices'].tolist() for r in ref['steps']]
        assert torch.equal(agent.dones_buf.cpu(), ref['mb_dones'])
        torch.testing.assert_close(agent.values.cpu().unsqueeze(2), ref['mb_values'], rtol=1e-4, atol=1e-5)
        _check_epoch(agent, ref['state'], ref['dataset'], {'a': ref['a_losses'], 'c': ref['c_losses'], 'e': ref['entropies']},
                     ref['last_lr'], g['units'], lstm=g['rnn_units'] > 0)
        assert agent.game_rewards.current_size == ref['game_rewards_size']
        torch.testing.assert_close(agent.game_rewards.mean, ref['game_rewards_mean'].reshape(-1), rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(agent.game_lengths.mean, ref['game_lengths_mean'].reshape(-1), rtol=1e-4, atol=1e-5)


def test_layerwise_tensor_core_path_tracks_fp32_agent():
    """mixed_precision: True with G = 4 on an MLP wider than the fused tiles runs every GEMM on the tensor cores layer by layer; bf16
    tolerance class against the fp32 agent (as tests/test_agent_gpu.py::test_layerwise_tensor_core_path_tracks_fp32_agent)"""
    N, G, H, D, A, mb, units = 64, 4, 8, 44, 5, 1024, [512, 256, 128]
    obs_tape, done_tape, tout_tape = O.make_tapes(H + 1, N * G, D, seed=61, p_done=0.1)
    params = O.init_params(D, units, A, seed=7)
    noise = torch.randn(H, N * G, A, generator=torch.Generator().manual_seed(5)).to(DEV)
    agents = []
    for mp in (False, True):
        env = TapeEnvGPU(obs_tape, done_tape, tout_tape, A)
        base_info = env.get_env_info
        env.get_env_info = lambda base_info=base_info: {**base_info(), 'agents': G}
        a = make_agent({'mixed_precision': mp, 'mini_epochs': 2, 'b200_cuda_graph': False}, N, H, D, A, units, mb, env, params)
        assert a.gemm_tc == mp and not a.use_tc and a.num_rows == N * G
        a.epoch_num += 1
        a.train_epoch(noise=noise)
        agents.append(a)
    f, t = agents
    torch.testing.assert_close(t.values, f.values, rtol=0, atol=6e-2)
    torch.testing.assert_close(t.mus, f.mus, rtol=0, atol=6e-2)
    torch.testing.assert_close(t.last_stats[:, 0], f.last_stats[:, 0], rtol=0.1, atol=2e-2)
    torch.testing.assert_close(t.last_stats[:, 1], f.last_stats[:, 1], rtol=0.1, atol=2e-2)
    # the same done rows feed both meters; the rewards they average come from actions of two precisions
    assert torch.equal(t.meter[3:5], f.meter[3:5]) and int(f.meter[4]) > 0
    torch.testing.assert_close(t.meter[:3], f.meter[:3], rtol=0, atol=2e-2)


def _synth_agent(N, G, graph, mixed_precision=True):
    import bench
    from rl_games_b200.runner import Runner
    w = dict(bench.WORKLOADS['c2'], num_actors=N)
    params = bench.make_params(w, DEV, 'b200_synthetic', False, graph=graph, mixed_precision=mixed_precision)
    params['config']['env_config'] = dict(params['config'].get('env_config', {}), agents=G)
    params['config']['minibatch_size'] = w['minibatch']
    r = Runner()
    r.load({'params': params})
    agent = r.algo_factory.create(r.algo_name, base_name='ma_gpu', params=r.params)
    agent.init_tensors()
    agent.obs = agent.env_reset()
    return agent


def test_fused_wgmma_agent_with_four_agents_trains_like_the_same_rows_as_one_agent():
    """c2-like geometry (16384 rows x horizon 16, obs 60, 8 actions, [256, 128, 64], minibatch 32768) on the fused kernels: 4096 envs x 4
    agents and 16384 envs x 1 agent are the same rows, so the rollout, the update and the weights are bit-identical; only the meters
    differ, and they follow dones.nonzero()[::4] replayed in torch from the arena's done flags"""
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    a1, a4 = _synth_agent(16384, 1, False), _synth_agent(4096, 4, False)
    assert a1.use_tc and a4.use_tc and a4.num_rows == a1.num_rows == 16384
    for a in (a1, a4):
        a.epoch_num += 1
        a.train_epoch()
    torch.cuda.synchronize()
    for x, y in ((a1.values, a4.values), (a1.rewards, a4.rewards), (a1.dones_buf, a4.dones_buf), (a1.model.flat, a4.model.flat)):
        assert torch.equal(x, y)
    # the env's dones of rollout step t are the arena's dones of step t + 1 (the last ones are the agent's current dones)
    H = a4.horizon_length
    step_dones = [a4.dones_buf[t + 1] if t + 1 < H else a4.dones for t in range(H)]
    n_done = [int(d.sum()) for d in step_dones]
    assert sum(n_done) > 0
    assert int(a1.meter[4].item()) == sum(n_done)
    # torch replay of the reference's accounting at this geometry: no time-outs inside the first horizon (max_len 100) and a unit reward
    # shaper, so the arena's shaped rewards are the env's rewards
    ep = torch.zeros(3, 16384, device=DEV)
    zeros = torch.zeros(16384, dtype=torch.uint8, device=DEV)
    for G, agent in ((1, a1), (4, a4)):
        ep.zero_()
        meter = [0.0] * 5
        for t in range(H):
            _ref_step(agent.rewards[t], step_dones[t], zeros, agent.values[t], ep, meter, G, agent.games_to_track)
        assert int(agent.meter[4].item()) == meter[4] and agent.game_rewards.current_size == meter[3]
        torch.testing.assert_close(agent.meter[:4].cpu(), torch.tensor(meter[:4], dtype=torch.float64), rtol=1e-9, atol=1e-9)
        torch.testing.assert_close(agent.ep_state, ep, rtol=1e-6, atol=1e-5)


def test_whole_epoch_cuda_graph_matches_eager_epochs_with_agents():
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    eager, graph = _synth_agent(1024, 4, False), _synth_agent(1024, 4, True)
    for _ in range(3):
        for a in (eager, graph):
            a.epoch_num += 1
            a.train_epoch()
    torch.cuda.synchronize()
    assert graph._graph_epoch is not None and eager._graph_epoch is None
    assert torch.equal(eager.meter, graph.meter)
    assert torch.equal(eager.model.flat, graph.model.flat)
