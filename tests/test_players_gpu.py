"""The CUDA players on the GPU: the deterministic categorical head kernel against torch.argmax at every head layout; every player family
against the reference's players on their recorded tapes (tests/golden/players_*.pt: fp32 within 1e-5, the bf16 tensor-core arms within a
stated bf16 bound, argmax exact on rows with a clear margin, recurrent states included); a policy trained here against the reference's player
on the same checkpoint; sampled actions from noise / uniform tapes; and the graph-replayed step against the eager step, bit for bit, over
episodes with dones."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import test_players_cpu as PC  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _argmax_ref(z, masks, sizes):
    out, off = [], 0
    for k in sizes:
        zj, mj = z[:, off:off + k], masks[:, off:off + k].bool()
        a = torch.where(mj, zj, torch.full_like(zj, -float('inf'))).argmax(dim=1)
        out.append(torch.where(mj.any(dim=1), a, torch.zeros_like(a)))
        off += k
    return torch.stack(out, dim=1)


def _layouts():
    g = np.random.default_rng(0)
    lay = [[k] for k in range(1, 65)] + [[64] * h for h in range(1, 9)]
    lay += [list(g.integers(1, 65, size=h)) for h in range(2, 9) for _ in range(4)]
    return lay


@pytest.mark.parametrize('ld_pad', [0, 3])
def test_categorical_argmax_matches_torch_argmax_at_every_layout(ld_pad):
    from rl_games_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(1)
    N = 515
    for sizes in _layouts():
        sizes = [int(k) for k in sizes]
        K = sum(sizes)
        ld = K + ld_pad
        # few distinct values: many ties, which go to the lowest index
        z = torch.randint(-3, 4, (N, ld), generator=g, device=DEV).float() * 0.5
        masks = (torch.rand(N, K, generator=g, device=DEV) < 0.7).to(torch.uint8)
        masks[:7] = 0                                           # all-masked rows
        masks[7:9] = 1
        hs = sizes if len(sizes) > 1 else None
        out = torch.full((N, len(sizes)), -1, dtype=torch.int64, device=DEV)
        ops.categorical_argmax(z, ld, K, masks, out, N, head_sizes=hs)
        assert torch.equal(out, _argmax_ref(z[:, :K], masks, sizes)), sizes
        ops.categorical_argmax(z, ld, K, None, out, N, head_sizes=hs)
        assert torch.equal(out, _argmax_ref(z[:, :K], torch.ones_like(masks), sizes)), sizes


def _gpu_params(algo, env, net, over=None, player=None):
    p = PC._params(algo, env, net, over, player)
    p['config']['device_name'] = DEV
    return p


def _to_dev_env(env):
    step, reset = env.step, env.reset
    env.reset = lambda: reset().to(DEV)
    env.step = lambda a: tuple(x.to(DEV) if torch.is_tensor(x) else x for x in step(a))
    return env


MLP3 = dict(PC.MLP, mlp={'units': [64, 32, 16], 'activation': 'elu', 'initializer': {'name': 'default'}})


def _cont_ref(p, obs):
    """fp64 forward of the continuous policy (trunk, optional LSTM, head), from the player's own weights"""
    m = p.model
    r = m.running_mean_std
    x = torch.clamp((obs.double() - r.running_mean) / torch.sqrt(r.running_var + 1e-5), -5, 5)
    h = x
    for W, b in zip(m.W, m.b):
        h = torch.nn.functional.elu(h @ W.double().t() + b.double())
    head = h @ m.W_head.double().t() + m.b_head.double()
    return head[:, 1:]


@pytest.mark.parametrize('arm', ['fp32', 'tc_fused', 'tc_rollout_fp32'])
def test_continuous_deterministic_actions(arm):
    from rl_games_b200.common import Box
    from rl_games_b200.players import PpoPlayerContinuous
    over = {'fp32': {'mixed_precision': False}, 'tc_fused': {'mixed_precision': True},
            'tc_rollout_fp32': {'mixed_precision': True, 'b200_rollout_fp32': True}}[arm]
    env = _to_dev_env(PC._Env(300, 12, Box(np.array([-2.0, 0.0, -1.0]), np.array([2.0, 1.0, 1.0]), (3,))))
    p = PpoPlayerContinuous(_gpu_params('a2c_continuous', env, MLP3, over))
    assert p.use_tc == (arm != 'fp32') and p.rollout_fp32 == (arm == 'tc_rollout_fp32')
    PC._randomise(p.model)
    with torch.no_grad():
        p.model.flat.mul_(0.3)
    p._weights_loaded()
    obs = env.reset()
    p.get_batch_size(obs, 1)
    a = p.get_action(obs, True)
    mu = _cont_ref(p, obs).float()
    want = torch.clamp(mu, -1, 1) * (p.actions_high - p.actions_low) / 2 + (p.actions_high + p.actions_low) / 2
    # bf16 operands, fp32 accumulation over <= 64-wide layers: a few bf16 ulps of the O(1) activations
    tol = 1e-5 if arm != 'tc_fused' else 3e-2
    torch.testing.assert_close(a, want, rtol=0, atol=tol)
    p.noise = torch.randn(300, 3, device=DEV)
    p.clip_actions = False
    a = p.get_action(obs, False)
    sig = torch.exp(p.model.sigma)
    torch.testing.assert_close(a, mu + sig * p.noise, rtol=0, atol=tol * 4)


def test_discrete_deterministic_and_sampled_actions():
    from rl_games_b200.common import Discrete, Tuple
    from rl_games_b200.players import PpoPlayerDiscrete
    sizes = [5, 7, 3]
    K = sum(sizes)
    g = torch.Generator(device=DEV).manual_seed(3)
    masks = (torch.rand(257, K, generator=g, device=DEV) < 0.7).to(torch.uint8)
    env = _to_dev_env(PC._Env(257, 10, Tuple([Discrete(k) for k in sizes]), masks=masks))
    net = dict(PC.DISCRETE, space={'multi_discrete': None})
    for over in ({}, {'mixed_precision': True}):
        params = _gpu_params('a2c_discrete', env, net, over)
        params['model']['name'] = 'multi_discrete_a2c'
        p = PpoPlayerDiscrete(params)
        PC._randomise(p.model, 3)
        p._weights_loaded()
        obs = env.reset()
        p.get_batch_size(obs, 1)
        a = p.get_masked_action(obs, masks, True)
        z = p.r_a[-1][:, 1:]
        assert torch.equal(a, _argmax_ref(z, masks, sizes))
        # sampled: the inverse-CDF draw of the uniform tape, restated in the kernel's fp32 order of operations (cat_lse, cat_sample_row)
        p.u = torch.rand(len(sizes), 257, generator=g, device=DEV)
        a = p.get_masked_action(obs, masks, False)
        off, want, near = 0, [], torch.zeros(257, dtype=torch.bool, device=DEV)
        for j, k in enumerate(sizes):
            zj = torch.where(masks[:, off:off + k].bool(), z[:, off:off + k], torch.tensor(-1e8, device=DEV))
            m = zj.max(-1).values
            s_ = torch.zeros_like(m)
            for i in range(k):
                s_ = s_ + torch.exp(zj[:, i] - m)
            lse = m + torch.log(s_)
            cdf, cnt, last = torch.zeros_like(m), torch.zeros_like(m, dtype=torch.int64), torch.zeros_like(m, dtype=torch.int64)
            for i in range(k):
                pi = torch.exp(zj[:, i] - lse)
                cdf = cdf + pi
                cnt += (cdf <= p.u[j]).long()
                last = torch.where(pi > 0, torch.full_like(last, i), last)
                near |= (cdf - p.u[j]).abs() < 1e-6         # a uniform within an ulp or two of a cdf step: exp / log may round apart
            want.append(torch.minimum(cnt, last))
            off += k
        assert int(near.sum()) < 3
        assert torch.equal(a[~near], torch.stack(want, -1)[~near])


def test_sac_deterministic_and_sampled_actions():
    from rl_games_b200.common import Box
    from rl_games_b200.players import SACPlayer
    env = _to_dev_env(PC._Env(129, 6, Box(np.array([-2.0, 0.0]), np.array([2.0, 1.0]), (2,))))
    p = SACPlayer(_gpu_params('sac', env, PC.SAC_NET, {'normalize_input': False}))
    with torch.no_grad():
        p.model.actor.flat.copy_(torch.randn(p.model.actor.flat.shape, generator=torch.Generator().manual_seed(5)).to(DEV) * 0.3)
    obs = env.reset()
    p.get_batch_size(obs, 1)
    a = p.get_action(obs, True)
    h = obs.double()
    for lay in p.model.actor_mlp[:-1]:
        h = torch.relu(h @ lay.W.double().t() + lay.b.double())
    head = h @ p.model.actor_mlp[-1].W.double().t() + p.model.actor_mlp[-1].b.double()
    mu, raw = head[:, :2], head[:, 2:]
    sc, bi = p.action_scale.double(), p.action_bias.double()
    lo, hi = p.action_low.double(), p.action_high.double()
    torch.testing.assert_close(a.double(), (torch.tanh(mu) * sc + bi).clamp(lo, hi), rtol=0, atol=1e-5)
    p.noise = torch.randn(129, 2, device=DEV)
    a = p.get_action(obs, False)
    ls = -5 + 0.5 * 7 * (torch.tanh(raw) + 1)
    x = mu + p.noise.double() * ls.exp()
    torch.testing.assert_close(a.double(), (torch.tanh(x) * sc + bi).clamp(lo, hi), rtol=0, atol=1e-5)


def _episode(p, env, steps, deterministic):
    obs = env.reset()
    p.get_batch_size(obs, 1)
    p.init_rnn()
    acts = []
    for _ in range(steps):
        a = p.get_action(obs, deterministic)
        acts.append(a.clone())
        obs, r, done, _ = env.step(a)
        p._done_rows(done)
    torch.cuda.synchronize()
    return torch.stack(acts)


@pytest.mark.parametrize('case', ['lstm_ln', 'lstm_after', 'mlp_tc', 'sd_sigma', 'discrete', 'sac'])
def test_graph_replay_equals_eager_bit_for_bit(case):
    from rl_games_b200.common import Box, Discrete
    from rl_games_b200 import players
    box = Box(-np.ones(3), np.ones(3), (3,))
    if case == 'discrete':
        mk = lambda: _to_dev_env(PC._Env(64, 10, Discrete(6)))                              # noqa: E731
        build = lambda env, over: players.PpoPlayerDiscrete(_gpu_params('a2c_discrete', env, PC.DISCRETE, over))   # noqa: E731
    elif case == 'sac':
        mk = lambda: _to_dev_env(PC._Env(64, 10, box))                                      # noqa: E731
        build = lambda env, over: players.SACPlayer(_gpu_params('sac', env, PC.SAC_NET, over))   # noqa: E731
    else:
        net = {'lstm_ln': dict(PC.MLP, rnn={'name': 'lstm', 'units': 32, 'layers': 1, 'before_mlp': True, 'layer_norm': True}),
               'lstm_after': dict(PC.MLP, rnn={'name': 'lstm', 'units': 32, 'layers': 1, 'before_mlp': False}),
               'mlp_tc': MLP3,
               'sd_sigma': dict(PC.MLP, space={'continuous': dict(PC.MLP['space']['continuous'], fixed_sigma=False)})}[case]
        mk = lambda: _to_dev_env(PC._Env(64, 10, box))                                      # noqa: E731
        build = lambda env, over: players.PpoPlayerContinuous(_gpu_params('a2c_continuous', env, net, dict(over, mixed_precision=case != 'sd_sigma')))   # noqa: E731
    runs = []
    for graph in (False, True):
        env = mk()
        p = build(env, {'b200_cuda_graph': graph})
        model = p.model
        flat = model.actor.flat if case == 'sac' else model.flat
        with torch.no_grad():
            flat.copy_(torch.randn(flat.shape, generator=torch.Generator().manual_seed(9)).to(DEV) * 0.3)
        if case != 'sac':
            p._weights_loaded()
        runs.append(torch.cat([_episode(p, env, 12, True).float().flatten(), _episode(p, env, 12, False).float().flatten()]))
        if graph:
            assert len(p._graphs) == 2
    assert any(bool(d.any()) for d in env.dones)
    assert torch.equal(runs[0], runs[1])


# ---------------------------------------------------------------------------------------------------------------- against the reference players
GOLDEN = os.path.join(HERE, 'golden')
FIXTURES = sorted(f[len('players_'):-3] for f in os.listdir(GOLDEN) if f.startswith('players_') and f.endswith('.pt'))
# bf16 operands with fp32 accumulation (fused wgmma MLP, layer-wise wgmma GEMMs and LSTM gates): |got - ref| <= BF16_ATOL + BF16_RTOL |ref|.
# The absolute part covers a few bf16 ulps (2^-8 relative) of the O(1) pre-activations; the relative part covers outputs that pass
# through exp (a state-dependent sigma of ~8 carries the head's absolute bf16 error as a relative one)
BF16_ATOL, BF16_RTOL = 5e-2, 2e-2


def _fixture_player(fx, over, tmp_path):
    from rl_games_b200.common import Box, Discrete, Tuple
    from rl_games_b200 import players
    if fx['frames']:
        obs_space = Box(0, 255, tuple(fx['frames']), np.uint8)
    else:
        obs_space = Box(-np.inf, np.inf, (fx['obs'].shape[-1],))
    K = fx['K']
    if fx['algo'] == 'a2c_discrete':
        space = Tuple([Discrete(k) for k in K]) if isinstance(K, list) else Discrete(K)
    else:
        space = Box(fx['low'], fx['high'], (len(fx['low']),))
    params = {k: v for k, v in fx['params'].items()}
    config = dict(params['config'], device_name=DEV, b200_cuda_graph=True, **over)
    config.update(env_info={'observation_space': obs_space, 'action_space': space, 'agents': fx['agents']}, vec_env=None)
    params['config'] = config
    cls = {'a2c_continuous': players.PpoPlayerContinuous, 'a2c_discrete': players.PpoPlayerDiscrete, 'sac': players.SACPlayer}[fx['algo']]
    p = cls(params)
    fn = str(tmp_path / 'ck.pth')
    torch.save(fx['state'], fn)
    p.restore(fn)
    return p


@pytest.mark.parametrize('arm', ['fp32', 'bf16'])
@pytest.mark.parametrize('case', FIXTURES)
def test_players_match_the_reference_players(case, arm, tmp_path):
    fx = torch.load(os.path.join(GOLDEN, f'players_{case}.pt'), weights_only=False)
    if fx['algo'] == 'sac' and arm == 'bf16':
        pytest.skip("the SAC rollout's actor runs on the fp32 kernels whatever mixed_precision says (as SACAgent's)")
    p = _fixture_player(fx, {'mixed_precision': arm == 'bf16'}, tmp_path)
    tol, rtol = (1e-5, 0) if arm == 'fp32' else (BF16_ATOL, BF16_RTOL)
    clear_rows = 0
    for t in range(fx['obs'].shape[0]):
        obs = fx['obs'][t].to(DEV)
        if t == 0:
            p.get_batch_size(obs, 1)
            p.init_rnn()
        if fx['masks'] is not None:
            a = p.get_masked_action(obs, fx['masks'][t].to(DEV), True)
        else:
            a = p.get_action(obs, True)
        want = fx['actions'][t].to(DEV)
        if fx['algo'] == 'a2c_discrete':
            clear = fx['clear'][t].to(DEV)
            got = a.reshape(clear.shape)
            assert torch.equal(got[clear], want.reshape(clear.shape)[clear]), (t, got, want)
            clear_rows += int(clear.sum())
        else:
            torch.testing.assert_close(a, want, rtol=rtol, atol=tol)
            if fx['algo'] == 'a2c_continuous':
                torch.testing.assert_close(p.mus[0], fx['mu'][t].to(DEV), rtol=rtol, atol=tol)
                torch.testing.assert_close(p.sigmas[0], fx['sigma'][t].to(DEV), rtol=rtol, atol=tol)
        if fx['rnn_h'] is not None:
            torch.testing.assert_close(p.rnn_h, fx['rnn_h'][t].to(DEV), rtol=rtol, atol=tol)
            torch.testing.assert_close(p.rnn_c, fx['rnn_c'][t].to(DEV), rtol=rtol, atol=tol)
        p._done_rows(fx['dones'][t].to(DEV))
    if fx['algo'] == 'a2c_discrete':
        assert clear_rows >= fx['clear'].numel() // 2


def test_trained_checkpoint_plays_like_the_reference_player(tmp_path):
    """a policy trained for a few epochs here, played here and by the reference's player on the same checkpoint"""
    from oracle import ppo_oracle as O, ref_arm
    if not ref_arm.available():
        pytest.skip('reference rl_games not present (oracle/_ref)')
    import test_agent_gpu as TA
    from rl_games_b200.players import PpoPlayerContinuous
    N, H, D, A, units, mb = 64, 8, 6, 3, [32, 16], 128
    obs_tape, done_tape, tout_tape = O.make_tapes(H + 1, N, D, seed=1)
    agent = TA.make_agent({'mini_epochs': 2}, N, H, D, A, units, mb, TA.TapeEnvGPU(obs_tape, done_tape, tout_tape, A),
                          O.init_params(D, units, A, seed=2))
    for _ in range(3):
        agent.epoch_num += 1
        agent.train_epoch()
    agent.save(str(tmp_path / 'ck'))
    fn = str(tmp_path / 'ck.pth')
    ref_arm.import_reference()
    import gymnasium as gym
    from rl_games.algos_torch.players import PpoPlayerContinuous as RefPlayer
    low, high = -np.ones(A, np.float32), np.ones(A, np.float32)
    mk = lambda dev, spaces: {'seed': 7, 'algo': {'name': 'a2c_continuous'}, 'model': {'name': 'continuous_a2c_logstd'},   # noqa: E731
                              'network': agent.network_params,
                              'config': {'env_name': 'tape', 'env_info': spaces, 'vec_env': None, 'device_name': dev,
                                         'normalize_input': True, 'normalize_value': True, 'mixed_precision': False}}
    from rl_games_b200.common import Box
    ours = PpoPlayerContinuous(mk(DEV, {'observation_space': Box(-np.inf, np.inf, (D,)), 'action_space': Box(low, high, (A,))}))
    ref = RefPlayer(mk('cpu', {'observation_space': gym.spaces.Box(-np.inf, np.inf, (D,), np.float32),
                               'action_space': gym.spaces.Box(low, high, (A,), np.float32)}))
    ours.restore(fn)
    ref.restore(fn)
    obs = torch.randn(5, N, D, generator=torch.Generator().manual_seed(4)) * 2
    ours.get_batch_size(obs[0], 1)
    ref.get_batch_size(obs[0], 1)
    for t in range(obs.shape[0]):
        a = ours.get_action(obs[t].to(DEV), True)
        with torch.no_grad():
            want = ref.get_action(obs[t], True)
        torch.testing.assert_close(a.cpu(), want, rtol=0, atol=1e-5)
