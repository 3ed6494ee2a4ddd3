"""The wide categorical kernels (csrc/discrete.cu categorical_{sample,loss}_wide_kernel, csrc/player.cu categorical_argmax_wide_kernel)
on the GPU: against fp64 at single heads of 65, 362 and 4672 actions and at 9, 64 and 1792 heads, with unmasked, masked and all-masked
heads, on NaN-filled output buffers; the Philox draws bit for bit; the argmax exhaustively at head sizes 65-256; repeated runs bit-equal;
the agent against the reference's golden runs (tests/golden/gen_golden_cat_wide.py); the player on a wide-head checkpoint."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _cat_wide_ref as W  # noqa: E402
from oracle import ppo_discrete_oracle as DO  # noqa: E402
from oracle.ppo_oracle import actor_loss, critic_loss  # noqa: E402

pytestmark = [pytest.mark.gpu]
DEV = 'cuda:0'
MICRORTS_HEADS = [6, 4, 4, 4, 4, 7, 49] * 256
_g64 = np.random.default_rng(64)
LAYOUTS = {'K65': (65, None), 'K362': (362, None), 'K4672': (4672, None),
           'h9': (None, [3, 70, 5, 1, 65, 4, 9, 2, 6]), 'h64': (None, [int(k) for k in _g64.integers(1, 80, 64)]),
           'h1792': (None, MICRORTS_HEADS)}
ROWS = {'K65': 600, 'K362': 400, 'K4672': 200, 'h9': 600, 'h64': 300, 'h1792': 96}


def _layout(name):
    K, sizes = LAYOUTS[name]
    sizes = sizes or [K]
    return sum(sizes), sizes, (None if len(sizes) == 1 else sizes)


def _inputs(name, masked, seed):
    """logits [M, K], masks (None, or per row: unmasked, random legal subsets, or every third head fully masked)"""
    K, sizes, _ = _layout(name)
    M = ROWS[name]
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(M, K, generator=g) * 2
    if not masked:
        return z, None
    mk = torch.rand(M, K, generator=g) < 0.5
    off = 0
    for j, k in enumerate(sizes):
        mk[torch.arange(M), off + torch.randint(0, k, (M,), generator=g)] = True          # one legal action per head ...
        if j % 3 == 1:
            mk[2::3, off:off + k] = False                                                   # ... except whole heads of every third row
        off += k
    mk[0::3] = True
    return z, mk


def _heads64(z, mk, sizes):
    """per head (fp64 normalised logits, probs, entropy, all-masked flag); -1e8 for masked logits.  A fully masked head's normalised
    logits are what the reference computes in its fp32: every logit -1e8 and the log-sum-exp -1e8 + log K rounded to fp32 (a step of
    8 at 1e8), so its neglogp is 0 or 8, not log K; its entropy and gradient are 0"""
    out, off = [], 0
    for k in sizes:
        zz = z[:, off:off + k].double()
        mm = None if mk is None else mk[:, off:off + k]
        nl, p, e = DO.categorical_masked(zz, mm)
        dead = torch.zeros(z.shape[0], dtype=torch.bool, device=z.device) if mm is None else ~mm.any(1)
        nl32 = DO.categorical_masked(z[:, off:off + k].detach().float(), mm)[0].double() if mm is not None else nl
        nl = torch.where(dead.unsqueeze(1), nl32, nl)
        out.append((nl, p, e, dead))
        off += k
    return out


def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, float('nan'), dtype=dtype, device=DEV) if dtype.is_floating_point else torch.full(shape, -7, dtype=dtype,
                                                                                                              device=DEV)


def _sample(name, z, mk, u=None, seed=0, epoch=None, step=0):
    from rl_games_b200 import ops
    K, sizes, hs = _layout(name)
    M = z.shape[0]
    nh = len(sizes)
    head = torch.cat([torch.randn(M, 1), z], 1).to(DEV)
    acts, nlp, vals = _nan(M, nh, dtype=torch.int64), _nan(M), _nan(M)
    ops.categorical_sample(head[:, 1:], 1 + K, K, head, 1 + K, None if mk is None else mk.to(torch.uint8).to(DEV),
                           None if u is None else u.to(DEV).contiguous(), seed, epoch, step, None, None, False, acts, nlp, vals,
                           None, None, None, None, M, head_sizes=hs)
    torch.cuda.synchronize()
    return acts.cpu(), nlp.cpu(), vals.cpu(), head[:, 0].cpu()


@pytest.mark.parametrize('masked', [False, True])
@pytest.mark.parametrize('name', list(LAYOUTS))
def test_wide_sample_on_a_tape_vs_fp64(name, masked):
    """actions equal the inverse-cdf rule in the kernel's summation order (tests/_cat_wide_ref.py) except where u lies within 1e-4 of a
    cdf value; neglogp the fp64 sum over heads; values copied"""
    K, sizes, hs = _layout(name)
    z, mk = _inputs(name, masked, seed=len(name) + masked)
    M, nh = z.shape[0], len(sizes)
    u = torch.rand(nh, M, generator=torch.Generator().manual_seed(9))
    acts, nlp, vals, v_ref = _sample(name, z, mk, u)
    torch.testing.assert_close(vals, v_ref, rtol=0, atol=0)
    heads = _heads64(z, mk, sizes)
    a_ref, near = [], []
    off = 0
    for j, (nl, p, e, dead) in enumerate(heads):
        zz = z[:, off:off + sizes[j]].double()
        if mk is not None:
            zz = torch.where(mk[:, off:off + sizes[j]], zz, torch.tensor(-1e8, dtype=torch.float64))
        lse32 = torch.logsumexp(zz, 1).float().double()                      # the kernel's lse, to within an ulp of fp32
        p32 = torch.exp(zz - lse32.unsqueeze(1)).float().numpy()
        a, dist = W.wide_inverse_cdf(p32, u[j].numpy())
        a_ref.append(torch.from_numpy(a))
        near.append(torch.from_numpy(dist < 1e-4))
        off += sizes[j]
    a_ref, near = torch.stack(a_ref, 1), torch.stack(near, 1)
    ok = (acts == a_ref) | near
    assert ok.all(), (acts[~ok], a_ref[~ok])
    assert ((acts >= 0) & (acts < torch.tensor(sizes))).all()
    if mk is not None:                                                      # a legal action wherever the head has one
        off = 0
        for j, k in enumerate(sizes):
            legal = mk[:, off:off + k].gather(1, acts[:, j:j + 1]).squeeze(1)
            assert (legal | ~mk[:, off:off + k].any(1)).all()
            off += k
    same = (acts == a_ref).all(1)
    assert same.float().mean() > 0.9
    nlp_ref = sum(-nl.gather(1, a_ref[:, j:j + 1]).squeeze(1) for j, (nl, _, _, _) in enumerate(heads))
    torch.testing.assert_close(nlp[same].double(), nlp_ref[same], rtol=2e-5, atol=2e-4)


@pytest.mark.parametrize('name', ['K362', 'h9', 'h1792'])
def test_wide_sample_philox_draws_bit_exact(name):
    """without a tape, each head draws the Philox uniform of tests/_cat_wide_ref.py: feeding those uniforms as a tape gives the same
    actions and neglogp bit for bit (a different uniform would move the actions of most rows)"""
    K, sizes, hs = _layout(name)
    z, mk = _inputs(name, True, seed=5)
    M = z.shape[0]
    ep = torch.tensor([3], dtype=torch.int64, device=DEV)
    a1, n1, _, _ = _sample(name, z, mk, None, seed=0xBADC0DE, epoch=ep, step=7)
    u = torch.from_numpy(W.categorical_uniforms_wide(0xBADC0DE, M, len(sizes), 3, 7)).float()
    a2, n2, _, _ = _sample(name, z, mk, u)
    assert torch.equal(a1, a2) and torch.equal(n1, n2)
    a3, _, _, _ = _sample(name, z, mk, None, seed=0xBADC0DE, epoch=ep, step=8)
    assert (a3 != a1).any()


def _loss(name, z, mk, acts, value, old_nlp, adv, old_v, ret, rmask, cfg, d_ld_pad=3):
    from rl_games_b200 import ops
    K, sizes, hs = _layout(name)
    M = z.shape[0]
    d = lambda t: None if t is None else t.to(DEV).contiguous()          # noqa: E731
    dl = _nan(M, K + d_ld_pad)
    dv = _nan(M, 1)
    part = _nan(ops.categorical_loss_partial_rows(M, K, hs), 8, dtype=torch.float64)
    inv = None if rmask is None else torch.tensor([1.0 / float(rmask.sum())], device=DEV)
    nb = ops.categorical_loss(d(z), K, K, d(value), 1, d(acts), None if mk is None else d(mk.to(torch.uint8)), d(old_v), d(ret), d(old_nlp),
                              d(adv), d(rmask), M, 0, M, cfg, inv, dl, K + d_ld_pad, dv, 1, part, head_sizes=hs)
    torch.cuda.synchronize()
    return nb, part.cpu(), dl[:, :K].cpu(), dv.cpu()


def _loss_case(name, masked, seed):
    K, sizes, _ = _layout(name)
    z, mk = _inputs(name, masked, seed)
    M = z.shape[0]
    g = torch.Generator().manual_seed(seed + 100)
    heads = _heads64(z, mk, sizes)
    acts = torch.stack([DO.sample_inverse_cdf(p.float(), torch.rand(M, generator=g)) for _, p, _, _ in heads], 1)
    nlp = sum(-nl.gather(1, acts[:, j:j + 1]).squeeze(1) for j, (nl, _, _, _) in enumerate(heads))
    old_nlp = (nlp + torch.randn(M, generator=g, dtype=torch.float64) * 0.05).float()
    adv, old_v, ret, value = (torch.randn(M, generator=g) for _ in range(4))
    rmask = (torch.rand(M, generator=g) < 0.8).float() if masked else None
    return z, mk, acts, value, old_nlp, adv, old_v, ret, rmask


@pytest.mark.parametrize('masked', [False, True])
@pytest.mark.parametrize('name', list(LAYOUTS))
def test_wide_loss_and_gradients_vs_fp64(name, masked):
    """loss pieces (partial rows, one per row), d(loss)/d(logits) for every head and d(loss)/d(value) against fp64 autograd"""
    from rl_games_b200 import ops
    K, sizes, _ = _layout(name)
    z, mk, acts, value, old_nlp, adv, old_v, ret, rmask = _loss_case(name, masked, seed=11 + masked)
    M = z.shape[0]
    cfg = ops.CatLossCfg(0.2, 1.5, 0.02, 1, 0, 1)
    nb, part, dl, dv = _loss(name, z, mk, acts, value, old_nlp, adv, old_v, ret, rmask, cfg)
    assert nb == M and torch.isfinite(part).all() and torch.isfinite(dl).all()
    z64 = z.double().requires_grad_(True)
    v64 = value.double().requires_grad_(True)
    heads = _heads64(z64, mk, sizes)
    nlp = sum(-nl.gather(1, acts[:, j:j + 1]).squeeze(1) for j, (nl, _, _, _) in enumerate(heads))
    ent = sum(e for _, _, e, _ in heads)
    a = actor_loss(old_nlp.double(), nlp, adv.double(), True, 0.2)
    c = critic_loss(old_v.double(), v64, 0.2, ret.double(), True)
    w = torch.full((M,), 1.0 / M, dtype=torch.float64) if rmask is None else rmask.double() / rmask.sum()
    la, lc, le = (a * w).sum(), (c * w).sum(), (ent * w).sum()
    (la + 0.5 * 1.5 * lc - 0.02 * le).backward()
    kl = (0.5 * (old_nlp.double() - nlp.detach()) ** 2 * w).sum()
    got = part[:, :4].sum(0)
    want = torch.stack([la, lc, le, kl]).detach()
    torch.testing.assert_close(got, want, rtol=2e-4, atol=1e-5 * float(want.abs().max()))
    torch.testing.assert_close(part[:, 4].sum(), torch.tensor(float(M if rmask is None else rmask.sum()), dtype=torch.float64))
    gz = z64.grad
    torch.testing.assert_close(dl.double(), gz, rtol=2e-3, atol=2e-4 * float(gz.abs().max()))
    torch.testing.assert_close(dv.squeeze(1).double(), v64.grad, rtol=1e-4, atol=1e-8)
    if mk is not None:
        assert (dl[~mk] == 0).all()


@pytest.mark.parametrize('name', ['K4672', 'h64', 'h1792'])
def test_wide_kernels_repeat_bit_for_bit(name):
    from rl_games_b200 import ops
    z, mk, acts, value, old_nlp, adv, old_v, ret, rmask = _loss_case(name, True, seed=3)
    cfg = ops.CatLossCfg(0.2, 1.0, 0.01, 1, 0, 1)
    r1 = _loss(name, z, mk, acts, value, old_nlp, adv, old_v, ret, rmask, cfg)
    r2 = _loss(name, z, mk, acts, value, old_nlp, adv, old_v, ret, rmask, cfg)
    assert all(torch.equal(x, y) for x, y in zip(r1[1:], r2[1:]))
    ep = torch.zeros(1, dtype=torch.int64, device=DEV)
    s1, s2 = _sample(name, z, mk, None, 1, ep, 2), _sample(name, z, mk, None, 1, ep, 2)
    assert torch.equal(s1[0], s2[0]) and torch.equal(s1[1], s2[1])


def _argmax(z, mk, sizes):
    from rl_games_b200 import ops
    M, K = z.shape
    out = _nan(M, len(sizes), dtype=torch.int64)
    ops.categorical_argmax(z.to(DEV), K, K, None if mk is None else mk.to(torch.uint8).to(DEV), out, M,
                           head_sizes=None if len(sizes) == 1 else sizes)
    torch.cuda.synchronize()
    return out.cpu()


def _argmax_ref(z, mk, sizes):
    out, off = [], 0
    for k in sizes:
        zz = z[:, off:off + k]
        if mk is not None:
            zz = torch.where(mk[:, off:off + k], zz, torch.tensor(float('-inf')))
        a = torch.argmax(zz, 1)
        if mk is not None:
            a = torch.where(mk[:, off:off + k].any(1), a, torch.zeros_like(a))
        out.append(a)
        off += k
    return torch.stack(out, 1)


def test_wide_argmax_exhaustive_head_sizes_65_to_256():
    """every head size 65-256, alone and as the second of two heads, with ties (small integer logits), NaN and masked / all-masked rows;
    against torch.argmax (ties: lowest index; NaN: the first NaN) over the allowed logits, all-masked heads play 0"""
    g = torch.Generator().manual_seed(1)
    for k in range(65, 257):
        for sizes in ([k], [3, k]):
            K, M = sum(sizes), 96
            z = torch.randint(-3, 4, (M, K), generator=g).float()
            z[5::7, torch.randint(0, K, (1,), generator=g)] = float('nan')
            mk = torch.rand(M, K, generator=g) < 0.5
            mk[3::4] = False
            mk[0::4] = True
            for m in (None, mk):
                got = _argmax(z, m, sizes)
                ref = _argmax_ref(z, m, sizes)
                assert torch.equal(got, ref), (k, sizes, m is None)


@pytest.mark.parametrize('name', list(LAYOUTS))
def test_wide_argmax_layouts(name):
    K, sizes, _ = _layout(name)
    z, mk = _inputs(name, True, seed=8)
    z[1::5] = torch.round(z[1::5])                                      # ties
    for m in (None, mk):
        assert torch.equal(_argmax(z, m, sizes), _argmax_ref(z, m, sizes))


# --------------------------------------------------------------------------------------------------------- agent and player
WIDE_GOLDENS = ['agent_discrete_wide362.pt', 'agent_multidiscrete_wide.pt']


@pytest.mark.parametrize('name', WIDE_GOLDENS)
def test_wide_agent_matches_reference_golden(name):
    import test_discrete_gpu as TD
    TD.test_discrete_agent_matches_reference_golden(name)


def _gpu_agent(g, over=None):
    import test_discrete_gpu as TD
    from rl_games_b200.runner import Runner
    env = TD.DiscreteTapeEnvGPU(g)
    cfgk = g['config']
    config = {k: v for k, v in cfgk.items() if k not in ('device', 'torch_compile')}
    config.update({'device': DEV, 'env_info': env.get_env_info(), 'vec_env': env, 'reward_shaper': {'scale_value': 0.1},
                   'train_dir': '/tmp/b200_wide_runs', 'lr_schedule': cfgk.get('lr_schedule', None)})
    config.update(over or {})
    multi = isinstance(g['K'], (list, tuple))
    network = {'name': 'actor_critic', 'separate': g['separate'], 'space': {'multi_discrete' if multi else 'discrete': None},
               'mlp': {'units': g['units'], 'activation': 'relu', 'initializer': {'name': 'default'}}}
    r = Runner()
    r.load({'params': {'seed': 1, 'algo': {'name': 'a2c_discrete'}, 'model': {'name': 'multi_discrete_a2c' if multi else 'discrete_a2c'},
                       'network': network, 'config': config}})
    r.params['config']['vec_env'] = env
    agent = r.algo_factory.create(r.algo_name, base_name='wide', params=r.params)
    agent.model.load_state_dict({k: v.to(DEV) for k, v in g['init_state'].items()}, strict=False)
    agent.init_tensors()
    agent.obs = agent.env_reset()
    return agent, network, config


@pytest.mark.parametrize('name', WIDE_GOLDENS)
def test_wide_agent_mixed_precision_stays_near_the_golden(name):
    """bf16 tensor-core layers, fp32 categorical kernels: losses and entropies near the reference's fp32 run, weights after the epochs'
    Adam steps within 5e-2 of their max-norm (Adam turns bf16 noise on near-zero gradients into steps of up to the learning rate)"""
    g = torch.load(os.path.join(HERE, 'golden', name), weights_only=False)
    agent, _, _ = _gpu_agent(g, {'mixed_precision': True})
    for ep, ref in enumerate(g['epochs_out']):
        agent.epoch_num += 1
        res = agent.train_epoch(u=g['u'][ep].to(DEV))
        torch.testing.assert_close(torch.stack(res[6]).cpu(), ref['entropies'], rtol=2e-2, atol=1e-3)
        torch.testing.assert_close(torch.stack(res[5]).cpu(), ref['c_losses'], rtol=5e-2, atol=1e-3)
    sd = agent.model.state_dict()
    for k in g['param_order']:
        r = g['epochs_out'][-1]['state'][k]
        torch.testing.assert_close(sd[k].cpu(), r, rtol=0, atol=5e-2 * float(r.abs().max()) + 1e-6, msg=lambda m: k + ': ' + m)


@pytest.mark.parametrize('use_graph', [False, True])
@pytest.mark.parametrize('name', WIDE_GOLDENS)
def test_wide_player_plays_the_reference_rule_on_a_trained_checkpoint(name, use_graph, tmp_path):
    """train the golden run's two epochs, save, restore into PpoPlayerDiscrete: deterministic actions are the per-head argmax of the
    masked logits of the oracle network (pinned to the reference) on the checkpoint's weights; sampled actions on a uniform tape
    follow the inverse-cdf rule; eager and CUDA-graph replay"""
    from rl_games_b200.players import PpoPlayerDiscrete
    g = torch.load(os.path.join(HERE, 'golden', name), weights_only=False)
    agent, network, config = _gpu_agent(g)
    for ep in range(len(g['epochs_out'])):
        agent.epoch_num += 1
        agent.train_epoch(u=g['u'][ep].to(DEV))
    fn = str(tmp_path / 'wide')
    agent.save(fn)
    multi = isinstance(g['K'], (list, tuple))
    sizes = list(g['K']) if multi else [g['K']]
    env_info = agent.env_info
    pconfig = {k: v for k, v in config.items() if k not in ('vec_env',)}
    pconfig.update({'env_info': env_info, 'player': {'use_vecenv': False}, 'b200_cuda_graph': use_graph})
    player = PpoPlayerDiscrete({'seed': 1, 'algo': {'name': 'a2c_discrete'}, 'model': {'name': 'multi_discrete_a2c' if multi else 'discrete_a2c'},
                                'network': network, 'config': pconfig})
    player.restore(fn + '.pth')
    player.get_batch_size(g['obs_tape'][0], 1)
    sd = {k: v.cpu() for k, v in player.model.state_dict().items() if k.startswith('a2c_network')}
    model = DO.DiscreteOracleModel(sd, g['D'], g['units'], g['K'], g['separate'])
    for step in range(3):
        obs = g['obs_tape'][step]
        mk = g['mask_tape'][step]
        with torch.no_grad():
            a_out = model._mlp(obs, 'actor_mlp')
            names = [f'a2c_network.logits.{j}' for j in range(len(sizes))] if multi else ['a2c_network.logits']
            logits = torch.cat([torch.nn.functional.linear(a_out, model.p[n + '.weight'], model.p[n + '.bias']) for n in names], 1)
        ref = _argmax_ref(logits.detach().float(), mk, sizes)
        got = player.get_masked_action(obs.to(DEV), mk.to(DEV), is_deterministic=True).cpu().reshape(ref.shape[0], -1)
        top2 = []
        off = 0
        for k in sizes:                       # rows whose top-two margin is wide enough for fp32 vs the oracle's arithmetic
            zz = torch.where(mk[:, off:off + k], logits.detach()[:, off:off + k], torch.tensor(-1e8))
            t = zz.topk(min(2, k), 1).values
            top2.append((t[:, 0] - t[:, -1] > 1e-4) | (k == 1))
            off += k
        clear = torch.stack(top2, 1)
        assert torch.equal(got[clear], ref[clear])
