"""State-dependent sigma heads (fixed_sigma: False) on the GPU: the fp32 head kernels (ppo_head_loss_sd / policy_head_sample_sd)
against autograd of a torch restatement, the agent against the reference's golden runs (eager and CUDA graph), and the layer-wise
tensor-core path against the fp32 agent."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from oracle import ppo_oracle as O  # noqa: E402
from test_agent_gpu import DEV, TapeEnvGPU, make_agent  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')

@pytest.fixture(autouse=True)
def _fp32_matmuls():
    """the torch restatements are fp32 references: keep their GEMMs off TF32, which constructing the reference's Runner (other tests of
    the same process do) switches on for the whole process"""
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = tf32


_PARAMS = [('exp', 0.0, None), ('exp', 0.1, (-1.0, 0.4)), ('softplus', 0.2, None), ('linear', 0.0, None)]


def _loss_cfg(ppo=1, smooth=1, clip_value=1, bounds=0.001, bound_type=1):
    from rl_games_b200 import ops
    return ops.LossCfg(0.2, 2.0, bounds, int(bounds > 0), bound_type, clip_value, smooth, ppo)


@pytest.mark.parametrize('A', [3, 8, 15])
@pytest.mark.parametrize('param,min_sigma,bounds', _PARAMS)
def test_head_loss_kernel_matches_autograd(A, param, min_sigma, bounds):
    """M = 1000 (a partial last block), chunked arena rows, masked rows, entropy bonus, bound loss"""
    import _torch_ops_sd as S
    from rl_games_b200 import ops
    g = torch.Generator().manual_seed(A)
    M, Hl, epm, N = 1000, 64, 250, 400
    HR = 1 + 2 * A
    a_last = torch.nn.functional.elu(torch.randn(M, Hl, generator=g)).to(DEV)
    W = (torch.randn(HR, Hl, generator=g) * 0.1).to(DEV)
    b = (torch.randn(HR, generator=g) * 0.3).to(DEV)
    rows = 4 * N            # arena: 4 chunks of epm rows, stride N
    f = lambda *s: torch.randn(*s, generator=g).to(DEV)     # noqa: E731
    actions, old_mu = f(rows, A), f(rows, A)
    old_sigma = (torch.rand(rows, A, generator=g) + 0.3).to(DEV)
    old_v, ret, adv = f(rows), f(rows), f(rows)
    old_nlp = (torch.randn(rows, generator=g) * 0.3 + 3.0).to(DEV)
    mask = (torch.rand(rows, generator=g) < 0.8).float().to(DEV)
    m_ = torch.arange(M)
    ridx = ((m_ // epm) * N + m_ % epm).to(DEV)
    inv = (1.0 / mask[ridx].sum()).reshape(1)
    ent = torch.tensor([0.01], device=DEV)
    cfg, scfg = _loss_cfg(), ops.sigma_cfg(param, min_sigma, bounds)
    # reference: autograd of the torch restatement
    al = a_last.clone().requires_grad_(True)
    head = al @ W.t() + b
    head.retain_grad()
    value, mu = head[:, :1], head[:, 1:A + 1]
    sg, ls = S.apply_sigma(head[:, A + 1:], param, min_sigma, bounds)
    nlp = O.neglogp_fn(actions[ridx], mu, sg, ls)
    w = mask[ridx] * inv
    a = O.actor_loss(old_nlp[ridx], nlp, adv[ridx], True, 0.2, smooth=True)
    c = O.critic_loss(old_v[ridx].unsqueeze(1), value, 0.2, ret[ridx].unsqueeze(1), True).squeeze(1)
    e = (0.5 + 0.9189385332046727 + torch.log(sg)).sum(-1)
    bl = O.bound_loss(mu, 0.001)
    loss = (a * w).sum() + (c * w).sum() - 0.01 * (e * w).sum() + 0.001 * (bl * w).sum()
    loss.backward()
    d_alast_ref = al.grad * torch.where(a_last > 0, torch.ones_like(a_last), a_last + 1.0)
    # kernel, twice: identical bytes
    outs = []
    for _ in range(2):
        omu, osg = old_mu.clone(), old_sigma.clone()
        d_head, d_alast = torch.zeros(M, HR, device=DEV), torch.zeros(M, Hl, device=DEV)
        partials = torch.zeros(64, ops.loss_partial_stride(), dtype=torch.float64, device=DEV)
        nb = ops.ppo_head_loss_sd(a_last, W, b, scfg, ent, actions, omu, osg, old_v, ret, old_nlp, adv, mask, epm, N, M, A, cfg, inv,
                                  d_head, d_alast, 1, partials)
        stats, d_ls, kl = torch.zeros(16, device=DEV), torch.full((A,), 7.0, device=DEV), torch.zeros(1, device=DEV)
        ops.ppo_loss_finalize(partials, nb, A, torch.zeros(1, device=DEV), stats, d_ls, kl)
        torch.cuda.synchronize()
        outs.append((omu, osg, d_head, d_alast, stats, d_ls))
    for x, y in zip(*outs):
        assert torch.equal(x, y)
    omu, osg, d_head, d_alast, stats, d_ls = outs[0]
    torch.testing.assert_close(d_head, head.grad, rtol=1e-4, atol=1e-7)
    torch.testing.assert_close(d_alast, d_alast_ref, rtol=1e-4, atol=1e-7)
    torch.testing.assert_close(omu[ridx], mu.detach(), rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(osg[ridx], sg.detach(), rtol=1e-5, atol=1e-6)
    assert torch.equal(d_ls, torch.zeros(A, device=DEV))        # the dead fixed-sigma block gets exactly 0
    torch.testing.assert_close(stats[0], (a * w).sum().detach(), rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(stats[2], (e * w).sum().detach(), rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize('A', [3, 15])
@pytest.mark.parametrize('param,min_sigma,bounds', _PARAMS)
def test_rollout_head_kernel_matches_torch(A, param, min_sigma, bounds):
    import _torch_ops_sd as S
    from rl_games_b200 import ops
    g = torch.Generator().manual_seed(40 + A)
    N, Hl, HR = 1000, 32, 1 + 2 * A
    a_last = torch.randn(N, Hl, generator=g).to(DEV)
    W, b = (torch.randn(HR, Hl, generator=g) * 0.2).to(DEV), (torch.randn(HR, generator=g) * 0.3).to(DEV)
    noise = torch.randn(N, A, generator=g).to(DEV)
    f = lambda *s: torch.zeros(*s, device=DEV)      # noqa: E731
    acts, mus, sgs, nlp, vals = f(N, A), f(N, A), f(N, A), f(N), f(N)
    ops.policy_head_sample_sd(a_last, W, b, ops.sigma_cfg(param, min_sigma, bounds), None, None, False, noise, 0, None, 0, acts, mus, sgs,
                              nlp, vals, None, False, None, None, None, None, None, None, N, A)
    head = a_last @ W.t() + b
    sg, ls = S.apply_sigma(head[:, A + 1:], param, min_sigma, bounds)
    mu = head[:, 1:A + 1]
    torch.testing.assert_close(vals, head[:, 0], rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(mus, mu, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(sgs, sg, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(acts, mu + sg * noise, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(nlp, O.neglogp_fn(mu + sg * noise, mu, sg, ls), rtol=1e-5, atol=1e-4)


@pytest.mark.parametrize('param,min_sigma,bounds', _PARAMS)
def test_rollout_and_update_heads_share_arithmetic(param, min_sigma, bounds):
    """The loss kernel re-evaluates exactly what the rollout kernel sampled from the same activations: mu, sigma and neglogp are
    bit-identical, so the first update's probability ratio is exactly 1 (no clipped row)"""
    from rl_games_b200 import ops
    A, N, Hl, HR = 8, 1000, 64, 17
    g = torch.Generator().manual_seed(77)
    a_last = torch.nn.functional.elu(torch.randn(N, Hl, generator=g)).to(DEV)
    W, b = (torch.randn(HR, Hl, generator=g) * 0.2).to(DEV), (torch.randn(HR, generator=g) * 0.3).to(DEV)
    scfg = ops.sigma_cfg(param, min_sigma, bounds)
    f = lambda *s: torch.zeros(*s, device=DEV)      # noqa: E731
    acts, mus, sgs, nlp, vals = f(N, A), f(N, A), f(N, A), f(N), f(N)
    ops.policy_head_sample_sd(a_last, W, b, scfg, None, None, False, None, 123, None, 0, acts, mus, sgs, nlp, vals, None, False, None,
                              None, None, None, None, None, N, A)
    omu, osg, nlp_out = mus.clone(), sgs.clone(), f(N)
    adv, ret = torch.randn(N, generator=g).to(DEV), torch.randn(N, generator=g).to(DEV)
    partials = torch.zeros(64, ops.loss_partial_stride(), dtype=torch.float64, device=DEV)
    nb = ops.ppo_head_loss_sd(a_last, W, b, scfg, torch.tensor([0.01], device=DEV), acts, omu, osg, vals, ret, nlp, adv, None, N, N, N, A,
                              _loss_cfg(), None, f(N, HR), f(N, Hl), 1, partials, neglogp_out=nlp_out)
    stats = f(16)
    ops.ppo_loss_finalize(partials, nb, A, f(1), stats, f(A), None)
    torch.cuda.synchronize()
    assert torch.equal(nlp_out, nlp)
    assert torch.equal(omu, mus) and torch.equal(osg, sgs)
    assert float(stats[6]) == 0.0                  # clip fraction: no row left the trust region


def _golden_sd(name, graph, extra=None):
    g = torch.load(os.path.join(GOLDEN, name), weights_only=False)
    cfgk = g['config']
    over = {k: cfgk[k] for k in ('clip_value', 'use_smooth_clamp', 'bound_loss_type', 'bounds_loss_coef', 'entropy_coef', 'truncate_grads',
                                 'value_bootstrap', 'mini_epochs', 'lr_schedule', 'critic_coef', 'learning_rate', 'kl_threshold',
                                 'normalize_input', 'normalize_value', 'normalize_advantage', 'clip_actions', 'e_clip', 'tau', 'gamma')
            if k in cfgk}
    over.setdefault('lr_schedule', None)
    over['b200_cuda_graph'] = graph
    over.update(extra or {})
    env = TapeEnvGPU(g['obs_tape'], g['done_tape'], g['timeout_tape'], g['A'], g['autoreset'], g.get('act_bounds', (-1.0, 1.0)))
    agent = make_agent(over, g['N'], g['H'], g['D'], g['A'], g['units'], g['mb'], env, g['init_state'], space_over=g['space_over'])
    return g, agent


@pytest.mark.parametrize('name', ['agent_sdsigma.pt', 'agent_sdsigma_softplus.pt', 'agent_fixedsigma_softplus.pt', 'agent_fixedsigma_bounds.pt'])
@pytest.mark.parametrize('graph', [False, True])
def test_state_dependent_agent_matches_reference_golden(name, graph):
    """agent_fixedsigma_*.pt: a fixed sigma in softplus / clamped exp, mapped outside the kernels with its gradient chain"""
    g, agent = _golden_sd(name, graph)
    assert not agent.use_tc and not agent.gemm_tc
    fl = O.swap_and_flatten01
    for ep, ref in enumerate(g['epochs_out']):
        agent.epoch_num += 1
        agent.train_epoch(noise=g['noise'][ep].to(DEV))
        ds = ref['dataset']
        assert torch.equal(agent.dones_buf.cpu(), ref['mb_dones'])
        torch.testing.assert_close(agent.values.cpu().unsqueeze(2), ref['mb_values'], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(fl(agent.neglogpacs).cpu(), ds['old_logp_actions'], rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(fl(agent.actions).cpu(), ds['actions'], rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(fl(agent.advs_n).cpu(), ds['advantages'], rtol=2e-4, atol=2e-5)
        torch.testing.assert_close(fl(agent.sigmas).cpu(), ds['sigma'], rtol=1e-4, atol=1e-6)
        st, nmb = agent.last_stats, agent.num_minibatches
        for col, key in ((0, 'a_losses'), (1, 'c_losses'), (2, 'entropies')):
            torch.testing.assert_close(st[:, col], ref[key], rtol=2e-3, atol=2e-6, msg=lambda m: key + ': ' + m)
        torch.testing.assert_close(torch.stack([st[e * nmb:(e + 1) * nmb, 4].mean() for e in range(agent.mini_epochs_num)]), ref['kls'],
                                   rtol=2e-3, atol=2e-6)
        assert agent.last_lr == pytest.approx(ref['last_lr'], rel=1e-12)
        sd = agent.model.state_dict()
        for k in g['param_order']:
            torch.testing.assert_close(sd[k].cpu(), ref['state'][k], rtol=1e-3, atol=2e-5, msg=lambda m: k + ': ' + m)
        if not g['space_over'].get('fixed_sigma', True):
            assert torch.equal(agent.model.sigma.cpu(), torch.zeros(g['A']))


def test_layerwise_tensor_core_state_dependent_agent_tracks_fp32_agent():
    """mixed_precision: True with [512,256,128]: every GEMM on the tensor cores (gemm_tc.cu), the same fp32 head kernels; against the
    fp32 agent on the same tapes / weights / noise, bf16 tolerance class (as test_agent_gpu's layer-wise tests)"""
    N, H, D, A, mb, units = 256, 8, 44, 8, 1024, [512, 256, 128]
    space_over = {'fixed_sigma': False, 'sigma_parametrization': 'softplus', 'min_sigma': 0.2,
                  'sigma_init': {'name': 'const_initializer', 'val': -1.05}}
    obs_tape, done_tape, tout_tape = O.make_tapes(H + 1, N, D, seed=52, p_done=0.08)
    g = torch.Generator().manual_seed(17)
    noise = torch.randn(H, N, A, generator=g).to(DEV)
    agents, params = [], None
    for mp in (False, True):
        a = make_agent({'mixed_precision': mp, 'mini_epochs': 2, 'b200_cuda_graph': False, 'entropy_coef': 0.01}, N, H, D, A, units, mb,
                       TapeEnvGPU(obs_tape, done_tape, tout_tape, A), params or {}, space_over=space_over)
        if params is None:
            params = {k: v.cpu().clone() for k, v in a.model.state_dict().items()}
        assert a.gemm_tc == mp and not a.use_tc
        a.epoch_num += 1
        a.train_epoch(noise=noise)
        agents.append(a)
    f, t = agents
    torch.testing.assert_close(t.values, f.values, rtol=0, atol=6e-2)
    torch.testing.assert_close(t.mus, f.mus, rtol=0, atol=6e-2)
    torch.testing.assert_close(t.sigmas, f.sigmas, rtol=0, atol=2e-2)
    sf, st = f.last_stats, t.last_stats
    torch.testing.assert_close(st[:, 0], sf[:, 0], rtol=0.1, atol=2e-2)
    torch.testing.assert_close(st[:, 1], sf[:, 1], rtol=0.1, atol=2e-2)
    torch.testing.assert_close(st[:, 2], sf[:, 2], rtol=1e-2, atol=1e-3)
    sdf, sdt = f.model.state_dict(), t.model.state_dict()
    for k in params:
        if k.endswith('weight'):
            du_f = (sdf[k].cpu() - params[k]).flatten()
            du_t = (sdt[k].cpu() - params[k]).flatten()
            cos = float(du_f @ du_t / (du_f.norm() * du_t.norm() + 1e-20))
            assert cos > 0.8, (k, cos)
