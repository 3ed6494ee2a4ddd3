"""SAC on the GPU: every csrc/sac.cu kernel against torch autograd of the reference's maths (sac_helper.py SquashedNormal,
network_builder.py DiagGaussianActor, sac_agent.py update_critic / update_actor_and_alpha, experience.py VectorizedReplayBuffer), and the
whole agent against the reference's golden runs, eager and CUDA-graph."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _sac_golden as SG  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ACTS = [1, 6, 8, 17]


def _box(A, g):
    low = -1.0 - torch.rand(A, generator=g) * 2
    high = low + 0.5 + torch.rand(A, generator=g) * 3
    scale, bias = (high - low) / 2, (high + low) / 2
    lss = float(torch.log(scale.clamp_min(1e-8)).sum())
    return [t.to(DEV) for t in (scale, bias, low, high)], lss


def _ref_squash(head, eps, A, bounds, box, lss):
    """DiagGaussianActor.forward + SquashedNormal.rsample + _env_log_prob + rescale_actions, in torch"""
    mu, ls = head.chunk(2, dim=-1)
    lo, hi = bounds
    ls = torch.tanh(ls)
    ls = lo + 0.5 * (hi - lo) * (ls + 1)
    std = ls.exp()
    x = mu + eps * std
    y = torch.tanh(x)
    nlp = -((x - mu) ** 2) / (2 * std ** 2) - std.log() - math.log(math.sqrt(2 * math.pi))
    jac = 2.0 * (math.log(2.0) - x - torch.nn.functional.softplus(-2.0 * x))
    logp = (nlp - jac).sum(-1) - lss
    sc, bi, low, high = box
    act = (y * sc + bi).clamp(low, high)
    return act, logp


@pytest.mark.parametrize('A', ACTS)
@pytest.mark.parametrize('M', [1, 255, 1000])
def test_squash_forward_and_backward_match_autograd(A, M):
    g = torch.Generator().manual_seed(A * 1000 + M)
    head = (torch.randn(M, 2 * A, generator=g) * 1.5).to(DEV)
    eps = torch.randn(M, A, generator=g).to(DEV)
    box, lss = _box(A, g)
    bounds = (-5.0, 2.0)
    from rl_games_b200 import ops
    ld = A + 3
    dst = torch.full((M, ld), float('nan'), device=DEV)            # unzeroed scratch: only the action columns may be written
    logp = torch.full((M,), float('nan'), device=DEV)
    eps_out = torch.full((M, A), float('nan'), device=DEV)
    ops.sac_squash_fwd(head, M, A, bounds, eps, 0, None, 1, box, lss, dst=dst[:, 3:], dst_ld=ld, eps_out=eps_out, logp=logp)
    h64 = head.double().requires_grad_(True)
    act_r, logp_r = _ref_squash(h64, eps.double(), A, bounds, [t.double() for t in box], lss)
    torch.testing.assert_close(dst[:, 3:].double(), act_r, rtol=1e-5, atol=1e-5)
    assert torch.isnan(dst[:, :3]).all()
    torch.testing.assert_close(logp.double(), logp_r, rtol=1e-4, atol=1e-4)
    assert torch.equal(eps_out, eps)
    # backward: L = mean(c * logp) + sum(w * act) with w the critics' action-column gradients
    la = torch.tensor([math.log(0.3)], device=DEV)
    w1, w2 = torch.randn(M, ld, generator=g).to(DEV), torch.randn(M, ld, generator=g).to(DEV)
    d_head = torch.full((M, 2 * A), float('nan'), device=DEV)
    ops.sac_squash_bwd(head, eps, M, A, bounds, box, w1[:, 3:], w2[:, 3:], ld, la, 0.01, d_head)
    c = max(0.3, 0.01)
    L = (c * logp_r).mean() + ((w1[:, 3:] + w2[:, 3:]).double() * act_r).sum()
    L.backward()
    torch.testing.assert_close(d_head.double(), h64.grad, rtol=2e-4, atol=2e-5)


@pytest.mark.parametrize('B', [1, 257, 4096])
def test_critic_and_actor_loss_match_autograd(B):
    from rl_games_b200 import ops
    g = torch.Generator().manual_seed(B)
    q1, q2, q1t, q2t, lp = [torch.randn(B, generator=g).to(DEV) for _ in range(5)]
    q2[::7] = q1[::7]                                           # ties: torch.min's backward splits them in halves
    r = torch.randn(B, generator=g).to(DEV)
    nd = (torch.rand(B, generator=g) > 0.3).float().to(DEV)
    la = torch.tensor([math.log(0.4)], device=DEV)
    dq1, dq2, stats = [torch.full((B,), float('nan'), device=DEV) for _ in range(2)] + [torch.zeros(8, device=DEV)]
    ops.sac_critic_loss(q1, q2, q1t, q2t, lp, r, nd, la, 0.97, B, dq1, dq2, stats)
    a = 0.4
    Q1, Q2 = q1.double().requires_grad_(True), q2.double().requires_grad_(True)
    tq = r.double() + nd.double() * 0.97 * (torch.min(q1t, q2t).double() - a * lp.double())
    l1, l2 = torch.nn.functional.mse_loss(Q1, tq), torch.nn.functional.mse_loss(Q2, tq)
    (0.5 * (l1 + l2)).backward()
    torch.testing.assert_close(stats[:3].double(), torch.stack([0.5 * (l1 + l2), l1, l2]).detach(), rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(dq1.double(), Q1.grad, rtol=1e-5, atol=1e-8)
    torch.testing.assert_close(dq2.double(), Q2.grad, rtol=1e-5, atol=1e-8)
    dla = torch.zeros(1, device=DEV)
    ops.sac_actor_loss(q1, q2, lp, la, 0.01, -3.0, True, B, dq1, dq2, dla, stats)
    Q1, Q2 = q1.double().requires_grad_(True), q2.double().requires_grad_(True)
    LA = la.double().requires_grad_(True)
    actor_loss = (max(a, 0.01) * lp.double() - torch.min(Q1, Q2)).mean()
    alpha_loss = (LA.exp() * (-lp.double() - (-3.0))).mean()
    (actor_loss + alpha_loss).backward()
    torch.testing.assert_close(dq1.double(), Q1.grad, rtol=1e-5, atol=1e-8)
    torch.testing.assert_close(dq2.double(), Q2.grad, rtol=1e-5, atol=1e-8)
    torch.testing.assert_close(dla.double(), LA.grad, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(stats[3].double(), actor_loss.detach(), rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(stats[4].double(), -lp.double().mean(), rtol=1e-5, atol=1e-6)


def _rb(cap, D, A):
    f = lambda *s: torch.full(s, float('nan'), device=DEV)      # noqa: E731
    return {'obs': f(cap, D), 'act': f(cap, A), 'rew': f(cap), 'next': f(cap, D), 'term': torch.full((cap,), 7, dtype=torch.uint8, device=DEV),
            'trunc': torch.full((cap,), 7, dtype=torch.uint8, device=DEV), 'state': torch.zeros(2, dtype=torch.int64, device=DEV)}


@pytest.mark.parametrize('N,next_step', [(5, False), (1037, True), (3000, False), (2500, True)])
def test_replay_insert_matches_the_reference_buffer(N, next_step):
    """experience.py VectorizedReplayBuffer.add of _store_transitions' rows, over several steps so that the ring wraps"""
    from rl_games_b200 import ops
    g = torch.Generator().manual_seed(N)
    D, A, cap = 7, 3, int(N * 2.5)
    rb = _rb(cap, D, A)
    ref = {k: torch.zeros(cap, *s) for k, s in (('obs', (D,)), ('act', (A,)), ('rew', ()), ('next', (D,)), ('term', ()), ('trunc', ()))}
    idx, full = 0, False
    prev = torch.zeros(N, dtype=torch.uint8, device=DEV)
    prev_ref = torch.zeros(N, dtype=torch.bool)
    ep = torch.zeros(2 * N, device=DEV)
    meter = torch.zeros(3, dtype=torch.float64, device=DEV)
    slot = torch.full((N,), -5, dtype=torch.int32, device=DEV)
    ts, tr = torch.full((N,), 9, dtype=torch.uint8, device=DEV), torch.full((N,), 9, dtype=torch.uint8, device=DEV)
    for step in range(5):
        obs, nxt, fin = torch.randn(N, D, generator=g), torch.randn(N, D, generator=g), torch.randn(N, D, generator=g)
        act, rew = torch.randn(N, A, generator=g), torch.randn(N, generator=g)
        done = torch.rand(N, generator=g) < 0.3
        tout = done & (torch.rand(N, generator=g) < 0.5)
        ops.sac_replay_insert(obs.to(DEV), act.to(DEV), rew.to(DEV), nxt.to(DEV), None if next_step else fin.to(DEV), done.to(torch.uint8).to(DEV),
                              tout.to(torch.uint8).to(DEV), True, next_step, prev, rb, slot, ts, tr, ep, meter, 100)
        live = ~prev_ref if next_step else torch.ones(N, dtype=torch.bool)
        rows = live.nonzero().reshape(-1)
        nx = nxt.clone()
        if not next_step:
            nx[tout] = fin[tout]
        for r in rows.tolist():
            ref['obs'][idx], ref['act'][idx], ref['rew'][idx], ref['next'][idx] = obs[r], act[r], rew[r], nx[r]
            ref['term'][idx], ref['trunc'][idx] = float(done[r] and not tout[r]), float(tout[r])
            idx = (idx + 1) % cap
            full = full or idx == 0
        prev_ref = done.clone()
    st = rb['state'].cpu()
    assert int(st[0]) == idx and int(st[1]) == (cap if full else idx)
    n = int(st[1])
    for k in ('obs', 'act', 'rew', 'next'):
        assert torch.equal(rb[k][:n].cpu(), ref[k][:n]), k
    assert torch.equal(rb['term'][:n].cpu().float(), ref['term'][:n]) and torch.equal(rb['trunc'][:n].cpu().float(), ref['trunc'][:n])


def test_replay_sample_gathers_normalises_and_is_uniform():
    from rl_games_b200 import ops
    g = torch.Generator().manual_seed(3)
    D, A, cap, fill, B = 6, 4, 5000, 3001, 4099
    rb = _rb(cap, D, A)
    rb['obs'][:fill] = torch.randn(fill, D, generator=g).to(DEV) * 4
    rb['next'][:fill] = torch.randn(fill, D, generator=g).to(DEV) * 4
    rb['act'][:fill] = torch.randn(fill, A, generator=g).to(DEV)
    rb['rew'][:fill] = torch.randn(fill, generator=g).to(DEV)
    rb['term'][:fill] = (torch.rand(fill, generator=g) < 0.2).to(torch.uint8).to(DEV)
    rb['state'].copy_(torch.tensor([fill, fill]))
    mean, std = torch.randn(D, generator=g).to(DEV), (torch.rand(D, generator=g) + 0.5).to(DEV)
    xc, xp, xn = [torch.full((B, D + A), float('nan'), device=DEV) for _ in range(3)]
    rw, nd = torch.empty(B, device=DEV), torch.empty(B, device=DEV)
    tape = torch.randint(0, fill, (B,), generator=g).to(DEV)
    idx_out = torch.empty(B, dtype=torch.int64, device=DEV)
    ops.sac_replay_sample(rb, B, tape, 0, None, mean, std, xc, xp, xn, rw, nd, idx_out)
    assert torch.equal(idx_out, tape)
    nrm = lambda x: torch.clamp((x - mean) / std, -5, 5)      # noqa: E731
    assert torch.equal(xc[:, :D], nrm(rb['obs'][tape])) and torch.equal(xp[:, :D], xc[:, :D]) and torch.equal(xn[:, :D], nrm(rb['next'][tape]))
    assert torch.equal(xc[:, D:], rb['act'][tape]) and torch.equal(rw, rb['rew'][tape]) and torch.equal(nd, 1.0 - rb['term'][tape].float())
    # Philox path: deterministic per (seed, counter), in range, uniform over the fill
    ctr = torch.zeros(1, dtype=torch.int64, device=DEV)
    counts = torch.zeros(fill, dtype=torch.int64)
    outs = []
    for k in range(40):
        ops.sac_replay_sample(rb, B, None, 99, ctr, None, None, xc, xp, xn, rw, nd, idx_out)
        outs.append(idx_out.clone())
        ops.bump_u64(ctr)
        counts += torch.bincount(idx_out.cpu(), minlength=fill)
    ctr.zero_()
    ops.sac_replay_sample(rb, B, None, 99, ctr, None, None, xc, xp, xn, rw, nd, idx_out)
    assert torch.equal(idx_out, outs[0]) and not torch.equal(outs[0], outs[1])
    assert int(torch.cat(outs).min()) >= 0 and int(torch.cat(outs).max()) < fill
    expect = 40 * B / fill
    chi2 = float(((counts.double() - expect) ** 2 / expect).sum())
    assert abs(chi2 - (fill - 1)) < 6 * math.sqrt(2 * (fill - 1)), chi2


@pytest.mark.parametrize('A', ACTS)
def test_squash_philox_noise_is_standard_normal_and_deterministic(A):
    from rl_games_b200 import ops
    M = 20011
    box = [torch.ones(A, device=DEV), torch.zeros(A, device=DEV), -torch.ones(A, device=DEV), torch.ones(A, device=DEV)]
    head = torch.zeros(M, 2 * A, device=DEV)
    ctr = torch.tensor([5], dtype=torch.int64, device=DEV)
    e1, e2, e3 = [torch.empty(M, A, device=DEV) for _ in range(3)]
    ops.sac_squash_fwd(head, M, A, (-5, 2), None, 7, ctr, 1, box, 0.0, eps_out=e1)
    ops.sac_squash_fwd(head, M, A, (-5, 2), None, 7, ctr, 1, box, 0.0, eps_out=e2)
    ops.sac_squash_fwd(head, M, A, (-5, 2), None, 7, ctr, 0, box, 0.0, eps_out=e3)
    assert torch.equal(e1, e2) and not torch.equal(e1, e3)
    x = e1.double().reshape(-1)
    assert abs(float(x.mean())) < 5 / math.sqrt(x.numel()) and abs(float(x.var()) - 1) < 0.03
    assert abs(float((x ** 3).mean())) < 0.05 and abs(float((x ** 4).mean()) - 3) < 0.15
    # the squashed, rescaled sample: a = clamp(tanh(mu + std * eps) * scale + bias); with mu = 0, log_std = lo + (hi-lo)/2 the moments
    # of tanh(std * eps) are those of the same transform of a torch normal sample
    act = torch.empty(M, A, device=DEV)
    ops.sac_squash_fwd(head, M, A, (-5, 2), None, 7, ctr, 1, box, 0.0, dst=act, dst_ld=A)
    std = math.exp(-5 + 0.5 * 7 * 1.0)
    ref = torch.tanh(std * torch.randn(10 ** 6, dtype=torch.float64, generator=torch.Generator().manual_seed(1)))
    assert abs(float(act.double().abs().mean()) - float(ref.abs().mean())) < 0.01


@pytest.mark.parametrize('fixture', SG.FIXTURES)
def test_agent_replays_the_reference_golden_run(fixture, tmp_path):
    g = SG.load(fixture)
    a = SG.make_agent(g, DEV, tmp_path, over={'mixed_precision': False})
    rows = SG.run(a, g)
    SG.compare(a, g, rows, rtol=2e-3, atol=2e-4)


@pytest.mark.parametrize('fixture', SG.FIXTURES)
def test_cuda_graph_updates_match_eager_updates_bit_for_bit(fixture, tmp_path):
    """device RNG path (no tapes): the captured critic-only / critic+actor graphs replay exactly what the eager updates compute"""
    g = SG.load(fixture)
    outs = []
    for graph in (False, True):
        a = SG.make_agent(g, DEV, tmp_path / str(graph), over={'mixed_precision': False, 'b200_cuda_graph': graph})
        rows = SG.run(a, g, use_tapes=False)
        torch.cuda.synchronize()
        if graph:
            assert len(a._graphs) == (2 if a.policy_frequency > 1 else 1)
        outs.append((torch.stack([r[0] if r[1] else torch.cat([r[0][:3], torch.zeros(5)]) for r in rows]), a.model.actor.flat.clone(), a.model.critic.flat.clone(), a.model.critic_target.flat.clone(),
                     a.model.log_alpha.clone()))
    for x, y in zip(*outs):
        assert torch.equal(x, y)


@pytest.mark.parametrize('fixture', SG.FIXTURES)
def test_mixed_precision_tracks_fp32(fixture, tmp_path):
    """layer-wise bf16 wgmma GEMMs (mixed_precision: True) against the fp32 agent on the same tapes: per-update critic losses within 5 %
    (+ 2e-2 absolute) and final weights within 2e-2"""
    g = SG.load(fixture)
    res = []
    for mp in (False, True):
        a = SG.make_agent(g, DEV, tmp_path / str(mp), over={'mixed_precision': mp})
        rows = SG.run(a, g)
        res.append((torch.stack([r[0] for r in rows]), a.model.actor.flat.cpu(), a.model.critic.flat.cpu()))
    torch.testing.assert_close(res[1][0][:, :3], res[0][0][:, :3], rtol=5e-2, atol=2e-2)
    torch.testing.assert_close(res[1][1], res[0][1], rtol=0, atol=2e-2)
    torch.testing.assert_close(res[1][2], res[0][2], rtol=0, atol=2e-2)


def test_uniform_actions_philox_range_determinism_and_moments():
    from rl_games_b200 import ops
    N, A = 40009, 17
    g = torch.Generator().manual_seed(2)
    low = (-1 - torch.rand(A, generator=g) * 3).to(DEV)
    high = low + (0.1 + torch.rand(A, generator=g) * 4).to(DEV)
    ctr = torch.tensor([3], dtype=torch.int64, device=DEV)
    a1, a2, a3 = [torch.full((N, A), float('nan'), device=DEV) for _ in range(3)]
    ops.sac_uniform_actions(low, high, None, 5, ctr, a1, N, A)
    ops.sac_uniform_actions(low, high, None, 5, ctr, a2, N, A)
    ops.bump_u64(ctr)
    ops.sac_uniform_actions(low, high, None, 5, ctr, a3, N, A)
    assert torch.equal(a1, a2) and not torch.equal(a1, a3)
    u = (a1 - low) / (high - low)
    assert bool((u >= 0).all()) and bool((u < 1).all())
    n = u.numel()
    assert abs(float(u.double().mean()) - 0.5) < 5 * math.sqrt(1 / 12 / n)
    assert abs(float(u.double().var()) - 1 / 12) < 2e-3
    counts = torch.histc(u.double().cpu(), bins=64, min=0.0, max=1.0)
    chi2 = float(((counts - n / 64) ** 2 / (n / 64)).sum())
    assert chi2 < 63 + 6 * math.sqrt(2 * 63), chi2
    # tape path: low + (high - low) * u exactly
    tape = torch.rand(N, A, generator=g).to(DEV)
    ops.sac_uniform_actions(low, high, tape, 5, None, a1, N, A)
    assert torch.equal(a1, low + (high - low) * tape)


@pytest.mark.parametrize('tau', [0.005, 0.05, 0.5, 0.9])
def test_polyak_is_torch_lerp_bit_for_bit(tau):
    from rl_games_b200 import ops
    g = torch.Generator().manual_seed(int(tau * 1000))
    n = 100003
    tgt, src = torch.randn(n, generator=g).to(DEV), torch.randn(n, generator=g).to(DEV)
    ref = tgt.clone().lerp_(src, tau)
    ops.sac_polyak(tgt, src, tau)
    assert torch.equal(tgt, ref)


@pytest.mark.parametrize('n_params', [1, 66433])
def test_adam_then_polyak_matches_the_unfused_reference_sequence(n_params):
    """sac_agent.py update: critic_optimizer.step() (torch.optim.Adam(fused=True)), then target.lerp_(critic, tau), over several steps on
    the same device, with the gradient-norm clip inactive (clip_coef clamps to exactly 1.0).  The Polyak step alone is bit-exact
    (test_polyak_is_torch_lerp_bit_for_bit).  adam_step is the existing optimiser kernel of the PPO path: it restates torch's fused Adam
    in its CPU form (exp_avg by lerp, bias corrections from fp64 running products), while torch's CUDA fused Adam updates exp_avg as
    beta1 * m + (1 - beta1) * g; over five steps the two differ by at most a few fp32 ulps (4.8e-7 measured on an H100), which is the
    bound asserted here."""
    from rl_games_b200 import ops
    g = torch.Generator().manual_seed(n_params)
    p0 = torch.randn(n_params, generator=g).to(DEV)
    tgt0 = torch.randn(n_params, generator=g).to(DEV)
    grads = [torch.randn(n_params, generator=g).to(DEV) * 1e-3 for _ in range(5)]
    lr, betas, tau = 3e-4, (0.9, 0.999), 0.005
    # reference
    p = torch.nn.Parameter(p0.clone())
    tgt_r = tgt0.clone()
    opt = torch.optim.Adam([p], lr=lr, betas=betas, fused=True)
    for gr in grads:
        p.grad = gr.clone()
        torch.nn.utils.clip_grad_norm_([p], 1e6)
        opt.step()
        tgt_r.lerp_(p.data, tau)
    # kernels
    flat, m, v, tgt = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0), tgt0.clone()
    state = torch.zeros(8, dtype=torch.float64, device=DEV)
    state[0] = lr
    cfg = ops.OptCfg(betas[0], betas[1], 1e-8, 0.0, 1e6, 0.0, 0.0, 0.0, 1.0, 1.0, 1, 0)
    counter = torch.zeros(1, dtype=torch.int32, device=DEV)
    for gr in grads:
        ops.adam_step(flat, gr, m, v, state, None, cfg, None, counter)
        ops.sac_polyak(tgt, flat, tau)
    st = opt.state[p]
    torch.testing.assert_close(flat, p.data, rtol=2e-6, atol=1e-7)
    torch.testing.assert_close(m, st['exp_avg'], rtol=2e-6, atol=1e-10)
    torch.testing.assert_close(v, st['exp_avg_sq'], rtol=2e-6, atol=1e-14)
    torch.testing.assert_close(tgt, tgt_r, rtol=2e-6, atol=1e-7)


@pytest.mark.parametrize('fixture', SG.FIXTURES)
def test_captured_updates_replay_the_golden_run(fixture, tmp_path):
    """tapes fed through fixed device buffers into the CUDA-graph updates: the captured path against the reference's golden run"""
    g = SG.load(fixture)
    a = SG.make_agent(g, DEV, tmp_path, over={'mixed_precision': False, 'b200_cuda_graph': True})
    rows = SG.run(a, g)
    assert len(a._graphs) == (2 if a.policy_frequency > 1 else 1)
    SG.compare(a, g, rows, rtol=2e-3, atol=2e-4)


@pytest.mark.parametrize('fixture', SG.FIXTURES)
def test_default_configuration_graph_with_mixed_precision(fixture, tmp_path):
    """the defaults (mixed_precision and b200_cuda_graph on): captured updates equal eager ones bit for bit on the device RNG path, and on
    the golden tapes the run tracks the reference within the mixed-precision tolerance"""
    g = SG.load(fixture)
    outs = []
    for graph in (False, True):
        a = SG.make_agent(g, DEV, tmp_path / str(graph), over={'mixed_precision': True, 'b200_cuda_graph': graph})
        rows = SG.run(a, g, use_tapes=False)
        outs.append((torch.stack([r[0] if r[1] else torch.cat([r[0][:3], torch.zeros(5)]) for r in rows]), a.model.actor.flat.clone(),
                     a.model.critic.flat.clone(), a.model.critic_target.flat.clone(), a.model.log_alpha.clone()))
    for x, y in zip(*outs):
        assert torch.equal(x, y)
    a = SG.make_agent(g, DEV, tmp_path / 'golden', over={'mixed_precision': True, 'b200_cuda_graph': True})
    rows = SG.run(a, g)
    ref = g['losses']
    c = torch.stack([r[0][1:3] for r in rows])
    torch.testing.assert_close(c, torch.tensor([[r['c1'], r['c2']] for r in ref]), rtol=5e-2, atol=2e-2)
    torch.testing.assert_close(a.model.critic.flat.cpu(), torch.cat([v.reshape(-1) for v in g['state']['critic'].values()]), rtol=0, atol=2e-2)
