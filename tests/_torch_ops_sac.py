"""Torch (CPU) stand-ins for the SAC ops of ``rl_games_b200.ops`` (csrc/sac.cu) -- TEST INFRASTRUCTURE ONLY.  They restate what each
kernel does, argument for argument, so that the host logic of ``rl_games_b200.agent_sac`` can be run against the reference's golden runs
without a GPU.  Installed by monkeypatching inside one test; they prove nothing about the kernels (tests/test_sac_gpu.py does that)."""
import math

import torch

import _torch_ops as T


def _rng_free(x, what):
    if x is None:
        raise AssertionError(f'{what}: the CPU stand-ins replay tapes only (no device Philox)')
    return x


def sac_replay_insert(obs, action, reward, next_obs, final_obs, dones_u8, time_outs_u8, value_bootstrap, next_step, prev_dones_u8, rb, slot,
                      term_scratch, trunc_scratch, ep_state, meter, games_to_track):
    N = obs.shape[0]
    cap = rb['obs'].shape[0]
    d = dones_u8.bool()
    tr = (time_outs_u8.bool() if (time_outs_u8 is not None and value_bootstrap) else torch.zeros(N, dtype=torch.bool))
    term = d & ~tr
    live = ~prev_dones_u8.bool() if next_step else torch.ones(N, dtype=torch.bool)
    rows = live.nonzero().reshape(-1)
    nx = next_obs.clone()
    if not next_step:
        nx[tr] = (final_obs if final_obs is not None else obs)[tr]
    head = int(rb['state'][0])
    for k, r in enumerate(rows.tolist()):
        s = (head + k) % cap
        rb['obs'][s], rb['act'][s], rb['rew'][s], rb['next'][s] = obs[r], action[r], reward[r], nx[r]
        rb['term'][s], rb['trunc'][s] = int(term[r]), int(tr[r])
    n = rows.numel()
    rb['state'][0] = (head + n) % cap
    rb['state'][1] = min(cap, int(rb['state'][1]) + n)
    cr, cl = ep_state[:N], ep_state[N:]
    cr.add_(reward * live.float())
    cl.add_(live.float())
    sel = (d & live).nonzero().reshape(-1)
    if sel.numel():
        k = sel.numel()
        size = min(k, games_to_track)
        old = min(games_to_track - size, int(meter[2]))
        tot = old + size
        meter[0] = (float(meter[0]) * old + float(cr[sel].double().mean()) * size) / tot
        meter[1] = (float(meter[1]) * old + float(cl[sel].double().mean()) * size) / tot
        meter[2] = tot
    cr.mul_(1.0 - d.float())
    cl.mul_(1.0 - d.float())
    prev_dones_u8.copy_(d.to(torch.uint8))


def sac_replay_sample(rb, B, idx_tape, seed, rng_ctr, norm_mean, norm_std, x_cur, x_pi, x_next, reward, not_done, idx_out=None):
    k = _rng_free(idx_tape, 'sac_replay_sample').long()
    D = rb['obs'].shape[1]
    o, n = rb['obs'][k], rb['next'][k]
    if norm_mean is not None:
        o, n = T._norm(o, norm_mean, norm_std), T._norm(n, norm_mean, norm_std)
    x_cur[:B, :D], x_pi[:B, :D], x_next[:B, :D] = o, o, n
    x_cur[:B, D:] = rb['act'][k]
    reward[:B] = rb['rew'][k]
    not_done[:B] = 1.0 - rb['term'][k].float()
    if idx_out is not None:
        idx_out[:B] = k


def _squash(head, A, bounds, eps, box, lss):
    mu, raw = head[:, :A], head[:, A:2 * A]
    lo, hi = bounds
    t = torch.tanh(raw)
    ls = lo + 0.5 * (hi - lo) * (t + 1)
    sd = ls.exp()
    x = mu + eps * sd
    y = torch.tanh(x)
    nlp = -((x - mu) ** 2) / (2 * sd ** 2) - sd.log() - math.log(math.sqrt(2 * math.pi))
    jac = 2.0 * (math.log(2.0) - x - torch.nn.functional.softplus(-2.0 * x))
    logp = (-jac + nlp).sum(-1) - lss
    sc, bi, low, high = box
    return (y * sc + bi).clamp(low, high), logp


def sac_squash_fwd(head, M, A, log_std_bounds, noise, seed, rng_ctr, site, act, log_action_scale_sum, dst=None, dst_ld=0, eps_out=None,
                   logp=None):
    eps = _rng_free(noise, 'sac_squash_fwd')
    a, lp = _squash(head[:M], A, log_std_bounds, eps, act, log_action_scale_sum)
    if dst is not None:
        dst[:M, :A] = a
    if eps_out is not None:
        eps_out[:M] = eps
    if logp is not None:
        logp[:M] = lp


def sac_uniform_actions(low, high, u_tape, seed, rng_ctr, out, N, A):
    out.copy_(low + (high - low) * _rng_free(u_tape, 'sac_uniform_actions'))


def sac_critic_loss(q1, q2, q1t, q2t, logp_next, reward, not_done, log_alpha, gamma, B, dq1, dq2, stats):
    q1, q2, q1t, q2t = q1.reshape(-1), q2.reshape(-1), q1t.reshape(-1), q2t.reshape(-1)
    tq = reward + not_done * gamma * (torch.min(q1t, q2t) - log_alpha.exp() * logp_next)
    e1, e2 = q1 - tq, q2 - tq
    l1, l2 = (e1 * e1).mean(), (e2 * e2).mean()
    stats[0], stats[1], stats[2] = 0.5 * (l1 + l2), l1, l2
    dq1.reshape(-1)[:] = e1 / B
    dq2.reshape(-1)[:] = e2 / B


def sac_actor_loss(q1, q2, logp, log_alpha, min_alpha, target_entropy, learnable, B, dq1, dq2, d_log_alpha, stats):
    q1, q2 = q1.reshape(-1), q2.reshape(-1)
    alpha = log_alpha.exp()
    stats[3] = (torch.clamp_min(alpha, min_alpha) * logp - torch.min(q1, q2)).mean()
    stats[4] = -logp.mean()
    m = (-logp - target_entropy).mean()
    stats[6] = alpha[0] * m if learnable else 0.0
    if learnable:
        d_log_alpha[0] = alpha[0] * m
    g = -1.0 / B
    dq1.reshape(-1)[:] = torch.where(q1 < q2, g, torch.where(q1 == q2, 0.5 * g, 0.0))
    dq2.reshape(-1)[:] = torch.where(q2 < q1, g, torch.where(q1 == q2, 0.5 * g, 0.0))


def sac_squash_bwd(head, eps, M, A, log_std_bounds, act, dxa1, dxa2, dx_ld, log_alpha, min_alpha, d_head):
    h = head[:M].detach().clone().requires_grad_(True)
    a, lp = _squash(h, A, log_std_bounds, eps[:M], act, 0.0)
    c = torch.clamp_min(log_alpha.exp(), min_alpha)[0]
    L = (c * lp).mean() + ((dxa1[:M, :A] + dxa2[:M, :A]) * a).sum()
    L.backward()
    d_head[:M] = h.grad


def sac_polyak(target, src, tau, log_alpha=None, alpha_stat=None):
    target.lerp_(src, tau)
    if alpha_stat is not None:
        alpha_stat[0] = log_alpha.exp()[0]


def _adam_step(params, grads, exp_avg, exp_avg_sq, state_d, kl_dev, cfg, stats_out, counter, n=None, **kw):
    """torch.optim.Adam(fused) with clip_grad_norm_ (adam.cu adam_step_kernel)"""
    n = params.numel() if n is None else n
    g = grads[:n].clone()
    if cfg.truncate_grads:
        tn = torch.linalg.vector_norm(g)
        g = g * torch.clamp(cfg.grad_norm / (tn + 1e-6), max=1.0)
    lr, step = float(state_d[0]), float(state_d[1]) + 1
    m, v = exp_avg[:n], exp_avg_sq[:n]
    m.lerp_(g, 1 - cfg.beta1)
    v.mul_(cfg.beta2).addcmul_(g, g, value=1 - cfg.beta2)
    bc1, bc2 = 1 - cfg.beta1 ** step, 1 - cfg.beta2 ** step
    params[:n] -= (lr / bc1) * m / (v.sqrt() / math.sqrt(bc2) + cfg.eps)
    state_d[1] = step
    state_d[2] = cfg.beta1 ** step
    state_d[3] = cfg.beta2 ** step


def _bump(t):
    t.add_(1)


def install(monkeypatch):
    from rl_games_b200 import ops
    for name in ('linear_fwd', 'linear_bwd_data', 'linear_bwd_weight', 'reduce_splits', 'moments_update', 'refresh_norm'):
        monkeypatch.setattr(ops, name, getattr(T, name))
    for name in ('linear_fwd_tc', 'linear_bwd_data_tc', 'linear_bwd_weight_tc'):
        base = getattr(T, name[:-3])
        monkeypatch.setattr(ops, name, lambda *a, _b=base, bf16_arena=None, **k: _b(*a, **k))
    for name in ('sac_replay_insert', 'sac_replay_sample', 'sac_squash_fwd', 'sac_uniform_actions', 'sac_critic_loss', 'sac_actor_loss',
                 'sac_squash_bwd', 'sac_polyak'):
        monkeypatch.setattr(ops, name, globals()[name])
    monkeypatch.setattr(ops, 'adam_step', _adam_step)
    monkeypatch.setattr(ops, 'bump_u64', _bump)
