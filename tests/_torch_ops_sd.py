"""Torch (CPU) stand-ins for the state-dependent sigma entry points (ppo_head_loss_sd, policy_head_sample_sd) -- TEST INFRASTRUCTURE
ONLY, in addition to tests/_torch_ops.py (whose stand-ins are used unchanged for everything else).  The sigma parametrisation is
restated from models.py apply_sigma_parametrization; the gradients come from autograd."""
import math

import torch

import _torch_ops as T
from oracle import ppo_oracle as O

PARAM_NAMES = {0: 'exp', 1: 'softplus', 2: 'linear'}


def apply_sigma(raw, parametrization, min_sigma=0.0, logstd_bounds=None):
    """models.py apply_sigma_parametrization: raw head output -> (sigma, logstd)"""
    if parametrization == 'softplus':
        sigma = torch.nn.functional.softplus(raw) + min_sigma
    elif parametrization in ('linear', 'scalar'):
        floor = max(min_sigma, 1e-3)
        sigma = floor + torch.nn.functional.softplus(raw - floor)
    else:
        if logstd_bounds is not None:
            raw = torch.clamp(raw, logstd_bounds[0], logstd_bounds[1])
        sigma = torch.exp(raw)
        if min_sigma > 0:
            sigma = sigma + min_sigma
        else:
            return sigma, raw
    return sigma, torch.log(sigma)


def _apply_cfg(raw, c):
    bounds = (c.logstd_lo, c.logstd_hi) if c.has_logstd_bounds else None
    return apply_sigma(raw, PARAM_NAMES[c.parametrization], c.min_sigma, bounds)


def policy_head_sample_sd(a_last, W_head, b_head, sigma_cfg, vms_mean, vms_var, normalize_value, noise, seed, rng_epoch, step_index, actions,
                          mus, sigmas, neglogp, values, env_actions, clip_actions, act_low, act_high, dones_cur, dones_out, prev_dones,
                          valid_out, N, A, values_only=False):
    head = a_last[:N] @ W_head.t() + b_head
    val = head[:, 0]
    if normalize_value:
        val = torch.sqrt(vms_var.float() + 1e-5) * torch.clamp(val, -5.0, 5.0) + vms_mean.float()
    values.copy_(val)
    if values_only:
        return
    assert noise is not None, 'the host-logic test always supplies the normal tape'
    mu = head[:, 1:A + 1]
    sg, ls = _apply_cfg(head[:, A + 1:], sigma_cfg)
    act = mu + sg * noise
    actions.copy_(act); mus.copy_(mu); sigmas.copy_(sg)
    neglogp.copy_(O.neglogp_fn(act, mu, sg, ls))
    if env_actions is not None:
        ea = act
        if clip_actions:
            ea = torch.clamp(act, -1.0, 1.0) * ((act_high - act_low) * 0.5) + (act_high + act_low) * 0.5
        env_actions.copy_(ea)
    if dones_out is not None:
        dones_out.copy_(dones_cur)
    if valid_out is not None:
        valid_out.copy_(1.0 - prev_dones if prev_dones is not None else torch.ones(N))


def ppo_head_loss_sd(a_last, W_head, b_head, sigma_cfg, entropy_coef_dev, actions, old_mu, old_sigma, old_values_n, returns_n, old_neglogp,
                     advs_n, mask, rows_per_chunk, chunk_stride, M, A, cfg, inv_count, d_head, d_alast, act_last, partials, mu_out=None,
                     value_out=None, neglogp_out=None):
    """heads + calc_losses (entropy bonus included) + backward to (head, a_last); the scalars travel to _torch_ops.ppo_loss_finalize
    through its side channel with zero log-std slots, as the kernel's partial rows carry them"""
    def arena(t, width=1):
        return T._rows(t, M, width, rows_per_chunk, chunk_stride, width)
    al = a_last[:M].clone().requires_grad_(True)
    head = al @ W_head.t() + b_head
    head.retain_grad()
    value, mu = head[:, :1], head[:, 1:A + 1]
    sg, ls = _apply_cfg(head[:, A + 1:], sigma_cfg)
    act, omu, osg = arena(actions, A), arena(old_mu, A), arena(old_sigma, A)
    rm = None if mask is None else arena(mask).squeeze(1)
    nlp = O.neglogp_fn(act, mu, sg, ls)
    ent = (0.5 + 0.5 * math.log(2 * math.pi) + torch.log(sg)).sum(-1)
    a = O.actor_loss(arena(old_neglogp).squeeze(1), nlp, arena(advs_n).squeeze(1), bool(cfg.ppo), cfg.e_clip, smooth=bool(cfg.use_smooth_clamp))
    c = O.critic_loss(arena(old_values_n), value, cfg.e_clip, arena(returns_n), bool(cfg.clip_value)).squeeze(1)
    if cfg.has_bounds_loss and cfg.bound_loss_type == 1:
        b = O.bound_loss(mu, cfg.bounds_loss_coef)
    elif cfg.has_bounds_loss and cfg.bound_loss_type == 2:
        b = O.reg_loss(mu, cfg.bounds_loss_coef)
    else:
        b = torch.zeros(M)
    w = torch.full((M,), 1.0 / M) if inv_count is None else rm * inv_count[0]
    la, lc, le, lb = (a * w).sum(), (c * w).sum(), (ent * w).sum(), (b * w).sum()
    (la + 0.5 * cfg.critic_coef * lc - float(entropy_coef_dev[0]) * le + cfg.bounds_loss_coef * lb).backward()
    d_head[:M] = head.grad
    d_alast[:M] = al.grad * T._act_grad_from_out(a_last[:M], act_last)
    kl = (O.policy_kl(mu.detach(), sg.detach(), omu, osg, reduce=False) * w).sum()
    lr_ = arena(old_neglogp).squeeze(1) - nlp.detach()
    lo, hi = torch.log1p(torch.tensor(-cfg.e_clip)), torch.log1p(torch.tensor(cfg.e_clip))
    clipped = ((lr_ < lo) | (lr_ > hi)).float()
    mk = torch.ones(M) if rm is None else rm
    zero = torch.zeros(A)
    T._LOSS_SIDE['last'] = dict(stats=[la.detach(), lc.detach(), le.detach(), lb.detach(), kl, mk.sum(),
                                       (mk * clipped).sum() / mk.sum().clamp(min=1.0)], dls=zero, dent=zero)
    m_ = torch.arange(M)
    cidx = m_ // rows_per_chunk
    r = cidx * chunk_stride + (m_ - cidx * rows_per_chunk)
    idx = r.unsqueeze(1) * A + torch.arange(A).unsqueeze(0)
    T._flat(old_mu)[idx] = mu.detach()
    T._flat(old_sigma)[idx] = sg.detach()
    return 1


def install_sd(monkeypatch):
    """_torch_ops.install_continuous plus the state-dependent sigma stand-ins"""
    from rl_games_b200 import ops
    T.install_continuous(monkeypatch)
    monkeypatch.setattr(ops, 'policy_head_sample_sd', policy_head_sample_sd)
    monkeypatch.setattr(ops, 'ppo_head_loss_sd', ppo_head_loss_sd)
