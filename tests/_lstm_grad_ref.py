"""fp64 reference of ONE minibatch of a recurrent (LSTM) continuous PPO policy: the loss and the autograd gradient of every parameter
tensor, from the tensors the CUDA minibatch update reads -- TEST INFRASTRUCTURE ONLY (CPU).

Inputs are in the agent's time-major arena layout ([H, N, ...]: step t, env n).  Minibatch i = envs [i*epm, (i+1)*epm) x every step, in
the reference's flat order env*H + t (swap_and_flatten01, a2c_common.py:33-40), cut into sequences of seq_length consecutive steps of one
env: sequence env*(H/T) + j = steps j*T .. j*T + T-1, started from the rollout's snapshots rnn_h0[j, env] / rnn_c0[j, env]
(mb_rnn_states, a2c_common.py:1081-1083, :1193-1199) and reset by the train-time done flags before every step (RnnWithDones).  The model
is oracle.ppo_oracle's (lstm_with_dones, network_forward; tests/_lstm_ln_oracle.py's LayerNorm of the LSTM output for
rnn.layer_norm), LSTM before or after the MLP; the loss is the oracle's calc_losses (actor / critic / entropy / bound terms, apply_masks).

Observation normalisation takes the kernels' route: the running statistics (fp64 mean / var, int64 count) are a snapshot taken BEFORE the
update; when that update merges its own minibatch's moments at its start (the first update of an epoch, or every update when the
minibatch moments are not precomputed), the merge is replayed here with the oracle's RunningMeanStd (fp64 moments of the minibatch rows).
The CUDA update can not be asked for its statistics afterwards: with precomputed minibatch moments its optimiser kernel already merges the
NEXT minibatch's.  The rows are then normalised exactly as the kernels read them, in fp32 -- clamp((x - mean_f32) / std_f32, -5, 5) with
mean_f32 = float(mean), std_f32 = sqrt(float(var) + 1e-5) -- and promoted to fp64; everything after that is fp64."""
import math
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from oracle import ppo_oracle as O  # noqa: E402
import _lstm_ln_oracle as LO  # noqa: E402

LOSS_KEYS = ('e_clip', 'clip_value', 'use_smooth_clamp', 'ppo', 'critic_coef', 'entropy_coef', 'bounds_loss_coef', 'bound_loss_type')


def normalized_obs(x, obs_stats, merge):
    """x [R, D] fp32 rows of the minibatch; obs_stats = (running_mean f64, running_var f64, count i64) before the update.  Returns the
    rows as the kernels read them (fp64 promotion of the fp32 normalisation) and the statistics they were normalised with."""
    rms = O.RunningMeanStd((x.shape[1],))
    rms.load({'running_mean': obs_stats[0].cpu(), 'running_var': obs_stats[1].cpu(), 'count': obs_stats[2].cpu().reshape(())})
    if merge:
        x64 = x.double()
        rms.update_from_moments(x64.mean(0), x64.var(0, unbiased=False), x.shape[0])
    mean_f32 = rms.running_mean.float()
    std_f32 = torch.sqrt(rms.running_var.float() + rms.epsilon)
    return ((x.float() - mean_f32) / std_f32).clamp(-5.0, 5.0).double(), rms


class _RoundedOperands:
    """torch.nn.functional as oracle.ppo_oracle sees it while a reference of the layer-wise tensor-core path runs: F.linear rounds both
    operands to `dtype` (straight-through gradient) and multiplies in fp64, as the bf16-operand, fp32-accumulate GEMMs do; the heads, which
    run in fp32 kernels on that path too, stay exact"""

    def __init__(self, dtype, exact_weights):
        self.dtype, self.exact = dtype, exact_weights

    def __getattr__(self, name):
        return getattr(F, name)

    def linear(self, x, w, b=None):
        if any(w is e for e in self.exact):
            return F.linear(x, w, b)
        r = lambda t: t + (t.to(self.dtype).to(t.dtype) - t).detach()     # noqa: E731
        return F.linear(r(x), r(w), b)


def minibatch_loss_and_grads(params, batch, i, epm, seq_length, units, loss_cfg, rnn_before_mlp=True, layer_norm=False, activation='elu',
                             obs_stats=None, merge_obs_stats=True, gemm_operands=None):
    """params: {reference state-dict name: tensor} (oracle.ppo_oracle.param_names(.., lstm=True) / _lstm_ln_oracle.param_names).
    batch: arena tensors -- 'obses' [H,N,D], 'actions' [H,N,A], 'neglogpacs', 'old_values', 'returns', 'advantages' [H,N] (the prepared,
    normalised dataset), 'valid' [H,N] or None, 'rnn_h0' / 'rnn_c0' [H/T,N,Hd], 'dones' [H,N] (the train-time reset flags: the buffer's
    dones, or the next_step envs' rnn_dones).  loss_cfg: the loss options of oracle.ppo_oracle.DEFAULT_CFG (LOSS_KEYS).
    obs_stats None = no input normalisation.  gemm_operands (e.g. torch.bfloat16): the operands of every GEMM but the heads' are rounded
    to that type first, the forward of the layer-wise tensor-core path.  Returns (loss, {name: gradient}), fp64."""
    c = dict(O.DEFAULT_CFG)
    c.update({k: v for k, v in loss_cfg.items() if k in LOSS_KEYS})
    H, T = batch['obses'].shape[0], seq_length
    e0, e1 = i * epm, (i + 1) * epm
    S = epm * H // T

    def rows(name):
        return O.swap_and_flatten01(batch[name][:, e0:e1].cpu())

    obs = rows('obses')
    x = obs.double() if obs_stats is None else normalized_obs(obs, obs_stats, merge_obs_stats)[0]
    p = {k: v.detach().cpu().double().clone().requires_grad_(True) for k, v in params.items()}
    h0, c0 = (batch[k][:, e0:e1].cpu().transpose(0, 1).reshape(S, -1).double() for k in ('rnn_h0', 'rnn_c0'))
    dones = rows('dones').reshape(S, T).transpose(0, 1)

    def rnn(xf):
        out, _, _ = O.lstm_with_dones(p, xf.reshape(S, T, -1).transpose(0, 1), h0, c0, dones)
        if layer_norm:
            out = F.layer_norm(out, (out.shape[-1],), p[LO.LN_NAMES[0]], p[LO.LN_NAMES[1]], 1e-5)
        return out.transpose(0, 1).reshape(S * T, -1)

    if gemm_operands is not None:
        O.F = _RoundedOperands(gemm_operands, [p['a2c_network.value.weight'], p['a2c_network.mu.weight']])
    try:
        if rnn_before_mlp:
            mu, logstd, value = O.network_forward(p, rnn(x), len(units), activation)
        else:
            mu, logstd, value = O.network_forward(p, x, len(units), activation, heads_after=rnn)
    finally:
        O.F = F
    sigma = torch.exp(logstd)
    neglogp = O.neglogp_fn(rows('actions').double(), mu, sigma, logstd)
    a_loss = O.actor_loss(rows('neglogpacs').double(), neglogp, rows('advantages').double(), c['ppo'], c['e_clip'],
                          smooth=c['use_smooth_clamp'])
    c_loss = O.critic_loss(rows('old_values').double().unsqueeze(1), value, c['e_clip'], rows('returns').double().unsqueeze(1),
                           c['clip_value'])
    entropy = (0.5 + 0.5 * math.log(2 * math.pi) + logstd).sum(dim=-1)
    bcoef = c['bounds_loss_coef']
    if bcoef is None:
        b_loss = torch.zeros(mu.shape[0], dtype=torch.float64)
    elif c['bound_loss_type'] == 'regularisation':
        b_loss = O.reg_loss(mu, bcoef)
    else:
        b_loss = O.bound_loss(mu, bcoef)
    mask = None if batch.get('valid') is None else rows('valid').double()
    (a, cl, ent, b), _ = O.apply_masks([a_loss.unsqueeze(1), c_loss, entropy.unsqueeze(1), b_loss.unsqueeze(1)], mask)
    loss = a + 0.5 * cl * c['critic_coef'] - ent * c['entropy_coef'] + b * (bcoef or 0.0)
    names = list(params)
    grads = torch.autograd.grad(loss, [p[n] for n in names], allow_unused=True)
    return loss.detach(), {n: (g if g is not None else torch.zeros_like(p[n])) for n, g in zip(names, grads)}


def window_done_positions(dones, i, epm, seq_length):
    """the window positions (0 .. T-1) at which minibatch i has at least one reset flag (position 0: a reset entering the window)"""
    H = dones.shape[0]
    d = dones[:, i * epm:(i + 1) * epm].cpu().bool().reshape(H // seq_length, seq_length, -1)
    return sorted(int(t) for t in d.any(dim=2).any(dim=0).nonzero().flatten())


def grad_errors(g, g_ref):
    """(max |g - g_ref| / max |g_ref|, |g| / |g_ref|) of one tensor"""
    g, g_ref = g.double().cpu().reshape(-1), g_ref.double().cpu().reshape(-1)
    scale = float(g_ref.abs().max())
    err = float((g - g_ref).abs().max()) / max(scale, 1e-30)
    ratio = float(g.norm()) / max(float(g_ref.norm()), 1e-30)
    return err, ratio
