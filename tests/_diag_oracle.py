"""Reference semantics of the PPO diagnostics summaries (`use_diagnostics: True`) -- TEST INFRASTRUCTURE ONLY.

A restatement of rl_games.common.diagnostics.PpoDiagnostics (diagnostics.py:18-62) and of the two torch_ext helpers it calls
(explained_variance torch_ext.py:204-215, policy_clip_fraction :217-227, get_mean_var_with_masks :182-191), masked forms included;
the unmasked forms are oracle.ppo_oracle.explained_variance / policy_clip_fraction.  Compared against the reference's own golden runs
(tests/golden/diag_*.pt) by tests/test_diagnostics_cpu.py, and used there as the torch stand-in of b200rl_explained_variance_f32."""
import math

import torch

from oracle import ppo_oracle as O


def mean_var_with_masks(values, masks):
    """torch_ext.py:182-191: clamped denominators, Bessel factor"""
    sum_mask = masks.sum().clamp(min=1.0)
    vm = values * masks
    mean = vm.sum() / sum_mask
    min_sqr = (vm ** 2 / sum_mask).sum() - (vm / sum_mask).sum() ** 2
    return mean, min_sqr * sum_mask / (sum_mask - 1).clamp(min=1.0)


def explained_variance(y_pred, y, masks=None):
    """torch_ext.py:204-215: masked, var_y is the variance of the PREDICTION (y_pred), not of y"""
    if masks is None:
        return O.explained_variance(y_pred, y)
    masks = masks.unsqueeze(1)
    _, var_y = mean_var_with_masks(y_pred, masks)
    _, var_dy = mean_var_with_masks(y - y_pred, masks)
    return 1.0 - var_dy / var_y


def policy_clip_fraction(new_neglogp, old_neglogp, clip_param, masks=None):
    """torch_ext.py:217-227: masked, a per-row vector clip * m / sum(m) (sum(m) not clamped)"""
    if masks is None:
        return O.policy_clip_fraction(new_neglogp, old_neglogp, clip_param)
    logratio = old_neglogp - new_neglogp
    clip = torch.logical_or(logratio < math.log(1.0 - clip_param), logratio > math.log(1.0 + clip_param)).float()
    return clip * masks / masks.sum()


def scalars(mini_batches, epochs, mini_epochs, n_minibatches):
    """PpoDiagnostics over one train() run: mini_batch after every minibatch, mini_epoch after every mini-epoch, epoch() once per epoch,
    send_info at the top of write_stats.  mini_batches: the dicts mini_batch was handed, in call order; epochs: per epoch the
    normaliser statistics epoch() reads ({'epoch', 'rms_value': (mean, var), 'rms_advantage': (mean, sqrs)}).  Returns the
    (tag, value, step) rows the summary writer receives."""
    diag, out, it = {}, [], iter(mini_batches)
    exp_vars = []
    for ep in epochs:
        for k in range(mini_epochs):
            clip_fracs = []
            for _ in range(n_minibatches):
                b = next(it)
                exp_vars.append(explained_variance(b['values'], b['returns'], b['masks']))
                clip_fracs.append(policy_clip_fraction(b['new_neglogp'], b['old_neglogp'], b['e_clip'], b['masks']))
            diag[f'diagnostics/clip_frac/{k}'] = torch.stack(clip_fracs).mean()
        if 'rms_advantage' in ep:       # GeneralizedMovingStats.get_mean_std (moving_mean_std.py:42-60): max 1e5, eps 0
            mean, sqrs = ep['rms_advantage']
            std = torch.sqrt(torch.clamp_min(sqrs - mean.pow(2), 1 / 1e5 ** 2))
            diag['diagnostics/rms_advantage/mean'] = mean
            diag['diagnostics/rms_advantage/var'] = std * std
        if 'rms_value' in ep:
            diag['diagnostics/rms_value/mean'], diag['diagnostics/rms_value/var'] = ep['rms_value']
        diag['diagnostics/exp_var'] = torch.stack(exp_vars).mean()
        exp_vars = []
        out += [(t, float(v), ep['epoch']) for t, v in diag.items()]
    return out
