"""PPO diagnostics summaries (`use_diagnostics: True`), the reference's ``rl_games.common.diagnostics`` (diagnostics.py:18-62).

The reference computes every minibatch's explained variance and clip fraction with torch ops and a host copy per minibatch.  Here the
device writes them into the stats rows the agent reads back once per epoch (explained variance: b200rl_explained_variance_f32, once
per epoch after the dataset is prepared; clip fraction: the loss kernels' B200RL_STAT_CLIPFRAC), and the agent replays ``mini_batch`` /
``mini_epoch`` from those rows after the read-back.  The aggregation below is the reference's, quirks included:

* ``exp_var``: fp32 mean over every minibatch entry since the previous ``epoch()`` (all mini-epochs);
* ``clip_frac/<k>``: fp32 mean over the minibatches of mini-epoch k.  With masks the reference keeps the per-row vector
  ``clip * m / sum(m)`` and averages the stacked [n_minibatches, B] tensor, so the written value is mean_i(frac_i) / B, and a minibatch
  without a valid row gives NaN (the division by sum(m) is not clamped there);
* ``rms_value/{mean,var}``: the value normaliser's running statistics; ``rms_advantage/{mean,var}``: the EMA advantage normaliser's
  EFFECTIVE statistics (moving_mean_std.py:42-60: variance clamped to 1 / max^2 before the square root);
* every tag is written at the EPOCH number, and every key ever set is re-sent each epoch.
"""
import numpy as np


class DefaultDiagnostics:
    """no diagnostics (key absent or False, and every rank but 0)"""

    def send_info(self, writer):
        pass

    def epoch(self, agent, current_epoch):
        pass

    def mini_epoch(self, agent, miniepoch):
        pass

    def mini_batch(self, agent, batch, e_clip, minibatch):
        pass


class PpoDiagnostics(DefaultDiagnostics):
    def __init__(self):
        self.diag_dict = {}
        self.clip_fracs = []
        self.exp_vars = []
        self.current_epoch = 0

    def send_info(self, writer):
        if writer is None:
            return
        for k, v in self.diag_dict.items():
            writer.add_scalar(k, v, self.current_epoch)

    def epoch(self, agent, current_epoch):
        self.current_epoch = current_epoch
        for k, v in agent.diagnostics_normaliser_stats().items():
            self.diag_dict[k] = v
        self.diag_dict['diagnostics/exp_var'] = _mean32(self.exp_vars)
        self.exp_vars = []

    def mini_epoch(self, agent, miniepoch):
        self.diag_dict[f'diagnostics/clip_frac/{miniepoch}'] = _mean32(self.clip_fracs)
        self.clip_fracs = []

    def mini_batch(self, agent, batch, e_clip, minibatch):
        """batch: {'exp_var', 'clip_frac'} fp32 scalars of one minibatch, read back from its stats row; 'clip_frac' is already
        the reference's masked per-row share (frac / B) where the minibatch carries masks"""
        self.exp_vars.append(batch['exp_var'])
        self.clip_fracs.append(batch['clip_frac'])


def _mean32(xs):
    """fp32 mean of fp32 scalars, like torch.stack(xs).mean()"""
    return float(np.mean(np.asarray(xs, dtype=np.float32), dtype=np.float32))


def make_diagnostics(use_diagnostics, global_rank):
    """a2c_common.py:222-227: the diagnostics object on rank 0 only"""
    return PpoDiagnostics() if use_diagnostics and global_rank == 0 else DefaultDiagnostics()


def replay(agent, exp_var, clip_frac, sum_mask, masked, minibatch_size, n_minibatches, mini_epochs, e_clip):
    """calls mini_batch / mini_epoch in update order from one epoch's read-back per-update columns (host tensors of
    mini_epochs * n_minibatches entries, update u = mini-epoch u // n_minibatches, minibatch u % n_minibatches)"""
    d = agent.diagnostics
    ev = np.asarray(exp_var, dtype=np.float32)
    cf = np.asarray(clip_frac, dtype=np.float32)
    if masked:
        cf = np.where(np.asarray(sum_mask) > 0, cf / np.float32(minibatch_size), np.float32('nan')).astype(np.float32)
    for e in range(mini_epochs):
        for i in range(n_minibatches):
            u = e * n_minibatches + i
            d.mini_batch(agent, {'exp_var': ev[u], 'clip_frac': cf[u]}, e_clip, i)
        d.mini_epoch(agent, e)
