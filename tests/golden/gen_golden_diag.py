"""Golden runs of the REAL reference with `use_diagnostics: True` (a2c_common.py:222-227, common/diagnostics.py:18-62): the reference's
own train() loop (gen_golden.py's train_loop recipe) over two epochs, with every summary scalar recorded as (tag, value, step) through a
recording writer.  Besides the scalars, each fixture keeps what the reference's PpoDiagnostics was handed -- every mini_batch's
(values, returns, new / old neglogp, masks, e_clip) and, at every epoch(), the normaliser statistics -- so that the oracle
(tests/_diag_oracle.py) can restate the aggregation from the same inputs:

    python tests/golden/gen_golden_diag.py

writes tests/golden/diag_*.pt (committed)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from gen_golden import HERE, gen_agent, gen_agent_discrete  # noqa: E402

_REC = {}


def _install_recorder():
    from rl_games.common import diagnostics as D
    orig_mb, orig_ep = D.PpoDiagnostics.mini_batch, D.PpoDiagnostics.epoch

    def mini_batch(self, agent, batch, e_clip, minibatch):
        _REC.setdefault('mini_batches', []).append(
            {k: (v.detach().clone() if torch.is_tensor(v) else v) for k, v in batch.items()} | {'e_clip': float(e_clip)})
        return orig_mb(self, agent, batch, e_clip, minibatch)

    def epoch(self, agent, current_epoch):
        st = {'epoch': current_epoch, 'n_mini_batches': len(_REC.get('mini_batches', []))}
        if agent.normalize_value:
            st['rms_value'] = (agent.value_mean_std.running_mean.clone(), agent.value_mean_std.running_var.clone())
        if agent.normalize_rms_advantage:
            ams = agent.advantage_mean_std
            st['rms_advantage'] = (ams.mean.clone(), ams.sqrs.clone())
        _REC.setdefault('epochs', []).append(st)
        return orig_ep(self, agent, current_epoch)
    D.PpoDiagnostics.mini_batch, D.PpoDiagnostics.epoch = mini_batch, epoch


def _attach(name):
    path = os.path.join(HERE, name)
    g = torch.load(path, weights_only=False)
    g['diag_inputs'] = {'mini_batches': _REC.pop('mini_batches'), 'epochs': _REC.pop('epochs')}
    torch.save(g, path)
    print('recorded', len(g['diag_inputs']['mini_batches']), 'mini_batch calls into', path)


def gen_diag():
    import shutil
    _install_recorder()
    diag = {'use_diagnostics': True, 'max_epochs': 2, 'save_best_after': 10_000}
    # continuous MLP, normalize_value, no masks: 4 mini-epochs x 2 minibatches
    shutil.rmtree('/tmp/golden_runs', ignore_errors=True)
    gen_agent('diag_mlp.pt', seed=30, train_loop=True, overrides=diag)
    _attach('diag_mlp.pt')
    # next_step autoreset (masked rows) with the EMA advantage normaliser, 4 minibatches per mini-epoch
    shutil.rmtree('/tmp/golden_runs', ignore_errors=True)
    gen_agent('diag_masked_rmsadv.pt', N=16, seed=31, autoreset='next_step', train_loop=True,
              overrides=dict(diag, normalize_rms_advantage=True, adv_rms_momentum=0.5, mini_epochs=3))
    _attach('diag_masked_rmsadv.pt')
    # LSTM policy (masked rows as well)
    shutil.rmtree('/tmp/golden_runs', ignore_errors=True)
    gen_agent('diag_lstm.pt', seed=32, autoreset='next_step', train_loop=True,
              network_over={'rnn': {'name': 'lstm', 'units': 8, 'layers': 1, 'before_mlp': True}}, overrides=dict(diag, seq_length=4))
    _attach('diag_lstm.pt')
    # discrete agent, shared trunk, masked rows, value normaliser
    shutil.rmtree('/tmp/golden_runs', ignore_errors=True)
    gen_agent_discrete('diag_discrete.pt', separate=False, seed=33, autoreset='next_step', train_loop=True,
                       overrides=dict(diag, normalize_input=True, normalize_value=True))
    _attach('diag_discrete.pt')


if __name__ == '__main__':
    gen_diag()
