"""The fp64 minibatch-gradient reference of the LSTM policy (tests/_lstm_grad_ref.py) against the CPU oracle: on OracleAgent minibatches
with truncate_grads: False, the reference's gradient of every parameter tensor must equal the oracle's unclipped `last_grads` to fp32
accuracy.  The oracle is pinned to the real reference by the golden fixtures (tests/test_oracle_vs_golden.py), so this ties the fp64
reference -- which the GPU tests hold the CUDA minibatch gradient to -- to the reference as well.

Covered: LSTM before / after the MLP, rnn.layer_norm off / on, same_step / next_step autoreset (masked rows, train-time reset flags that also
fire entering the first real row after a filler row); every minibatch of one mini-epoch, each after the previous one's Adam step.
Measured: the worst deviation over all cases, minibatches and tensors -- of the relative error max |g - g_ref| / max |g_ref| and of the
norm ratio |g| / |g_ref| from 1 -- is 3.1e-5 (the oracle's fp32 arithmetic); the bound is 1e-4, about 3x that."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _lstm_grad_ref as GR  # noqa: E402
import _lstm_ln_oracle as LO  # noqa: E402
from oracle import ppo_oracle as O  # noqa: E402

TOL = 1e-4


def _arena(flat, N, H):
    """dataset rows (flat order env*H + t) -> the agent's time-major arena [H, N, ...]"""
    return None if flat is None else flat.reshape(N, H, *flat.shape[1:]).transpose(0, 1)


@pytest.mark.parametrize('before', [True, False], ids=['lstm_before_mlp', 'lstm_after_mlp'])
@pytest.mark.parametrize('layer_norm', [False, True], ids=['plain', 'layer_norm'])
@pytest.mark.parametrize('autoreset', ['same_step', 'next_step'])
def test_reference_gradient_matches_oracle(before, layer_norm, autoreset):
    N, H, D, A, units, hid, T, mb = 32, 8, 6, 3, [16, 8], 8, 4, 64
    obs_tape, done_tape, tout_tape = O.make_tapes(2 * H + 1, N, D, seed=3, p_done=0.2)
    cfg = {'rnn_units': hid, 'seq_length': T, 'rnn_before_mlp': before, 'mask_autoreset_rows': autoreset == 'next_step',
           'truncate_grads': False, 'mini_epochs': 1, 'entropy_coef': 0.01, 'bounds_loss_coef': 1e-3}
    g = torch.Generator().manual_seed(4)
    noise = torch.randn(2, H, N, A, generator=g)
    env = O.TapeEnv(obs_tape, done_tape, tout_tape)
    if layer_norm:
        params = LO.init_params(D, units, A, seed=5, rnn_units=hid, rnn_before_mlp=before, ln_seed=6)
        oag = LO.make_agent(env, params, D, A, units, N, H, mb, cfg)
    else:
        params = O.init_params(D, units, A, seed=5, rnn_units=hid, rnn_before_mlp=before)
        oag = O.OracleAgent(env, params, D, A, units, N, H, mb, cfg)
    oag.obs = oag.env_reset()
    oag.train_epoch(noise[0])              # non-zero window-initial states and moved statistics for the epoch under test
    oag.epoch_num += 1
    oag.prepare_dataset(oag.play_steps(noise[1]))
    ds = oag.dataset
    batch = {'obses': _arena(ds['obs'], N, H), 'actions': _arena(ds['actions'], N, H), 'neglogpacs': _arena(ds['old_logp_actions'], N, H),
             'old_values': _arena(ds['old_values'].squeeze(1), N, H), 'returns': _arena(ds['returns'].squeeze(1), N, H),
             'advantages': _arena(ds['advantages'], N, H), 'valid': _arena(ds['rnn_masks'], N, H), 'dones': _arena(ds['dones'], N, H)}
    batch['rnn_h0'], batch['rnn_c0'] = (s.reshape(N, H // T, hid).transpose(0, 1) for s in ds['rnn_states'])
    epm = mb // H
    assert (batch['valid'] is not None) == (autoreset == 'next_step')
    worst = 0.0
    for i in range(oag.num_minibatches):
        assert GR.window_done_positions(batch['dones'], i, epm, T) == list(range(T))
        rms = oag.model.running_mean_std
        stats = (rms.running_mean.clone(), rms.running_var.clone(), rms.count.clone())
        params_now = {n: oag.model.p[n].detach().clone() for n in oag.model.names}
        rms.train()
        oag.train_actor_critic(oag.get_minibatch(i))
        _, g_ref = GR.minibatch_loss_and_grads(params_now, batch, i, epm, T, units, oag.cfg, rnn_before_mlp=before, layer_norm=layer_norm,
                                               obs_stats=stats, merge_obs_stats=True)
        assert set(g_ref) == set(oag.model.names)
        for n, g_o in zip(oag.model.names, oag.last_grads):
            err, ratio = GR.grad_errors(g_o, g_ref[n])
            worst = max(worst, err, abs(ratio - 1.0))
            assert err < TOL and abs(ratio - 1.0) < TOL, (i, n, err, ratio)
        # the statistics the reference replayed are the ones the oracle normalised with
        torch.testing.assert_close(rms.running_mean, GR.normalized_obs(O.swap_and_flatten01(batch['obses'][:, i * epm:(i + 1) * epm]),
                                                                       stats, True)[1].running_mean, rtol=1e-6, atol=1e-7)
    print(f'lstm grad reference vs oracle ({before}, {layer_norm}, {autoreset}): worst {worst:.2e}')
