"""Golden runs of the REAL reference with a layer-normed LSTM (rnn.layer_norm: True; network_builder.py:279-280, :485-486).  Same
recipe as gen_golden.py (whose gen_agent it calls, with the LSTM fixtures' seq_length 4 and widths):

    python tests/golden/gen_golden_lstm_ln.py

writes tests/golden/agent_lstm_ln.pt (LSTM before the MLP), agent_lstm_ln_after.pt (after the MLP) and agent_lstm_ln_after_masked.pt
(after the MLP, next_step autoreset) (committed).  Each fixture records 'rnn_layer_norm': True.  Kept as a script of its own next to
gen_golden.py, whose groups it leaves unchanged: regenerate these fixtures with this script."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import gen_golden  # noqa: E402

_make_params = gen_golden.make_params


def _make_params_ln(*a, **kw):
    params = _make_params(*a, **kw)
    params['network']['rnn']['layer_norm'] = True
    return params


def _gen(name, **kw):
    gen_golden.make_params = _make_params_ln
    try:
        gen_golden.gen_agent(name, **kw)
    finally:
        gen_golden.make_params = _make_params
    path = os.path.join(gen_golden.HERE, name)
    g = torch.load(path, weights_only=False)
    assert 'a2c_network.layer_norm.weight' in g['init_state'], 'the reference built no LayerNorm'
    g['rnn_layer_norm'] = True
    torch.save(g, path)


def gen_lstm_ln():
    # the perturbation of gen_agent moves every bias (layer_norm.bias included) off zero; the LayerNorm weight starts at exactly one
    _gen('agent_lstm_ln.pt', seed=36, rnn_units=8, overrides={'seq_length': 4})
    _gen('agent_lstm_ln_after.pt', seed=37, rnn_units=12, rnn_before_mlp=False, overrides={'seq_length': 4})
    _gen('agent_lstm_ln_after_masked.pt', seed=38, rnn_units=12, rnn_before_mlp=False, autoreset='next_step', overrides={'seq_length': 4})


if __name__ == '__main__':
    gen_lstm_ln()
