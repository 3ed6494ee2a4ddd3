"""The CPU oracle (oracle/ppo_oracle.py) with rnn.layer_norm: True -- TEST INFRASTRUCTURE ONLY, kept beside the tests so that oracle/
stays as it is.  A2CBuilder.Network applies LayerNorm(rnn_units) to the LSTM output rows (network_builder.py:279-280, :485-486); the
carried (h, c) stay raw.  The parameters follow the reference's order: sigma, actor_mlp.*, rnn.rnn.*, layer_norm.*, value.*, mu.*."""
import torch
import torch.nn.functional as F

from oracle import ppo_oracle as O

LN_NAMES = ['a2c_network.layer_norm.weight', 'a2c_network.layer_norm.bias']


def param_names(n_layers):
    names = O.param_names(n_layers, lstm=True)
    i = names.index(O.RNN_NAMES[-1]) + 1
    return names[:i] + LN_NAMES + names[i:]


def init_params(obs_dim, units, act_dim, seed=0, rnn_units=8, rnn_before_mlp=True, ln_seed=None):
    """O.init_params plus the LayerNorm (torch's init: ones / zeros; ln_seed perturbs both so that neither is trivial)"""
    p = O.init_params(obs_dim, units, act_dim, seed=seed, rnn_units=rnn_units, rnn_before_mlp=rnn_before_mlp)
    p[LN_NAMES[0]], p[LN_NAMES[1]] = torch.ones(rnn_units), torch.zeros(rnn_units)
    if ln_seed is not None:
        g = torch.Generator().manual_seed(ln_seed)
        p[LN_NAMES[0]] += torch.randn(rnn_units, generator=g) * 0.1
        p[LN_NAMES[1]] += torch.randn(rnn_units, generator=g) * 0.1
    return {k: p[k] for k in param_names(len(units))}


class LnOracleModel(O.OracleModel):
    def forward(self, *a, **kw):
        plain = O.lstm_with_dones

        def ln_lstm(p, x, h, c, dones):
            out, h, c = plain(p, x, h, c, dones)
            return F.layer_norm(out, (out.shape[-1],), p[LN_NAMES[0]], p[LN_NAMES[1]], 1e-5), h, c
        O.lstm_with_dones = ln_lstm
        try:
            return super().forward(*a, **kw)
        finally:
            O.lstm_with_dones = plain


def make_agent(env, params, obs_dim, act_dim, units, num_actors, horizon, minibatch_size, cfg):
    """O.OracleAgent whose model is layer-normed; params must hold the LayerNorm tensors"""
    agent = O.OracleAgent(env, params, obs_dim, act_dim, units, num_actors, horizon, minibatch_size, cfg)
    agent.model.__class__ = LnOracleModel
    agent.model.names = param_names(len(units))
    agent.optimizer = O.Adam(agent.model.parameters(), agent.last_lr, eps=1e-8, weight_decay=agent.cfg['weight_decay'])
    return agent
