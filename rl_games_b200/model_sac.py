"""SAC model (models.py ModelSACContinuous around network_builder.py SACBuilder.Network) as flat fp32 parameter arenas.

Four parts, each one contiguous fp32 buffer with matching gradient and Adam-moment buffers:

    actor          [ W_0 | b_0 | ... | W_L | b_L ]            trunk MLP, then Linear(H, 2A) = (mu, raw log_std)
    critic         [ Q1: W_0 | b_0 | ... | W_L | b_L | Q2: same ]   each on [obs | action], output 1
    critic_target  same layout as critic, initialised as a copy
    log_alpha      one float

The state-dict keys are the reference's: ``sac_network.actor.trunk.{0,2,..}.{weight,bias}``, ``sac_network.critic.Q{1,2}.*``,
``sac_network.critic_target.Q{1,2}.*`` and ``running_mean_std.*`` with ``normalize_input``.  The parameter order of each part is
its ``parameters()`` order, which is also the index order of the reference's three Adam states (actor, critic, log_alpha).
"""
import math
from collections import OrderedDict

import torch

from . import ops
from .model import _RunningStats, _apply_init, _model_call


class _Arena:
    """one network part: flat parameters + gradients + Adam moments, laid out from an ordered (name, shape) list"""

    def __init__(self, sizes, device):
        self.layout, off = OrderedDict(), 0
        for n, shp in sizes:
            self.layout[n] = (off, shp)
            off += int(torch.Size(shp).numel())
        self.n = off
        self.flat = torch.zeros(off, dtype=torch.float32, device=device)
        self.grad = torch.zeros_like(self.flat)
        self.exp_avg = torch.zeros_like(self.flat)
        self.exp_avg_sq = torch.zeros_like(self.flat)

    def view(self, name, arena=None):
        off, shp = self.layout[name]
        arena = self.flat if arena is None else arena
        return arena[off:off + int(torch.Size(shp).numel())].view(shp)

    def views(self, arena=None):
        return [self.view(n, arena) for n in self.layout]


def _mlp_sizes(prefix, d_in, units, d_out):
    sizes, k, i = [], d_in, 0
    for u in list(units) + [d_out]:
        sizes += [(f'{prefix}{i}.weight', (u, k)), (f'{prefix}{i}.bias', (u,))]
        k, i = u, i + 2
    return sizes


def check_sac_network_params(network_params):
    """SACBuilder.Network.load options that change the maths and have no kernel here raise; nothing is silently ignored"""
    name = network_params.get('name', 'soft_actor_critic')
    if name != 'soft_actor_critic':
        raise NotImplementedError(f"network '{name}': only 'soft_actor_critic' (SACBuilder) is on the B200 SAC path")
    if 'cnn' in network_params:
        raise NotImplementedError("'cnn' networks are not supported by the SAC agent")
    if not network_params.get('separate', True):
        raise NotImplementedError("SAC 'separate: False' (the reference builds no critic without it)")
    mlp = network_params['mlp']
    if mlp.get('d2rl', False):
        raise NotImplementedError('mlp.d2rl')
    if network_params.get('normalization', None) not in (None, 'None'):
        raise NotImplementedError(f"normalization: {network_params['normalization']} (layer_norm / batch_norm inside the MLP)")
    if network_params.get('log_std_bounds') is None:
        raise NotImplementedError('SAC needs log_std_bounds (the reference actor unpacks it)')
    if mlp.get('activation', 'relu') not in ops.ACT:
        raise NotImplementedError(f"mlp activation '{mlp.get('activation')}'")


class SACModel:
    """Flat-arena SAC networks; ``actor`` / ``critic`` / ``critic_target`` are `_Arena`s, ``log_alpha`` a one-element tensor"""

    __call__ = _model_call

    def __init__(self, network_params, obs_dim, act_dim, device, normalize_input, init_alpha):
        check_sac_network_params(network_params)
        self.device = device
        self.D, self.A = obs_dim, act_dim
        mlp = network_params['mlp']
        self.units = list(mlp['units'])
        self.act_id = ops.ACT[mlp.get('activation', 'relu')]
        self.initializer = mlp.get('initializer', {'name': 'default'})
        self.log_std_bounds = tuple(float(v) for v in network_params['log_std_bounds'])
        self.normalize_input = bool(normalize_input)
        self.n_layers = len(self.units) + 1
        self.actor = _Arena(_mlp_sizes('trunk.', obs_dim, self.units, 2 * act_dim), device)
        q = _mlp_sizes('Q1.', obs_dim + act_dim, self.units, 1) + _mlp_sizes('Q2.', obs_dim + act_dim, self.units, 1)
        self.critic = _Arena(q, device)
        self.critic_target = _Arena(q, device)
        self.log_alpha = torch.full((1,), math.log(init_alpha), dtype=torch.float32, device=device)
        self.log_alpha_grad = torch.zeros(1, dtype=torch.float32, device=device)
        self.log_alpha_m = torch.zeros(1, dtype=torch.float32, device=device)
        self.log_alpha_v = torch.zeros(1, dtype=torch.float32, device=device)
        self.running_mean_std = _RunningStats(obs_dim, device) if self.normalize_input else None
        self._init_weights()

    # ------------------------------------------------------------------------------------------------ init (SACBuilder.Network)
    def _init_weights(self):
        """torch.nn.Linear's own init in construction order (actor trunk + head, Q1, Q2 of the critic, then the target's twins, whose
        draws are overwritten by the copy), then the configured initializer on every weight in module order and zero biases"""
        name = (self.initializer or {}).get('name', 'default')
        parts = [self.actor, self.critic, self.critic_target]
        with torch.no_grad():
            for p in parts:
                for n in p.layout:
                    if n.endswith('.weight'):
                        w = torch.empty(p.layout[n][1], dtype=torch.float32)
                        torch.nn.init.kaiming_uniform_(w, a=math.sqrt(5))
                        bound = 1.0 / math.sqrt(w.shape[1])
                        torch.empty(w.shape[0]).uniform_(-bound, bound)      # the bias draw, zeroed below
                        p.view(n).copy_(w)
            self.critic_target.flat.copy_(self.critic.flat)
            if name != 'default':                       # the reference's 'default' initializer is the identity: Linear's init stays
                for p in parts:
                    for n in p.layout:
                        if n.endswith('.weight'):
                            w = p.view(n).cpu()
                            _apply_init(w, self.initializer, w.shape[1])
                            p.view(n).copy_(w)
            for p in parts:
                for n in p.layout:
                    if n.endswith('.bias'):
                        p.view(n).zero_()

    # ------------------------------------------------------------------------------------------------ layer views
    def layers(self, arena, prefix=''):
        """[(W, b)] of one MLP: prefix '' = the actor trunk, 'Q1.' / 'Q2.' = a critic"""
        pre = 'trunk.' if prefix == '' else prefix
        return [(arena.view(f'{pre}{2 * i}.weight'), arena.view(f'{pre}{2 * i}.bias')) for i in range(self.n_layers)]

    # ------------------------------------------------------------------------------------------------ state dicts
    def part_state_dict(self, part):
        return OrderedDict((n, v.clone()) for n, v in zip(part.layout, part.views()))

    def load_part_state_dict(self, part, sd):
        sd = {k.replace('_orig_mod.', ''): v for k, v in sd.items()}
        missing = [n for n in part.layout if n not in sd]
        if missing:
            raise KeyError(f'missing keys in state_dict: {missing}')
        with torch.no_grad():
            for n, v in zip(part.layout, part.views()):
                v.copy_(sd[n].reshape(v.shape))

    def state_dict(self):
        """the reference's ModelSACContinuous.Network.state_dict() keys"""
        sd = OrderedDict()
        if self.normalize_input:
            sd.update(self.running_mean_std.state_dict('running_mean_std.'))
        for pname, part in (('actor', self.actor), ('critic', self.critic), ('critic_target', self.critic_target)):
            for n, v in zip(part.layout, part.views()):
                sd[f'sac_network.{pname}.{n}'] = v.clone()
        return sd

    def load_state_dict(self, sd, strict=True):
        for pname, part in (('actor', self.actor), ('critic', self.critic), ('critic_target', self.critic_target)):
            self.load_part_state_dict(part, {k[len(f'sac_network.{pname}.'):]: v for k, v in sd.items() if k.startswith(f'sac_network.{pname}.')})
        if self.normalize_input and 'running_mean_std.running_mean' in sd:
            self.running_mean_std.load_state_dict(sd, 'running_mean_std.')

    @staticmethod
    def adam_state_dict(ms, vs, step, lr, betas):
        """torch.optim.Adam(fused=True).state_dict() for parameters whose moments are the views ms / vs"""
        state = {i: {'step': torch.tensor(float(step)), 'exp_avg': m.detach().cpu().clone(), 'exp_avg_sq': v.detach().cpu().clone()}
                 for i, (m, v) in enumerate(zip(ms, vs))} if step > 0 else {}
        group = {'lr': lr, 'betas': tuple(betas), 'eps': 1e-08, 'weight_decay': 0, 'amsgrad': False, 'maximize': False, 'foreach': None,
                 'capturable': False, 'differentiable': False, 'fused': True, 'decoupled_weight_decay': False, 'params': list(range(len(ms)))}
        return {'state': state, 'param_groups': [group]}

    @staticmethod
    def load_adam_state_dict(ms, vs, osd):
        """returns the step count of the loaded state (0 when it holds none)"""
        st, step = osd.get('state', {}), 0
        for i in range(len(ms)):
            if i in st:
                ms[i].copy_(st[i]['exp_avg'].reshape(ms[i].shape))
                vs[i].copy_(st[i]['exp_avg_sq'].reshape(vs[i].shape))
                step = int(float(st[i]['step']))
        return step

    def eval(self):
        return self

    def train(self, mode=True):
        return self

    def is_rnn(self):
        return False
