"""Policy/value model object for the B200 PPO path.

Mirrors the call surface of the reference's ``ModelA2CContinuousLogStd.Network`` (models.py:304-364)
wrapped around ``A2CBuilder.Network`` (network_builder.py:211-593) for the subset on the hot path:
MLP trunk, continuous head with a fixed (``fixed_sigma: True``) or state-dependent (``fixed_sigma: False``) sigma in any of the
reference's sigma parametrisations, scalar value head, optional obs / value ``RunningMeanStd`` normalisers.

All parameters live in ONE flat fp32 arena (``self.flat``) with matching flat gradient / Adam-moment
arenas, so the optimiser, the gradient all-reduce and the checkpoint code each touch one buffer:

    [ sigma(A) | W_1 | b_1 | ... | W_L | b_L | W_head(A+1, H_L) | b_head(A+1) ]   (row 0 of the head = value)

An LSTM adds ``W_ih | W_hh | b_ih | b_hh`` after ``sigma``, and with ``rnn.layer_norm`` its LayerNorm's ``ln_w | ln_b`` after those.
A state-dependent sigma head (``fixed_sigma: False``) is A more head rows, ``W_head(1+2A, H_L) | b_head(1+2A)`` = (value, mu, sigma);
the leading ``sigma(A)`` block then stays in the arena as dead space that is always exactly zero (no state-dict key, no Adam state,
no gradient), so every offset convention of the fixed-sigma layout holds for both.

``state_dict()`` / ``load_state_dict()`` speak the reference's key names
(``a2c_network.sigma``, ``a2c_network.actor_mlp.{0,2,..}.{weight,bias}``, ``a2c_network.value.*``,
``a2c_network.mu.*``, ``running_mean_std.*``, ``value_mean_std.*``) so checkpoints interoperate with the
reference trainer and players.

``FlatParamModel`` owns what every flat-arena network shares -- the layout, ``view()``, the state dicts and the torch Adam state
dict -- for ``B200Model`` and for the discrete model (agent_discrete.py) and the central value net (agent_cv.py), which only define
their layouts and key names.
"""
import math
from collections import OrderedDict

import torch

from . import ops
from .layerwise import Layer


def _apply_init(t, spec, fan_in):
    """network_builder.py:61-72 init_factory for the names used by shipped configs."""
    name = (spec or {}).get('name', 'default')
    kw = {k: v for k, v in (spec or {}).items() if k != 'name'}
    if name == 'default':
        bound = 1.0 / math.sqrt(fan_in)      # torch.nn.Linear default: kaiming_uniform_(a=sqrt(5))
        t.uniform_(-bound, bound)
    elif name == 'const_initializer':
        t.fill_(kw.get('val', kw.get('value', 0)))
    elif name in ('orthogonal_initializer', 'orthogonal'):
        torch.nn.init.orthogonal_(t, **kw)
    elif name == 'glorot_normal_initializer':
        torch.nn.init.xavier_normal_(t, **kw)
    elif name == 'glorot_uniform_initializer':
        torch.nn.init.xavier_uniform_(t, **kw)
    elif name == 'random_uniform_initializer':
        torch.nn.init.uniform_(t, **kw)
    elif name == 'kaiming_normal':
        torch.nn.init.kaiming_normal_(t, **kw)
    elif name == 'variance_scaling_initializer':
        # torch_ext.py:114-144 (configs/mujoco/halfcheetah*.yaml): N(0, scale / fan) by inverse CDF of uniforms drawn from NUMPY's global
        # generator (the one the runner seeds), restricted to [-2, 2] in ABSOLUTE units -- not in sigmas -- and clamped there
        import numpy as np
        sigma = math.sqrt(kw.get('scale', 2.0) / torch.nn.init._calculate_correct_fan(t, kw.get('mode', 'fan_in')))
        u = torch.from_numpy(np.random.uniform(0, 1, tuple(t.shape)))
        std_normal = torch.distributions.Normal(0.0, 1.0, validate_args=False)
        lo = std_normal.cdf(torch.tensor(-2.0 / sigma, dtype=torch.float64))
        hi = std_normal.cdf(torch.tensor(2.0 / sigma, dtype=torch.float64))
        eps = torch.finfo(torch.float64).eps
        z = (2.0 * (lo + (hi - lo) * u) - 1.0).clamp(-1.0 + eps, 1.0 - eps)
        t.copy_((sigma * math.sqrt(2.0) * torch.erfinv(z)).clamp(-2.0, 2.0))
    else:
        raise ValueError(f'unsupported initializer {name}')


class _RunningStats:
    """Device-resident RunningMeanStd state (running_mean_std.py:19-53): fp64 mean/var, int64 count,
    plus the fp32 (mean, sqrt(var+eps)) copies the fused kernels read."""

    def __init__(self, size, device):
        self.size = size
        self.running_mean = torch.zeros(size, dtype=torch.float64, device=device)
        self.running_var = torch.ones(size, dtype=torch.float64, device=device)
        self.count = torch.ones(1, dtype=torch.int64, device=device)
        self.mean_f32 = torch.zeros(size, dtype=torch.float32, device=device)
        self.std_f32 = torch.ones(size, dtype=torch.float32, device=device)
        self.refresh()

    def refresh(self):
        ops.refresh_norm(self.running_mean, self.running_var, self.mean_f32, self.std_f32)

    @staticmethod
    def f32_pair(stats):
        """(mean_f32, std_f32) of `stats`, the `norm` operands of the kernels; (None, None) without a normaliser"""
        return (None, None) if stats is None else (stats.mean_f32, stats.std_f32)

    def state_dict(self, prefix):
        return OrderedDict([(prefix + 'running_mean', self.running_mean.clone()),
                            (prefix + 'running_var', self.running_var.clone()),
                            (prefix + 'count', self.count.reshape(()).clone())])

    def load_state_dict(self, sd, prefix=''):
        self.running_mean.copy_(sd[prefix + 'running_mean'].reshape(-1))
        self.running_var.copy_(sd[prefix + 'running_var'].reshape(-1))
        self.count.copy_(sd[prefix + 'count'].reshape(-1))
        self.refresh()

    def __call__(self, x, denorm=False):
        """Eval-mode forward (running_mean_std.py:104-113)."""
        return ops.normalize(x, self.running_mean, self.running_var, denorm=denorm)


def check_network_params(network_params):
    """Options of A2CBuilder.Network.load (network_builder.py:545-589) that change the maths and have no kernel here must fail loudly,
    never be ignored: a config that sets them would otherwise train a different network without a word."""
    name = network_params.get('name', 'actor_critic')
    if name != 'actor_critic':
        raise NotImplementedError(f"network '{name}': only 'actor_critic' (A2CBuilder) is on the B200 hot path")
    mlp = network_params['mlp']
    if mlp.get('d2rl', False):
        raise NotImplementedError('mlp.d2rl')
    if network_params.get('normalization', None) not in (None, 'None'):
        raise NotImplementedError(f"normalization: {network_params['normalization']} (layer_norm / batch_norm inside the MLP)")
    if network_params.get('joint_obs_actions', None) is not None:
        raise NotImplementedError('joint_obs_actions')
    # mlp.regularizer is read by no code path of the reference's torch builder either: ignored there, ignored here


class _NetworkView:
    """What Runner._override_sigma (torch_runner.py:52-60) touches: ``a2c_network.sigma`` / ``fixed_sigma``."""

    def __init__(self, model):
        self._m = model
        self.fixed_sigma = model.fixed_sigma

    @property
    def sigma(self):
        return self._m.sigma

    def is_rnn(self):
        return self._m.rnn_units > 0


def resolve_device(name):
    """torch.device for a config's `device` value.  An index-less 'cuda' (configs/ppo_cartpole.yaml, ppo_lunar_discrete.yaml) means the
    CURRENT device, as every torch op resolves it; it is made explicit here because raw pointers cross the C ABI and
    `torch.cuda.set_device` refuses a device without an index.  Anything else is returned as torch parses it."""
    dev = torch.device(name)
    if dev.type == 'cuda' and dev.index is None:
        dev = torch.device('cuda', torch.cuda.current_device())
    return dev


class CompileTolerantModel:
    """Mixin for agents: `Runner.run_train` of the reference wraps `agent.model` with torch.compile unless the YAML says
    `torch_compile: False` (torch_runner.py:282-312).  There is no nn.Module to compile here (the hand-written kernels subsume those
    fusions), so an assignment of anything that is not one of this package's models is ignored, once, with a note -- stock YAMLs
    run unchanged through the reference's own Runner."""

    @property
    def model(self):
        return self.__dict__.get('_b200_model')

    @model.setter
    def model(self, m):
        if self.__dict__.get('_b200_model') is not None and not hasattr(m, 'load_optimizer_state_dict'):
            if not self.__dict__.get('_b200_compile_noted'):
                print('b200: torch.compile of agent.model ignored (no nn.Module on this path; set torch_compile: False to silence)')
                self.__dict__['_b200_compile_noted'] = True
            return
        self.__dict__['_b200_model'] = m


def _model_call(self, *args, **kwargs):
    raise NotImplementedError('the B200 model is a flat parameter arena driven by fused kernels (agent.get_action_values / train_epoch); '
                              'it has no module-style forward')


class FlatParamModel:
    """All parameters of a network in ONE flat fp32 arena (``flat``) with matching Adam-moment arenas (``exp_avg``, ``exp_avg_sq``),
    laid out from an ordered ``(name, shape)`` list.  Subclasses define ``param_names()`` and ``_param_views(arena)``: the reference's
    state-dict keys and the matching views, in the reference's ``model.parameters()`` order, which is also the index order of the
    torch Adam state.  They also set ``device``, ``normalize_input`` / ``normalize_value`` and ``running_mean_std`` /
    ``value_mean_std``."""

    __call__ = _model_call

    # torch.optim.Adam param-group keys written after lr / betas / eps / weight_decay
    ADAM_GROUP_EXTRA = {'amsgrad': False, 'maximize': False, 'foreach': None, 'capturable': False, 'differentiable': False, 'fused': True,
                        'decoupled_weight_decay': False}

    def _init_arena(self, sizes, align=1):
        """layout[name] = (offset, shape); every tensor starts on a multiple of `align` elements"""
        self.layout, off = OrderedDict(), 0
        for n, shp in sizes:
            off = (off + align - 1) // align * align
            self.layout[n] = (off, shp)
            off += int(torch.Size(shp).numel())
        self.num_params = off
        self.flat = torch.zeros(off, dtype=torch.float32, device=self.device)
        self.exp_avg = torch.zeros_like(self.flat)
        self.exp_avg_sq = torch.zeros_like(self.flat)

    def _init_linear_default(self):
        """torch.nn.Linear default weights (U(-1/sqrt(fan_in), 1/sqrt(fan_in)), drawn in layout order), zero biases"""
        for n, (o, shp) in self.layout.items():
            if n.startswith('W'):
                bound = 1.0 / float(shp[1]) ** 0.5
                self.view(n).uniform_(-bound, bound)

    def view(self, name, arena=None):
        off, shp = self.layout[name]
        arena = self.flat if arena is None else arena
        return arena[off:off + int(torch.Size(shp).numel())].view(shp)

    def state_dict(self):
        sd = OrderedDict()
        if self.normalize_value:
            sd.update(self.value_mean_std.state_dict('value_mean_std.'))
        if self.normalize_input:
            sd.update(self.running_mean_std.state_dict('running_mean_std.'))
        for n, v in zip(self.param_names(), self._param_views()):
            sd[n] = v.clone()
        return sd

    def load_state_dict(self, sd, strict=True):
        sd = {k.replace('_orig_mod.', ''): v for k, v in sd.items()}
        missing = [n for n in self.param_names() if n not in sd]
        if missing and strict:
            raise KeyError(f'missing keys in state_dict: {missing}')
        with torch.no_grad():
            for n, v in zip(self.param_names(), self._param_views()):
                if n in sd:
                    v.copy_(sd[n].reshape(v.shape))
            if self.normalize_value and 'value_mean_std.running_mean' in sd:
                self.value_mean_std.load_state_dict(sd, 'value_mean_std.')
            if self.normalize_input and 'running_mean_std.running_mean' in sd:
                self.running_mean_std.load_state_dict(sd, 'running_mean_std.')

    def optimizer_state_dict(self, lr, step, weight_decay):
        """torch.optim.Adam.state_dict() layout (index-keyed, reference parameter order)."""
        state = {i: {'step': torch.tensor(float(step)), 'exp_avg': m.clone(), 'exp_avg_sq': v.clone()}
                 for i, (m, v) in enumerate(zip(self._param_views(self.exp_avg), self._param_views(self.exp_avg_sq)))}
        group = {'lr': lr, 'betas': (0.9, 0.999), 'eps': 1e-08, 'weight_decay': weight_decay, **self.ADAM_GROUP_EXTRA,
                 'params': list(range(len(state)))}
        return {'state': state, 'param_groups': [group]}

    def load_optimizer_state_dict(self, osd):
        """Returns (lr, step); lr is None when the dict has no param group."""
        st, step = osd.get('state', {}), 0
        ms, vs = self._param_views(self.exp_avg), self._param_views(self.exp_avg_sq)
        for i in range(len(ms)):
            if i in st:
                ms[i].copy_(st[i]['exp_avg'].reshape(ms[i].shape))
                vs[i].copy_(st[i]['exp_avg_sq'].reshape(vs[i].shape))
                step = int(float(st[i]['step']))
        return (osd['param_groups'][0]['lr'] if osd.get('param_groups') else None), step


class B200Model(FlatParamModel):
    RNN_KEYS = ('a2c_network.rnn.rnn.weight_ih_l0', 'a2c_network.rnn.rnn.weight_hh_l0', 'a2c_network.rnn.rnn.bias_ih_l0',
                'a2c_network.rnn.rnn.bias_hh_l0')
    LN_KEYS = ('a2c_network.layer_norm.weight', 'a2c_network.layer_norm.bias')

    def __init__(self, network_params, obs_dim, act_dim, device, normalize_input, normalize_value, value_size=1,
                 seed=None):
        if value_size != 1:
            raise NotImplementedError('value_size > 1 is not on the B200 hot path yet')
        check_network_params(network_params)
        mlp = network_params['mlp']
        self.units = list(mlp['units'])
        if len(self.units) == 0:
            raise NotImplementedError('empty MLP')
        self.activation = mlp.get('activation', 'elu')
        if self.activation not in ops.ACT:
            raise NotImplementedError(f'activation {self.activation}')
        self.act_id = ops.ACT[self.activation]
        # separate: True (network_builder.py:494-512; configs/ppo_continuous.yaml, ppo_lunar.yaml ...): actor_mlp feeds mu, critic_mlp feeds the
        # value.  Here the two trunks are ONE MLP of twice the width whose weights are block-structured -- layer 0 stacks [W_actor; W_critic] (both
        # read the observation), layers >= 1 are block-diagonal, the value row of the head reads the critic half and the mu rows the actor half --
        # so every kernel, arena and code path of the shared-trunk policy is used as it is.  The structural zeros stay exactly zero: their
        # gradient entries are masked before the optimiser (grad_mask), and a zero weight with a zero gradient is a fixed point of Adam and of
        # weight decay; multiplied by zero they add exact zeros to the products.  `units` = the EFFECTIVE widths everything downstream sees,
        # `trunk_units` = the reference's per-trunk widths (state-dict shapes).
        self.separate = bool(network_params.get('separate', False))
        self.trunk_units = list(self.units)
        if self.separate:
            if 'rnn' in network_params:
                raise NotImplementedError('separate actor/critic trunks with an rnn (two recurrent cores) are not on the B200 hot path')
            self.units = [2 * u for u in self.trunk_units]
        if 'cnn' in network_params:
            raise NotImplementedError("'cnn' networks are not on the B200 hot path yet")
        self.rnn_units = 0
        if 'rnn' in network_params:
            rnn = network_params['rnn']
            if rnn.get('name') != 'lstm' or rnn.get('layers', 1) != 1 \
                    or rnn.get('concat_input', False) or rnn.get('concat_output', False):
                raise NotImplementedError("rnn: only a single-layer 'lstm' (optionally layer-normed; no concat) is on the B200 hot path")
            self.rnn_units = int(rnn['units'])
        # rnn.layer_norm (network_builder.py:279-280, :485-486): LayerNorm(rnn_units) of the LSTM output rows; the carried (h, c) stay raw
        self.rnn_layer_norm = bool(self.rnn_units and network_params['rnn'].get('layer_norm', False))
        # placement (network_builder.py:253-272): before_mlp True = obs -> LSTM -> MLP -> heads (BASELINE configs[3]); False (the reference
        # default) = obs -> MLP -> LSTM -> heads.  Same parameter names and order either way, different shapes.
        self.rnn_before_mlp = bool(network_params.get('rnn', {}).get('before_mlp', False)) if self.rnn_units else True
        space = network_params['space']['continuous']
        # fixed_sigma: False (network_builder.py:324-348, :441-444): sigma = Linear(H_L, A) of the trunk output, one std per row
        self.fixed_sigma = bool(space.get('fixed_sigma', True))
        if not self.fixed_sigma:
            if self.separate:
                raise NotImplementedError('state-dependent sigma with separate actor/critic trunks is not on the B200 hot path')
            if 'rnn' in network_params:
                raise NotImplementedError('state-dependent sigma with an rnn is not on the B200 hot path')
        for k in ('mu_activation', 'sigma_activation'):
            if space.get(k, 'None') not in ('None', None):
                raise NotImplementedError(f'{k}={space[k]}')
        # models.py:272-302 apply_sigma_parametrization: 'exp' (clamped to logstd_bounds, floored by min_sigma), 'softplus', 'linear'
        # (alias 'scalar'); configs/mjlab/ppo_lift_cube_yam.yaml: exp + min_sigma 0.15, ppo_wujihand_reorient.yaml: softplus + 0.2
        self.sigma_parametrization = space.get('sigma_parametrization', 'exp')
        if self.sigma_parametrization not in ops.SIGMA_PARAM:
            raise NotImplementedError(f'sigma_parametrization {self.sigma_parametrization}')
        self.min_sigma = float(space.get('min_sigma', 0.0) or 0.0)
        bounds = space.get('logstd_bounds', None)
        self.logstd_bounds = (float(bounds[0]), float(bounds[1])) if bounds is not None and self.sigma_parametrization == 'exp' else None
        self.sigma_cfg = ops.sigma_cfg(self.sigma_parametrization, self.min_sigma, self.logstd_bounds)
        # a fixed sigma that is not the plain log-std is mapped outside the kernels (refresh_sigma_floor)
        self.sigma_transform = self.fixed_sigma and (self.sigma_parametrization != 'exp' or self.min_sigma > 0 or self.logstd_bounds is not None)
        self.head_rows = int(act_dim) + 1 if self.fixed_sigma else 1 + 2 * int(act_dim)      # (value, mu[, sigma]) rows of W_head
        if network_params.get('value_activation', 'None') not in ('None', None):
            raise NotImplementedError('value_activation')
        self.D, self.A = int(obs_dim), int(act_dim)
        self.device = torch.device(device)
        self.normalize_input, self.normalize_value = bool(normalize_input), bool(normalize_value)
        # ---- flat arenas ----
        sizes = [('sigma', (self.A,))]
        Hd = self.rnn_units
        self.rnn_in = (self.D if self.rnn_before_mlp else self.units[-1]) if Hd else 0      # input width of the LSTM
        if Hd:
            sizes += [('W_ih', (4 * Hd, self.rnn_in)), ('W_hh', (4 * Hd, Hd)), ('b_ih', (4 * Hd,)), ('b_hh', (4 * Hd,))]
            if self.rnn_layer_norm:
                sizes += [('ln_w', (Hd,)), ('ln_b', (Hd,))]
        ins = Hd if (Hd and self.rnn_before_mlp) else self.D
        for i, u in enumerate(self.units):
            sizes += [(f'W{i}', (u, ins)), (f'b{i}', (u,))]
            ins = u
        if Hd and not self.rnn_before_mlp:
            ins = Hd                     # the heads read the LSTM output
        self.Hl = ins
        sizes += [('W_head', (self.head_rows, ins)), ('b_head', (self.head_rows,))]
        # every tensor starts on an 8-element boundary (32 bytes in the fp32 arenas, 16 bytes in the bf16 twin the tensor-core GEMMs
        # read): weight rows can then be staged with 16-byte loads whatever the action count did to the offsets.  The gaps hold
        # zeros in every arena (weights, gradients, moments), so norms, Adam and the all-reduce are unaffected; layouts whose tensor
        # sizes are all multiples of 8 (the BASELINE MLPs with 8 actions) have no gaps at all.
        self._init_arena(sizes, align=8)
        off = self.num_params
        self.grad = torch.zeros(off, dtype=torch.float32, device=self.device)
        self.W = [self.view(f'W{i}') for i in range(len(self.units))]
        self.b = [self.view(f'b{i}') for i in range(len(self.units))]
        self.mlp = [Layer(self.W[i], self.b[i], self.layout[f'W{i}'][0], self.layout[f'b{i}'][0], self.act_id) for i in range(len(self.units))]
        self.sigma = self.view('sigma')
        if self.sigma_transform:
            # what the kernels are handed instead of the raw parameter, and the chain factor of its gradient (refresh_sigma_floor)
            self.logstd_eff = torch.zeros(self.A, dtype=torch.float32, device=self.device)
            self.sigma_chain = torch.ones(self.A, dtype=torch.float32, device=self.device)
        if self.rnn_units:
            self.W_ih, self.W_hh, self.b_ih, self.b_hh = (self.view(n) for n in ('W_ih', 'W_hh', 'b_ih', 'b_hh'))
        self.ln_w = self.view('ln_w') if self.rnn_layer_norm else None
        self.ln_b = self.view('ln_b') if self.rnn_layer_norm else None
        self.mlp_in = self.rnn_units if (self.rnn_units and self.rnn_before_mlp) else self.D
        self.W_head, self.b_head = self.view('W_head'), self.view('b_head')
        self.grad_mask = None
        if self.separate:       # 1 on the entries the reference has a parameter for, 0 on the structural zeros of the block layout
            self.grad_mask = torch.zeros(off, dtype=torch.float32, device=self.device)
            for v in self._param_views(self.grad_mask):
                v.fill_(1.0)
        self.g_sigma = self.view('sigma', self.grad)
        self.running_mean_std = _RunningStats(self.D, self.device) if self.normalize_input else None
        self.value_mean_std = _RunningStats(1, self.device)   # always allocated; used iff normalize_value
        self.a2c_network = _NetworkView(self)
        self._init_weights(network_params, seed)
        self.training = False

    # -------------------------------------------------------------------------------------------
    @property
    def logstd_in(self):
        """The log-std vector the fixed-sigma policy kernels read.  They compute sigma = exp(logstd) -- for any sigma other than the
        plain log-std (a floor, bounds, 'softplus' / 'linear') that is the EFFECTIVE log-std log(sigma(raw)) (models.py:272-302), kept
        in its own buffer by refresh_sigma_floor(); otherwise it is the parameter itself."""
        return self.logstd_eff if self.sigma_transform else self.sigma

    def refresh_sigma_floor(self):
        """After anything that changes the raw fixed sigma parameter (optimiser step, weight load): logstd_eff = log(sigma(raw)) and
        sigma_chain = d logstd_eff / d raw, the factor that turns the kernels' gradient with respect to the log-std they were handed
        into the gradient of the raw parameter.  In-place launches on [A] vectors (CUDA-graph capturable); a no-op for the plain
        log-std and for a state-dependent head, whose kernels apply the parametrisation per row."""
        if not self.sigma_transform:
            return
        if self.sigma_parametrization == 'exp' and self.logstd_bounds is None:     # exp(raw) + min_sigma
            torch.exp(self.sigma, out=self.sigma_chain)
            torch.add(self.sigma_chain, self.min_sigma, out=self.logstd_eff)
            self.sigma_chain.div_(self.logstd_eff)
            self.logstd_eff.log_()
            return
        raw = self.sigma
        if self.sigma_parametrization == 'exp':
            lo, hi = self.logstd_bounds
            g = ((raw >= lo) & (raw <= hi)).float()             # torch.clamp's gradient: 1 on the closed interval
            rc = raw.clamp(lo, hi)
            if self.min_sigma > 0:
                e = rc.exp()
                torch.add(e, self.min_sigma, out=self.logstd_eff)
                torch.mul(e, g, out=self.sigma_chain)
                self.sigma_chain.div_(self.logstd_eff)
                self.logstd_eff.log_()
            else:
                self.logstd_eff.copy_(rc)
                self.sigma_chain.copy_(g)
            return
        floor_ = max(self.min_sigma, 1e-3) if self.sigma_parametrization in ('linear', 'scalar') else self.min_sigma
        x = raw - floor_ if self.sigma_parametrization in ('linear', 'scalar') else raw
        torch.add(torch.nn.functional.softplus(x), floor_, out=self.logstd_eff)        # sigma
        z = x.exp()
        torch.where(x > 20.0, torch.ones_like(x), z / (z + 1.0), out=self.sigma_chain)  # softplus' (threshold 20)
        self.sigma_chain.div_(self.logstd_eff)
        self.logstd_eff.log_()

    def _init_weights(self, network_params, seed):
        """network_builder.py:326-348: mlp initializer on every Linear weight, zero biases, mu_init on mu.weight,
        sigma_init on the sigma parameter."""
        space = network_params['space']['continuous']
        mlp_init = network_params['mlp'].get('initializer', {'name': 'default'})
        cpu = {}
        if self.rnn_units:   # torch.nn.LSTM default init U(-1/sqrt(hid), 1/sqrt(hid)) for all four tensors (mlp_init does not touch it)
            Hd = self.rnn_units
            k = 1.0 / math.sqrt(Hd)
            for n, shp in (('W_ih', (4 * Hd, self.rnn_in)), ('W_hh', (4 * Hd, Hd)), ('b_ih', (4 * Hd,)), ('b_hh', (4 * Hd,))):
                cpu[n] = torch.empty(*shp).uniform_(-k, k)
            if self.rnn_layer_norm:      # torch.nn.LayerNorm's own init; the mlp initializer does not touch it
                cpu['ln_w'], cpu['ln_b'] = torch.ones(Hd), torch.zeros(Hd)
        mu_init = space.get('mu_init', {'name': 'default'})
        if self.separate:       # every Linear of both trunks and both heads is initialised on its own (true fan-in), written into its block
            blocks = self._param_views(self.flat)[1:]               # actor W, b ... critic W, b ... value W, b, mu W, b
            for k in range(0, len(blocks), 2):
                w = torch.empty(*blocks[k].shape)
                _apply_init(w, mlp_init, w.shape[1])
                if k == len(blocks) - 2 and mu_init.get('name', 'default') != 'default':
                    _apply_init(w, mu_init, w.shape[1])
                blocks[k].copy_(w)
        else:
            ins = self.mlp_in
            for i, u in enumerate(self.units):
                w = torch.empty(u, ins)
                _apply_init(w, mlp_init, ins)
                cpu[f'W{i}'] = w
                ins = u
            ins = self.Hl
            A = self.A
            wh = torch.empty(self.head_rows, ins)
            _apply_init(wh[:1], mlp_init, ins)                                   # value head: mlp_init
            _apply_init(wh[1:A + 1], mlp_init, ins)
            if mu_init.get('name', 'default') != 'default':
                _apply_init(wh[1:A + 1], mu_init, ins)
            sigma_init = space.get('sigma_init', {'name': 'const_initializer', 'val': 0})
            if not self.fixed_sigma:
                # network_builder.py:14-25 init_state_dependent_sigma_head, after the mlp_init pass over every Linear: a const
                # initializer writes the bias and zeroes the weight, anything else initialises the weight (bias stays zero)
                _apply_init(wh[A + 1:], mlp_init, ins)
                if sigma_init.get('name') == 'const_initializer':
                    wh[A + 1:].zero_()
                    cpu['b_head'] = torch.zeros(self.head_rows)
                    cpu['b_head'][A + 1:] = float(sigma_init.get('val', 0.0))
                else:
                    _apply_init(wh[A + 1:], sigma_init, ins)
            cpu['W_head'] = wh
        if self.fixed_sigma:
            sg = torch.empty(self.A)
            _apply_init(sg, space.get('sigma_init', {'name': 'const_initializer', 'val': 0}), 1)
            cpu['sigma'] = sg
        for n, t in cpu.items():
            self.view(n).copy_(t)

    # ------------------------------------------------------------------------------------------- nn.Module-ish
    def is_rnn(self):
        return self.rnn_units > 0

    def get_default_rnn_state(self, num_seqs=1):
        """network_builder.py:520-543 (lstm, not separate): (h, c) each [layers, num_seqs, units]"""
        if not self.rnn_units:
            return None
        return (torch.zeros((1, num_seqs, self.rnn_units), device=self.device), torch.zeros((1, num_seqs, self.rnn_units), device=self.device))

    def get_aux_loss(self):
        return None

    def eval(self):
        self.training = False
        return self

    def train(self, mode=True):
        self.training = mode
        return self

    def to(self, device):
        return self

    def parameters(self):
        """Reference parameter order (optimizer state is index-keyed): sigma, actor_mlp.*, [rnn.rnn.*, layer_norm.*], value.*, mu.* (state-dependent head:
        actor_mlp.*, value.*, mu.*, sigma.weight, sigma.bias)"""
        return self._param_views(self.flat)

    def _param_views(self, arena=None):
        if self.separate:
            return self._param_views_separate(arena)
        out = [self.view('sigma', arena)]
        for i in range(len(self.units)):
            out += [self.view(f'W{i}', arena), self.view(f'b{i}', arena)]
        if self.rnn_units:   # registration order in A2CBuilder.Network.__init__: actor_mlp placeholder precedes self.rnn
            out += [self.view(n, arena) for n in ('W_ih', 'W_hh', 'b_ih', 'b_hh')]
            if self.rnn_layer_norm:      # self.layer_norm is registered right after self.rnn
                out += [self.view('ln_w', arena), self.view('ln_b', arena)]
        wh, bh = self.view('W_head', arena), self.view('b_head', arena)
        A = self.A
        out += [wh[:1], bh[:1], wh[1:A + 1], bh[1:A + 1]]
        if not self.fixed_sigma:        # a Linear sigma head is registered after mu; the leading sigma block is dead space
            out = out[1:] + [wh[A + 1:], bh[A + 1:]]
        return out

    def _param_views_separate(self, arena):
        """separate: True -- the reference's parameters (order: sigma, actor_mlp.*, critic_mlp.*, value.*, mu.*) as block views of the
        double-width layout: trunk t of layer i owns rows [t u_i, (t + 1) u_i); layer 0 reads all observation columns, layers >= 1 the
        columns [t u_(i-1), (t + 1) u_(i-1)) of their own trunk; value = head row 0 on the critic half, mu = head rows 1.. on the actor half"""
        tu = self.trunk_units
        out = [self.view('sigma', arena)]
        for t in (0, 1):
            for i, u in enumerate(tu):
                w, b = self.view(f'W{i}', arena), self.view(f'b{i}', arena)
                cols = slice(None) if i == 0 else slice(t * tu[i - 1], (t + 1) * tu[i - 1])
                out += [w[t * u:(t + 1) * u, cols], b[t * u:(t + 1) * u]]
        wh, bh = self.view('W_head', arena), self.view('b_head', arena)
        out += [wh[:1, tu[-1]:], bh[:1], wh[1:, :tu[-1]], bh[1:]]
        return out

    def param_names(self):
        """state-dict keys of _param_views, in the same order: sigma, actor_mlp.*, [critic_mlp.*], [rnn.*], [layer_norm.*], value.*, mu.*; a
        state-dependent head: actor_mlp.*, value.*, mu.*, sigma.weight, sigma.bias"""
        if not self.fixed_sigma:
            keys = [f'a2c_network.actor_mlp.{2 * i}.{t}' for i in range(len(self.trunk_units)) for t in ('weight', 'bias')]
            return keys + ['a2c_network.value.weight', 'a2c_network.value.bias', 'a2c_network.mu.weight', 'a2c_network.mu.bias',
                           'a2c_network.sigma.weight', 'a2c_network.sigma.bias']
        keys = ['a2c_network.sigma']
        for trunk in (('actor_mlp', 'critic_mlp') if self.separate else ('actor_mlp',)):
            for i in range(len(self.trunk_units)):
                keys += [f'a2c_network.{trunk}.{2 * i}.weight', f'a2c_network.{trunk}.{2 * i}.bias']
        if self.rnn_units:
            keys += list(self.RNN_KEYS)
        if self.rnn_layer_norm:
            keys += list(self.LN_KEYS)
        return keys + ['a2c_network.value.weight', 'a2c_network.value.bias', 'a2c_network.mu.weight', 'a2c_network.mu.bias']

    def load_state_dict(self, sd, strict=True):
        """strict: the normaliser statistics are required as well"""
        sd = {k.replace('_orig_mod.', ''): v for k, v in sd.items()}
        missing = [k for k in self.state_dict() if k not in sd]
        if missing and strict:
            raise KeyError(f'missing keys in state_dict: {missing}')
        super().load_state_dict(sd, strict=False)
