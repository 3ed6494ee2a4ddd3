"""Discrete-action PPO agent on the fp32 CUDA kernels -- SURVEY.md 8a row a15 (reference: algos_torch/a2c_discrete.py
DiscreteA2CAgent + common/a2c_common.py:1205-1359 DiscreteA2CBase, models.py:62-125 ModelA2C, network_builder.py A2CBuilder with a
``discrete`` space, optionally ``separate: True`` actor/critic trunks, optional action masks).

STATUS: parity-green on an H100 (``tests/test_discrete_gpu.py``) against a CPU oracle that is pinned to the reference
(oracle/ppo_discrete_oracle.py, tests/golden/agent_discrete*.pt).  Everything except the two categorical kernels
(csrc/discrete.cu) reuses the kernels of the continuous path: linear_fwd / linear_bwd_* / reduce_splits (mlp_simt.cu), gae_fused, prepare_batch, moments_update,
mask_inv_counts (stats.cu, gae.cu), post_step (rollout.cu), adam_step (adam.cu).

Image observations (``cnn: {type: conv2d}`` on a rank-3 Box) run a conv trunk (csrc/conv.cu) in front of the MLP; see DESIGN.md §4.
Precision is read by value: ``mixed_precision: True`` runs every conv and linear layer of the rollout and the update on the bf16
tensor cores (csrc/conv_tc.cu, csrc/gemm_tc.cu; the categorical head kernels stay fp32), with the weights read from ``wbf``, a bf16
twin of the parameter arena refreshed after every optimiser step, weight load and weight broadcast; ``False`` or no key runs the fp32
kernels above.
Scope of this first edition: one GPU, eager launches (no CUDA graph), flat Box observations or conv2d frames, ``Discrete(K)`` or multi-discrete
``Tuple(Discrete(K_j))`` action spaces (K_j <= 64, <= 8 heads), no RNN, no central value.  The scheduler steps once per MINI-EPOCH on the mean KL like the reference
(a2c_common.py:1265-1272), which costs one host sync per mini-epoch.

The agent derives from ``a2c_base.A2CBase`` (shared with the continuous agent) and adds the action space, the model, the arena, the
env plumbing, the rollout, the update and its resume semantics.
"""
import time

import numpy as np
import torch
import torch.distributed as dist

from . import layerwise, ops
from .a2c_base import A2CBase
from .common import make_summary_writer
from .layerwise import Layer
from .model import _apply_init, check_network_params, FlatParamModel, _RunningStats


def discrete_spaces(observation_space, action_space, network_params, config):
    """(obs_shape, obs_dtype, head_sizes, actions_num, is_multi_discrete, mixed_precision) of a discrete policy, or the refusal of its
    spaces; the agent and the player both take them from here"""
    # flat Box observations, or rank-3 frames in front of a cnn (the model checks the cnn); the arena keeps the env's dtype
    # (experience.py:376): uint8 frames stay bytes and are scaled by 1/255 where the first conv and the normaliser read them
    is_dict = type(observation_space).__name__ == 'Dict'
    if is_dict or len(observation_space.shape) != 1 and ('cnn' not in network_params or len(observation_space.shape) != 3):
        raise NotImplementedError('only flat Box observations')
    obs_shape = observation_space.shape
    obs_dtype = torch.uint8 if len(obs_shape) == 3 and np.dtype(observation_space.dtype) == np.uint8 else torch.float32
    kind = type(action_space).__name__          # a2c_common.py:1211-1224
    if kind == 'Discrete':
        head_sizes, actions_num, is_multi_discrete = None, int(action_space.n), False
    elif kind == 'Tuple':
        head_sizes = [int(a.n) for a in action_space]
        actions_num, is_multi_discrete = sum(head_sizes), True      # width of the concatenated logits
        if len(head_sizes) > 8:
            raise NotImplementedError('more than 8 heads in a multi-discrete space')
    else:
        raise ValueError(f'Unsupported action space type for DiscreteA2CBase: {type(action_space)}')
    if max(head_sizes or [actions_num]) > 64:
        raise NotImplementedError('more than 64 actions in one discrete head')
    # True: every conv and linear layer on the bf16 tensor cores (conv_tc.cu, gemm_tc.cu); False or absent: the fp32 kernels
    mixed_precision = bool(config.get('mixed_precision') or False)
    return obs_shape, obs_dtype, head_sizes, actions_num, is_multi_discrete, mixed_precision


class DiscreteModel(FlatParamModel):
    """Flat fp32 parameter arena of A2CBuilder.Network for a discrete space.  Arena order: [actor conv trunk, [critic conv trunk]],
    actor MLP, [critic MLP], fused head W_head [1 + K, Hl] (row 0 = value, rows 1.. = logits) and b_head [1 + K]; ``_param_views``
    lists the tensors in the reference's ``model.parameters()`` order (actor_cnn.*, critic_cnn.*, actor_mlp.*, critic_mlp.*, value.*,
    logits.*) for state dicts and the index-keyed Adam state.

    ``obs_dim`` is the flat observation size, or the observation shape: a rank-3 shape with a plain ``conv2d`` cnn
    (network_builder.py:161-181) puts a convolutional trunk in front of each MLP."""

    def __init__(self, network_params, obs_dim, n_actions, device, normalize_input, normalize_value, head_sizes=None):
        self.head_sizes = list(head_sizes) if head_sizes else None          # multi-discrete: one logits head per Tuple component
        check_network_params(network_params)
        mlp = network_params['mlp']
        self.units = list(mlp['units'])
        if not self.units:
            raise NotImplementedError('empty MLP')
        self.activation = mlp.get('activation', 'relu')
        if self.activation not in ops.ACT:
            raise NotImplementedError(f'activation {self.activation}')
        self.act_id = ops.ACT[self.activation]
        if 'rnn' in network_params:
            raise NotImplementedError("'rnn' networks are not supported by the discrete B200 agent yet")
        self.obs_shape = tuple(obs_dim) if isinstance(obs_dim, (tuple, list, torch.Size)) else (int(obs_dim),)
        self.cnn = _ConvTrunk(network_params['cnn'], self.obs_shape) if 'cnn' in network_params else None
        mlp_init = mlp.get('initializer', {'name': 'default'})
        if self.cnn is None and mlp_init.get('name', 'default') != 'default':
            raise NotImplementedError("only the 'default' mlp initializer is mirrored for discrete models")
        self.separate = bool(network_params.get('separate', False))
        self.D, self.K = int(np.prod(self.obs_shape)), int(n_actions)
        self.mlp_in = self.cnn.out_size if self.cnn else self.D
        self.device = torch.device(device)
        self.normalize_input, self.normalize_value = bool(normalize_input), bool(normalize_value)
        sizes = []
        for p in (['a', 'c'] if self.separate and self.cnn else ['a'] if self.cnn else []):
            for i, (shp, _) in enumerate(self.cnn.layers):
                sizes += [(f'K{p}{i}', shp), (f'k{p}{i}', (shp[0],))]
        ins = self.mlp_in
        for i, u in enumerate(self.units):
            sizes += [(f'Wa{i}', (u, ins)), (f'ba{i}', (u,))]
            ins = u
        if self.separate:
            ins = self.mlp_in
            for i, u in enumerate(self.units):
                sizes += [(f'Wc{i}', (u, ins)), (f'bc{i}', (u,))]
                ins = u
        self.Hl = ins
        sizes += [('W_head', (1 + self.K, ins)), ('b_head', (1 + self.K,))]
        self._init_arena(sizes)
        if self.cnn:
            self._init_like_reference(mlp_init)
        else:
            self._init_linear_default()          # network_builder.py:332-340 with the 'default' initializer
        self.running_mean_std = _RunningStats(self.D, self.device) if self.normalize_input else None
        self.value_mean_std = _RunningStats(1, self.device) if self.normalize_value else None
        # the head is the linear output layer of the trunk's MLP: one MLP into [value | logits] when the trunk is shared; with separate
        # trunks the actor MLP ends in the logit rows of the head, the critic MLP in its value row
        wh, bh = self.view('W_head'), self.view('b_head')
        off_wh, off_bh = self.layout['W_head'][0], self.layout['b_head'][0]
        self.actor_mlp = self._trunk_layers('a')
        if self.separate:
            self.actor_mlp.append(Layer(wh[1:], bh[1:], off_wh + self.Hl, off_bh + 1, 0))
            self.critic_mlp = self._trunk_layers('c') + [Layer(wh[:1], bh[:1], off_wh, off_bh, 0)]
        else:
            self.actor_mlp.append(Layer(wh, bh, off_wh, off_bh, 0))
            self.critic_mlp = None
        # conv trunks: layer records of the actor's (shared) trunk and of the critic's; the conv parameters lead the arena
        self.actor_conv = self._conv_layers('a') if self.cnn else None
        self.critic_conv = self._conv_layers('c') if self.cnn and self.separate else None
        self.conv_params = self.layout['Wa0'][0]

    def _conv_layers(self, p):
        return [Layer(self.view(f'K{p}{i}'), self.view(f'k{p}{i}'), self.layout[f'K{p}{i}'][0], self.layout[f'k{p}{i}'][0], self.cnn.act)
                for i in range(len(self.cnn.layers))]

    def _init_like_reference(self, mlp_init):
        """A2CBuilder.Network.__init__ (network_builder.py:226-341) on torch's global generator, draw for draw: each Conv2d and Linear
        is constructed (torch's own init) in registration order, _calc_input_size draws its probe frame between the conv trunks and
        the MLPs, then the init loop applies the cnn initializer to every conv weight and the mlp initializer to every linear weight
        (a no-op for 'default'), zeroing every bias."""
        nn = torch.nn
        convs = [nn.Conv2d(shp[1], shp[0], (shp[2], shp[3]), stride=g[3], padding=g[4]) for _ in range(2 if self.separate else 1)
                 for shp, g in self.cnn.layers]
        torch.rand(1, *self.cnn.in_shape)
        lins, n_trunks = [], 2 if self.separate else 1
        for _ in range(n_trunks):
            ins = self.mlp_in
            for u in self.units:
                lins.append(nn.Linear(ins, u))
                ins = u
        lins.append(nn.Linear(self.Hl, 1))
        lins += [nn.Linear(self.Hl, k) for k in (self.head_sizes or [self.K])]
        with torch.no_grad():
            for mods, spec in ((convs, self.cnn.initializer), (lins, mlp_init)):
                for mod in mods:
                    if spec.get('name', 'default') != 'default':
                        _apply_init(mod.weight, spec, None)
                    mod.bias.zero_()
            for v, t in zip(self._param_views(), [t for mod in convs + lins for t in (mod.weight, mod.bias)]):
                v.copy_(t.reshape(v.shape))

    def _trunk_layers(self, p):
        return [Layer(self.view(f'W{p}{i}'), self.view(f'b{p}{i}'), self.layout[f'W{p}{i}'][0], self.layout[f'b{p}{i}'][0], self.act_id)
                for i in range(len(self.units))]

    def _param_views(self, arena=None):
        out = []
        for p in (['a', 'c'] if self.separate and self.cnn else ['a'] if self.cnn else []):
            for i in range(len(self.cnn.layers)):
                out += [self.view(f'K{p}{i}', arena), self.view(f'k{p}{i}', arena)]
        for p in (['a', 'c'] if self.separate else ['a']):
            for i in range(len(self.units)):
                out += [self.view(f'W{p}{i}', arena), self.view(f'b{p}{i}', arena)]
        wh, bh = self.view('W_head', arena), self.view('b_head', arena)
        out += [wh[:1], bh[:1]]
        if self.head_sizes is None:
            return out + [wh[1:], bh[1:]]
        off = 1
        for k in self.head_sizes:          # ModuleList of heads: logits.{j}.weight / bias (network_builder.py:304-305)
            out += [wh[off:off + k], bh[off:off + k]]
            off += k
        return out

    def param_names(self):
        names = []
        for pre in (['actor_cnn', 'critic_cnn'] if self.separate and self.cnn else ['actor_cnn'] if self.cnn else []):
            for i in range(len(self.cnn.layers)):
                names += [f'a2c_network.{pre}.{2 * i}.weight', f'a2c_network.{pre}.{2 * i}.bias']
        for pre in (['actor_mlp', 'critic_mlp'] if self.separate else ['actor_mlp']):
            for i in range(len(self.units)):
                names += [f'a2c_network.{pre}.{2 * i}.weight', f'a2c_network.{pre}.{2 * i}.bias']
        names += ['a2c_network.value.weight', 'a2c_network.value.bias']
        if self.head_sizes is None:
            return names + ['a2c_network.logits.weight', 'a2c_network.logits.bias']
        for j in range(len(self.head_sizes)):
            names += [f'a2c_network.logits.{j}.weight', f'a2c_network.logits.{j}.bias']
        return names

    def state_dict(self):
        sd = super().state_dict()
        if self.cnn and self.normalize_input:        # RunningMeanStd(obs_shape) keeps the frame's shape (models.py:31)
            for k in ('running_mean_std.running_mean', 'running_mean_std.running_var'):
                sd[k] = sd[k].reshape(self.obs_shape)
        return sd


class _ConvTrunk:
    """The geometry of a plain ``conv2d`` cnn (network_builder.py:161-181) on a rank-3 observation.  ``in_shape``: the network's
    (C, H, W) input, the env's (H, W, C) frame transposed when ``permute_input`` (the default, network_builder.py:360-361);
    ``layers``: ((Cout, C, KH, KW), (C, H, W, stride, pad)) per conv; ``out_shape`` / ``out_size``: the last conv's output and its
    flattened size, the MLP's input (_calc_input_size)."""

    REFUSED = {'conv2d_spatial_softargmax': 'a spatial soft-argmax head', 'conv2d_flatten': 'a flatten layer',
               'coord_conv2d': 'coordinate channels'}

    def __init__(self, cnn, obs_shape):
        ctype = cnn.get('type')
        if ctype != 'conv2d':
            why = self.REFUSED.get(ctype, 'only plain conv2d is built')
            raise NotImplementedError(f"'cnn' networks of type {ctype!r} ({why}) are not supported by the discrete B200 agent yet")
        if len(obs_shape) != 3:
            raise NotImplementedError(f"a 'conv2d' cnn needs a rank-3 Box observation, got shape {tuple(obs_shape)}")
        self.nhwc = bool(cnn.get('permute_input', True))
        self.in_shape = (obs_shape[2], obs_shape[0], obs_shape[1]) if self.nhwc else tuple(obs_shape)
        act = cnn.get('activation', 'relu')
        if act not in ops.ACT:
            raise NotImplementedError(f'cnn activation {act}')
        self.act = ops.ACT[act]
        self.initializer = dict(cnn.get('initializer') or {'name': 'default'})
        self.layers = []
        C, H, W = self.in_shape
        for conv in cnn['convs']:
            k, st, pad = conv['kernel_size'], conv['strides'], conv.get('padding', 0)
            if not all(isinstance(v, int) and not isinstance(v, bool) for v in (k, st, pad)) or k < 1 or st < 1 or pad < 0:
                raise NotImplementedError(f'conv2d kernel_size / strides / padding must be integers, got {k!r} / {st!r} / {pad!r}')
            Ho, Wo = (H + 2 * pad - k) // st + 1, (W + 2 * pad - k) // st + 1
            if Ho < 1 or Wo < 1:
                raise ValueError(f'conv2d kernel {k} does not fit a {H}x{W} input with padding {pad}')
            self.layers.append(((int(conv['filters']), C, k, k), (C, H, W, st, pad)))
            C, H, W = int(conv['filters']), Ho, Wo
        self.out_shape = (C, H, W)
        self.out_size = C * H * W


class DiscretePolicy:
    """The forward of a discrete policy, shared by the trainer (DiscreteA2CAgent) and the player (players.PpoPlayerDiscrete): the
    precision its conv and linear layers run on, its activation buffers and the conv + MLP forward.  The host class provides ``model``,
    ``actions_num`` and ``mixed_precision``."""
    wbf = None

    def _init_policy(self):
        """every conv and linear layer runs on one precision: fp32 CUDA cores, or bf16 tensor cores with the weights read from ``wbf``, a
        bf16 twin of the parameter arena (the categorical head kernels stay fp32 either way)"""
        m = self.model
        self.obs_norm = _RunningStats.f32_pair(m.running_mean_std)
        if self.mixed_precision:
            self.wbf = torch.empty(m.num_params, dtype=torch.bfloat16, device=m.device)
            self.kernels = layerwise.Kernels(tc=True, bf16_arena=(m.flat, self.wbf))
        else:
            self.kernels = layerwise.Kernels()

    def _repack(self):
        """the bf16 twin follows the fp32 arena: after every optimiser step, weight load and multi-GPU weight broadcast"""
        if self.wbf is not None:
            ops.cast_bf16(self.model.flat, self.wbf)

    def _alloc_rows(self, M):
        """(actor activations, critic activations, head output, actor conv activations, critic conv activations) for M rows: the MLP
        activations' last entry is the MLP's output layer, [value | logits] (shared trunk) or the logits / the value (separate trunks);
        the head output is its (logits, ld, value, value ld); the conv activations are NCHW rows of each conv trunk"""
        m, K = self.model, self.actions_num
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=m.device)   # noqa: E731
        acts_a = [f(M, u) for u in m.units] + [f(M, K if m.separate else 1 + K)]
        if m.separate:
            acts_c = [f(M, u) for u in m.units] + [f(M, 1)]
            out = (acts_a[-1], K, acts_c[-1], 1)
        else:
            acts_c, out = None, (acts_a[-1][:, 1:], K + 1, acts_a[-1], K + 1)
        conv = lambda: [f(M, shp[0], *self._conv_out(g, shp)) for shp, g in m.cnn.layers]   # noqa: E731
        return acts_a, acts_c, out, conv() if m.cnn else None, conv() if m.cnn and m.separate else None

    @staticmethod
    def _conv_out(g, shp):
        C, H, W, st, pad = g
        return (H + 2 * pad - shp[2]) // st + 1, (W + 2 * pad - shp[3]) // st + 1

    def _conv_forward(self, layers, x, acts, M, rows_per_chunk, chunk_stride):
        """acts[l] = act(conv_l(in_l)): in_0 = the observation rows (arena order, normalised), in_l = acts[l - 1]"""
        m = self.model
        for l, lay in enumerate(layers):
            g = m.cnn.layers[l][1]
            if l == 0:
                self.kernels.conv_fwd(x, lay.W, lay.b, acts[0], g, lay.act, M, nhwc=m.cnn.nhwc, rows_per_chunk=rows_per_chunk,
                                      chunk_stride=chunk_stride, x_ld=m.D, norm_mean=self.obs_norm[0], norm_std=self.obs_norm[1])
            else:
                self.kernels.conv_fwd(acts[l - 1], lay.W, lay.b, acts[l], g, lay.act, M)

    def _forward(self, x, acts_a, acts_c, M, rows_per_chunk=None, chunk_stride=0, conv=(None, None)):
        """the actor MLP into acts_a (its last entry: [value | logits], or the logits with separate trunks), the critic MLP into acts_c;
        with a cnn, each MLP reads its conv trunk's output (conv = (actor conv activations, critic conv activations))"""
        m = self.model
        if m.cnn:
            self._conv_forward(m.actor_conv, x, conv[0], M, rows_per_chunk, chunk_stride)
            layerwise.forward(self.kernels, m.actor_mlp, conv[0][-1].view(M, -1), acts_a, M, m.mlp_in)
            if m.separate:
                self._conv_forward(m.critic_conv, x, conv[1], M, rows_per_chunk, chunk_stride)
                layerwise.forward(self.kernels, m.critic_mlp, conv[1][-1].view(M, -1), acts_c, M, m.mlp_in)
            return
        layerwise.forward(self.kernels, m.actor_mlp, x, acts_a, M, m.D, rows_per_chunk, chunk_stride, self.obs_norm)
        if m.separate:
            layerwise.forward(self.kernels, m.critic_mlp, x, acts_c, M, m.D, rows_per_chunk, chunk_stride, self.obs_norm)


class DiscreteA2CAgent(DiscretePolicy, A2CBase):
    # torch_ext.AverageMeter means (float32) for the reward / episode-length summaries
    episode_summary_dtype = np.float32

    # multi-GPU (a2c_common.py:206-220): the per-minibatch gradient exchange is an NCCL all-reduce of the flat gradient in front of the
    # Adam kernel (which applies 1/world), the scheduler sees the rank-mean KL
    def __init__(self, base_name, params):
        super().__init__(base_name, params)
        self.model = DiscreteModel(self.network_params, self.obs_shape, self.actions_num, self.device_t, self.normalize_input,
                                   self.normalize_value, head_sizes=self.head_sizes)
        self.value_mean_std = self.model.value_mean_std
        self.rng_seed = int(self.config.get('b200_rng_seed', params.get('seed', 0) or 0))
        self.is_rnn, self.rnn_states, self.is_tensor_obses = False, None, True
        self.algo_observer.after_init(self)

    def _check_stats_sync_mode(self, mode):
        if mode != 'pooled':
            raise NotImplementedError("multi_gpu_sync_stats_mode: only 'pooled' for the discrete agent")
        return mode

    def _parse_config(self, config):
        if self.env_info.get('value_size', 1) != 1:
            raise NotImplementedError('value_size > 1')
        if config.get('central_value_config') is not None:
            raise NotImplementedError('central_value_config')
        # options of the reference agent that change what a run does and are not built for the discrete path: refuse, never ignore
        for key, bad in (('normalize_rms_advantage', bool(config.get('normalize_rms_advantage', False))),
                         ('epochs_between_resets', config.get('epochs_between_resets', 0) > 0),
                         ('self_play', config.get('self_play_config') is not None or bool(config.get('self_play', False)))):
            if bad:
                raise NotImplementedError(f'{key} is not built for the discrete B200 agent')
        self.has_central_value, self.central_value_net = False, None
        # multi-agent envs (the smac shape, a2c_common.py:340, :393): envs * agents independent actor rows, each with its own action mask
        self.num_agents, self.value_size = self.env_info.get('agents', 1), 1
        self.num_rows = self.num_actors * self.num_agents
        if self.mask_autoreset_rows and self.num_agents > 1:
            raise ValueError("PPO next_step autoreset masking does not support multi-agent envs; "
                             "wrap the env with a same_step autoreset adapter instead")
        self.observation_space = self.env_info['observation_space']
        (self.obs_shape, self.obs_dtype, self.head_sizes, self.actions_num, self.is_multi_discrete,
         self.mixed_precision) = discrete_spaces(self.observation_space, self.env_info['action_space'], self.network_params, config)
        self.is_discrete = True
        self.use_action_masks = bool(config.get('use_action_masks', False))

    def _make_writer(self):
        return make_summary_writer(self.summaries_dir)          # on every rank

    @property
    def stop_fn(self):
        """read from the config, unchecked (the continuous agent validates it at construction)"""
        return self.config.get('stop_fn', None)

    @staticmethod
    def _sync():
        torch.cuda.synchronize()

    # =============================================================================== allocation
    def init_tensors(self):
        if self._tensors_ready:
            return
        H, N, K, m, mb = self.horizon_length, self.num_rows, self.actions_num, self.model, self.minibatch_size
        D = m.D
        dev = self.device_t
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)   # noqa: E731
        self.obses = torch.zeros(H, N, D, dtype=self.obs_dtype, device=dev)
        self.actions = (torch.zeros(H, N, len(self.head_sizes), dtype=torch.int64, device=dev) if self.head_sizes
                        else torch.zeros(H, N, dtype=torch.int64, device=dev))
        self.neglogpacs, self.values, self.rewards = f(H, N), f(H, N), f(H, N)
        self.dones_buf = torch.zeros(H, N, dtype=torch.uint8, device=dev)
        self.action_masks = torch.ones(H, N, K, dtype=torch.uint8, device=dev) if self.use_action_masks else None
        self.valid = torch.ones(H, N, dtype=torch.float32, device=dev) if self.mask_autoreset_rows else None
        self.advs, self.returns = f(H, N), f(H, N)
        self.old_values_n, self.returns_n, self.advs_n = f(H, N), f(H, N), f(H, N)
        self.last_values = f(N)
        self.ep_state = f(3, N)
        self.dones = torch.ones(N, dtype=torch.uint8, device=dev)
        self.prev_dones = f(N) if self.mask_autoreset_rows else None
        self.meter = torch.zeros(8, dtype=torch.float64, device=dev)
        self.rng_epoch = torch.zeros(1, dtype=torch.int64, device=dev)
        # buffers of the rollout (r_) and training (t_) forwards and of the gradients (d_; the conv ones: pre-activation)
        self.r_a, self.r_c, self.r_out, self.r_ka, self.r_kc = self._alloc_rows(N)
        self.t_a, self.t_c, self.t_out, self.t_ka, self.t_kc = self._alloc_rows(mb)
        self.d_a, self.d_c, self.d_out, self.d_ka, self.d_kc = self._alloc_rows(mb)
        if self.mixed_precision:
            # tensor-core weight gradients: a CTA owns a [128 x <=128] tile of dW and a row split; the continuous agent's layer-wise
            # rule (16 splits at most) keeps enough CTAs per layer while the split partials stay small
            self.n_splits = max(1, min(16, mb // 512))
        else:
            self.n_splits = layerwise.n_splits(mb)
        self._init_policy()
        self._repack()
        # the conv weight gradients split over the output pixels' rows, so they take more split rows than the MLP (the leading
        # conv_params columns)
        self.conv_splits = layerwise.n_splits(mb * m.cnn.out_shape[1] * m.cnn.out_shape[2]) if m.cnn else 0
        self.part = f(max(self.n_splits, self.conv_splits), m.num_params)
        self.grad = f(m.num_params)
        self.diag_exp_var = f(self.num_minibatches) if self.diag_on else None
        self._diag_clip = []
        self.loss_partials = torch.zeros((mb + 255) // 256, 8, dtype=torch.float64, device=dev)
        self.gae_partials = torch.zeros(max(64, (N + 63) // 64), 8, dtype=torch.float64, device=dev)
        self.inv_counts = f(self.num_minibatches) if self.mask_autoreset_rows else None
        # uint8 frames update their statistics without partials (moments_update_u8); fp32 rows need NUM_SMS * 4 partial rows
        self.mom_scratch = (None if self.obs_dtype == torch.uint8 else
                            torch.zeros(ops.NUM_SMS * 4 * 2 * D, dtype=torch.float64, device=dev))
        self.post_scratch = torch.zeros(((N + 255) // 256) * 4, dtype=torch.float64, device=dev)
        self.post_ma = ops.post_step_ma_buffers(N, self.num_agents, dev) if self.num_agents > 1 else None
        self.counters = torch.zeros(4, dtype=torch.int32, device=dev)
        self.opt_state = torch.tensor([self.last_lr, 0.0, 0.0, 0.0], dtype=torch.float64, device=dev)
        self.adam_stats = f(16)
        self.opt_cfg = ops.OptCfg(0.9, 0.999, 1e-8, float(self.weight_decay), float(self.grad_norm), 0.0, 1e-6, 1e-2, 1.5,
                                  1.0 / self.world_size, int(bool(self.truncate_grads)), 0)
        rs = self.rewards_shaper
        self.shaper_cfg = ops.ShaperCfg(float(rs.scale_value), float(rs.shift_value), float(rs.min_val), float(rs.max_val),
                                        float(self.gamma), int(bool(rs.log_val)), int(bool(self.value_bootstrap)))
        self._tensors_ready = True

    # =============================================================================== env plumbing (tensor envs on the device)
    def _to_dev(self, x, dtype=None):
        t = x if torch.is_tensor(x) else torch.as_tensor(np.asarray(x))
        t = t.to(self.device_t)
        return t if dtype is None or t.dtype == dtype else t.to(dtype)

    def _obs_rows(self, o):
        """observations as arena rows: flat fp32, or image frames flattened in the env's layout and kept in the arena's dtype"""
        o = o['obs'] if isinstance(o, dict) else o
        if len(self.obs_shape) == 1:
            return self._to_dev(o, torch.float32).contiguous()
        o = self._to_dev(o, self.obs_dtype)
        return o.reshape(o.shape[0], -1).contiguous()

    def env_reset(self):
        return self._obs_rows(self.vec_env.reset())

    def env_step(self, actions):
        o, rewards, dones, infos = self.vec_env.step(actions)
        return self._obs_rows(o), self._to_dev(rewards, torch.float32), self._to_dev(dones), infos

    # =============================================================================== backward
    def _conv_backward(self, layers, x, acts, grads, M, rows_per_chunk, chunk_stride):
        """grads[-1] = dL/d(pre-activation of the last conv) in; weight gradients into the leading columns of `part`"""
        m, P = self.model, self.model.num_params
        for l in range(len(layers) - 1, -1, -1):
            lay, g = layers[l], m.cnn.layers[l][1]
            k = self.kernels
            if l == 0:
                k.conv_bwd_weight(grads[0], x, self.part[0, lay.w_off:], self.part[0, lay.b_off:], lay.W.shape, g, self.conv_splits, M, P,
                                  nhwc=m.cnn.nhwc, rows_per_chunk=rows_per_chunk, chunk_stride=chunk_stride, x_ld=m.D,
                                  norm_mean=self.obs_norm[0], norm_std=self.obs_norm[1])
            else:
                k.conv_bwd_weight(grads[l], acts[l - 1], self.part[0, lay.w_off:], self.part[0, lay.b_off:], lay.W.shape, g,
                                  self.conv_splits, M, P)
                k.conv_bwd_data(grads[l], lay.W, acts[l - 1], grads[l - 1], g, layers[l - 1].act, M)

    # =============================================================================== rollout
    def play_steps(self, u=None):
        """a2c_common.py:985-1069 for a discrete space; u: optional [H + 1, N] uniform tape (tests) -- else Philox."""
        self.init_tensors()
        H, N, K, m = self.horizon_length, self.num_rows, self.actions_num, self.model
        vm = m.value_mean_std
        step_time = 0.0
        for t in range(H):
            obs = self.obs
            self.obses[t].copy_(obs)
            masks = None
            if self.use_action_masks:          # a2c_common.py:995-997
                masks = self._to_dev(self.vec_env.get_action_masks()).to(torch.uint8).contiguous()
                self.action_masks[t].copy_(masks)
            self._forward(obs, self.r_a, self.r_c, N, conv=(self.r_ka, self.r_kc))
            lg, ld, vl, vld = self.r_out
            ops.categorical_sample(lg, ld, K, vl, vld, masks, None if u is None else u[t].contiguous(), self.rng_seed, self.rng_epoch, t,
                                   None if vm is None else vm.running_mean, None if vm is None else vm.running_var, self.normalize_value,
                                   self.actions[t], self.neglogpacs[t], self.values[t], self.dones, self.dones_buf[t], self.prev_dones,
                                   None if self.valid is None else self.valid[t], N, head_sizes=self.head_sizes)
            t0 = time.perf_counter()
            self.obs, rewards, dones, infos = self.env_step(self.actions[t])
            step_time += time.perf_counter() - t0
            tout = infos.get('time_outs') if (self.value_bootstrap and isinstance(infos, dict)) else None
            if tout is not None:
                tout = self._to_dev(tout)
            self._post_step(rewards, dones, tout, t, N)
            if getattr(self.algo_observer, 'wants_done_indices', True):
                self.algo_observer.process_infos(infos, self._done_indices())
            elif getattr(self.algo_observer, 'wants_infos', False):
                self.algo_observer.process_infos(infos, None)
        # get_values (a2c_common.py:603-626): the reference's forward samples here too; only the value is used
        self._forward(self.obs, self.r_a, self.r_c, N, conv=(self.r_ka, self.r_kc))
        lg, ld, vl, vld = self.r_out
        ops.categorical_sample(None, ld, K, vl, vld, None, None, 0, None, 0, None if vm is None else vm.running_mean,
                               None if vm is None else vm.running_var, self.normalize_value, None, None, self.last_values, None, None,
                               None, None, N, values_only=True)
        ops.bump_u64(self.rng_epoch)
        self._meter_cache = None
        return step_time

    def _gae_and_prepare(self):
        m = self.model
        nb = ops.gae_fused(self.rewards, self.values, self.dones_buf, self.last_values, self.dones, self.valid, self.advs, self.returns,
                           self.gae_partials, self.gamma, self.tau)
        vm = m.value_mean_std
        dummy = getattr(self, '_dummy_vms', None)
        if vm is None and dummy is None:
            dummy = self._dummy_vms = _RunningStats(1, self.device_t)
        s = vm if vm is not None else dummy
        ops.prepare_batch(self.values, self.returns, self.valid, self.gae_partials, nb, s.running_mean, s.running_var, s.count,
                          self.old_values_n, self.returns_n, self.advs_n, self.normalize_value, self.normalize_advantage)
        if self.mask_autoreset_rows:
            ops.mask_inv_counts(self.valid, self.horizon_length, self.num_rows, self.envs_per_mb, self.inv_counts)
        if self.diag_on:        # diagnostics/exp_var of every minibatch from the prepared dataset
            ops.explained_variance(self.old_values_n, self.returns_n, self.valid, self.horizon_length, self.num_rows, self.envs_per_mb,
                                   self.diag_exp_var)

    # =============================================================================== update
    def _minibatch_update(self, i):
        """calc_gradients (a2c_discrete.py:121-209) + trancate_gradients_and_step for minibatch i; returns a device row
        [a_loss, c_loss, entropy, kl] (masked means)."""
        m, H, N, K = self.model, self.horizon_length, self.num_rows, self.actions_num
        epm, mb, P, S = self.envs_per_mb, self.minibatch_size, self.model.num_params, self.n_splits
        e0 = i * epm
        x = self.obses[0, e0:]
        if self.normalize_input:      # set_train() re-arms the obs normaliser before every minibatch (see oracle/ppo_oracle.py)
            r = m.running_mean_std
            if self.obs_dtype == torch.uint8:
                ops.moments_update_u8(x, m.D, epm, H, N, r.running_mean, r.running_var, r.count, r.mean_f32, r.std_f32)
            else:
                ops.moments_update(x, m.D, epm, H, N, r.running_mean, r.running_var, r.count, r.mean_f32, r.std_f32, self.mom_scratch,
                                   self.counters[1:2])
        self._forward(x, self.t_a, self.t_c, mb, rows_per_chunk=epm, chunk_stride=N, conv=(self.t_ka, self.t_kc))
        lg, ld, vl, vld = self.t_out
        d_lg, d_ld, d_vl, d_vld = self.d_out
        cfg = ops.CatLossCfg(float(self.e_clip), float(self.critic_coef), float(self.entropy_coef), int(bool(self.clip_value)),
                             int(bool(self.use_smooth_clamp)), int(bool(self.ppo)))
        nb = ops.categorical_loss(lg, ld, K, vl, vld, self.actions[0, e0:], None if self.action_masks is None else self.action_masks[0, e0:],
                                  self.old_values_n[0, e0:], self.returns_n[0, e0:], self.neglogpacs[0, e0:], self.advs_n[0, e0:],
                                  None if self.valid is None else self.valid[0, e0:], epm, N, mb, cfg,
                                  None if self.inv_counts is None else self.inv_counts[i:i + 1], d_lg, d_ld, d_vl, d_vld,
                                  self.loss_partials, head_sizes=self.head_sizes)
        stats = self.loss_partials[:nb, :4].sum(dim=0).float()
        if self.diag_on:            # (sum mask, sum mask * clipped) of the minibatch: its clip fraction for diagnostics/clip_frac
            self._diag_clip.append(self.loss_partials[:nb, 4:6].sum(dim=0))
        # ---- backward through the MLP(s) [and the conv trunks]: split partial gradients, then one reduction ----
        if m.cnn:
            trunks = [(m.actor_mlp, m.actor_conv, self.t_a, self.d_a, self.t_ka, self.d_ka)]
            if m.separate:
                trunks.append((m.critic_mlp, m.critic_conv, self.t_c, self.d_c, self.t_kc, self.d_kc))
            for mlp, conv, acts, grads, kacts, kgrads in trunks:
                # dL/d(conv output) times the conv activation's derivative: the last conv's pre-activation gradient
                layerwise.backward(self.kernels, mlp, kacts[-1].view(mb, -1), acts, grads, self.part, P, S, mb, m.mlp_in,
                                   dx_out=kgrads[-1].view(mb, -1), dx_act=m.cnn.act)
                self._conv_backward(conv, x, kacts, kgrads, mb, epm, N)
            Pc = m.conv_params
            ops.reduce_splits(self.part, self.grad, Pc, self.conv_splits, split_stride=P)
            ops.reduce_splits(self.part[0, Pc:], self.grad[Pc:], P - Pc, S, split_stride=P)
        else:
            layerwise.backward(self.kernels, m.actor_mlp, x, self.t_a, self.d_a, self.part, P, S, mb, m.D, epm, N, self.obs_norm)
            if m.separate:
                layerwise.backward(self.kernels, m.critic_mlp, x, self.t_c, self.d_c, self.part, P, S, mb, m.D, epm, N, self.obs_norm)
            ops.reduce_splits(self.part, self.grad, P, S, split_stride=P)
        if self.multi_gpu:          # a2c_common.py:493-509 (the Adam kernel applies the 1/world scale)
            dist.all_reduce(self.grad, op=dist.ReduceOp.SUM)
        ops.adam_step(m.flat, self.grad, m.exp_avg, m.exp_avg_sq, self.opt_state, None, self.opt_cfg, self.adam_stats, self.counters[2:3],
                      n=P)
        self._repack()
        return stats

    def train_epoch(self, u=None):
        """DiscreteA2CBase.train_epoch (a2c_common.py:1233-1289): returns the reference's tuple."""
        self.init_tensors()
        if self.obs is None:
            self.obs = self.env_reset()
        t0 = time.perf_counter()
        step_time = self.play_steps(u)
        self._gae_and_prepare()
        self._sync()
        t1 = time.perf_counter()
        self.curr_frames = self.batch_size
        self.algo_observer.after_steps()
        rows, kls = [], []
        self._diag_clip = []
        for _ in range(self.mini_epochs_num):
            lr_used = self.last_lr          # what train_actor_critic returns for the minibatches of this mini-epoch (:1265, :1289)
            ep = [self._minibatch_update(i) for i in range(self.num_minibatches)]
            rows += ep
            av_kl = torch.stack([r[3] for r in ep]).mean()          # torch_ext.mean_list
            if self.multi_gpu:                                      # a2c_common.py:1272-1274
                dist.all_reduce(av_kl, op=dist.ReduceOp.SUM)
                av_kl = av_kl / self.world_size
            self.last_lr, self.entropy_coef = self.scheduler.update(self.last_lr, self.entropy_coef, self.epoch_num, self.frame,
                                                                    av_kl.item())                  # one host sync per mini-epoch (:1271)
            self.opt_state[0] = self.last_lr                        # update_lr
            kls.append(av_kl)
        self.sync_running_stats()
        if self.diag_on:
            clip_host = torch.empty(len(self._diag_clip), 2, dtype=torch.float64).pin_memory()
            ev_host = torch.empty(self.num_minibatches, dtype=torch.float32).pin_memory()
            clip_host.copy_(torch.stack(self._diag_clip), non_blocking=True)
            ev_host.copy_(self.diag_exp_var, non_blocking=True)
            self._diag_readback()
        self._sync()
        t2 = time.perf_counter()
        st = torch.stack(rows)
        self.last_stats = st
        if self.diag_on:
            # the loss kernels' clip fraction, as the continuous path's finalisation writes B200RL_STAT_CLIPFRAC
            clip = (clip_host[:, 1] / clip_host[:, 0].clamp(min=1.0)).float()
            self._replay_diagnostics(ev_host.repeat(self.mini_epochs_num), clip, clip_host[:, 0])
        a_losses, c_losses, entropies = list(st[:, 0]), list(st[:, 1]), list(st[:, 2])
        return step_time, t1 - t0, t2 - t1, t2 - t0, a_losses, c_losses, entropies, kls, lr_used, 1.0

    def train(self):
        self.mean_rewards = -float('inf')      # last_mean_rewards (best-ever watermark) is deliberately NOT reset here
        return super().train()

    # =============================================================================== weights / checkpoints (a2c_common.py:825-921)
    def set_weights(self, weights):
        super().set_weights(weights)
        self._repack()

    def get_full_state_weights(self):
        self.init_tensors()
        state = self.get_weights()
        state['epoch'], state['frame'] = self.epoch_num, self.frame
        step = float(self.opt_state.cpu()[1])
        state['optimizer'] = self.model.optimizer_state_dict(float(self.opt_state.cpu()[0]), step, self.weight_decay)      # the optimizer's own lr
        state['last_mean_rewards'] = self.last_mean_rewards
        return state

    def set_full_state_weights(self, weights, set_epoch=True):
        self.init_tensors()
        self.set_weights(weights)
        if set_epoch:
            self.epoch_num, self.frame = weights['epoch'], weights['frame']
        lr, step = self.model.load_optimizer_state_dict(weights['optimizer'])
        # a2c_common.py:852-866 restores the optimizer (its lr included) but not last_lr: the restored lr drives the optimiser until the
        # next scheduler step (end of the first mini-epoch), which continues from this agent's own last_lr
        opt_lr = float(lr) if lr is not None else self.last_lr
        self.opt_state.copy_(torch.tensor([opt_lr, float(step), 0.9 ** float(step) if step else 0.0,
                                           0.999 ** float(step) if step else 0.0], dtype=torch.float64))
        self.last_mean_rewards = weights.get('last_mean_rewards', -float('inf'))
