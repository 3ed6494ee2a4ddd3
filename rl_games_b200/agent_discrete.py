"""Discrete-action PPO agent on the fp32 CUDA kernels -- SURVEY.md 8a row a15 (reference: algos_torch/a2c_discrete.py
DiscreteA2CAgent + common/a2c_common.py:1205-1359 DiscreteA2CBase, models.py:62-125 ModelA2C, network_builder.py A2CBuilder with a
``discrete`` space, optionally ``separate: True`` actor/critic trunks, optional action masks).

STATUS: parity-green on an H100 (``tests/test_discrete_gpu.py``) against a CPU oracle that is pinned to the reference
(oracle/ppo_discrete_oracle.py, tests/golden/agent_discrete*.pt).  Everything except the two categorical kernels
(csrc/discrete.cu) reuses the kernels of the continuous path: linear_fwd / linear_bwd_* / reduce_splits (mlp_simt.cu), gae_fused, prepare_batch, moments_update,
mask_inv_counts (stats.cu, gae.cu), post_step (rollout.cu), adam_step (adam.cu).

Scope of this first edition: one GPU, eager launches (no CUDA graph), flat Box observations, ``Discrete(K)`` or multi-discrete
``Tuple(Discrete(K_j))`` action spaces (K_j <= 64, <= 8 heads), no RNN, no central value.  The scheduler steps once per MINI-EPOCH on the mean KL like the reference
(a2c_common.py:1265-1272), which costs one host sync per mini-epoch.

The agent derives from ``a2c_base.A2CBase`` (shared with the continuous agent) and adds the action space, the model, the arena, the
env plumbing, the rollout, the update and its resume semantics.
"""
import time

import numpy as np
import torch
import torch.distributed as dist

from . import ops
from .a2c_base import A2CBase
from .common import make_summary_writer
from .model import check_network_params, FlatParamModel, _RunningStats


class DiscreteModel(FlatParamModel):
    """Flat fp32 parameter arena of A2CBuilder.Network for a discrete space.  Arena order: actor trunk, [critic trunk], fused head
    W_head [1 + K, Hl] (row 0 = value, rows 1.. = logits) and b_head [1 + K]; ``_param_views`` lists the tensors in the reference's
    ``model.parameters()`` order (actor_mlp.*, critic_mlp.*, value.*, logits.*) for state dicts and the index-keyed Adam state."""

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
        if mlp.get('initializer', {'name': 'default'}).get('name', 'default') != 'default':
            raise NotImplementedError("only the 'default' mlp initializer is mirrored for discrete models")
        for k in ('cnn', 'rnn'):
            if k in network_params:
                raise NotImplementedError(f"'{k}' networks are not supported by the discrete B200 agent yet")
        self.separate = bool(network_params.get('separate', False))
        self.D, self.K = int(obs_dim), int(n_actions)
        self.device = torch.device(device)
        self.normalize_input, self.normalize_value = bool(normalize_input), bool(normalize_value)
        sizes, ins = [], self.D
        for i, u in enumerate(self.units):
            sizes += [(f'Wa{i}', (u, ins)), (f'ba{i}', (u,))]
            ins = u
        if self.separate:
            ins = self.D
            for i, u in enumerate(self.units):
                sizes += [(f'Wc{i}', (u, ins)), (f'bc{i}', (u,))]
                ins = u
        self.Hl = ins
        sizes += [('W_head', (1 + self.K, ins)), ('b_head', (1 + self.K,))]
        self._init_arena(sizes)
        self._init_linear_default()          # network_builder.py:332-340 with the 'default' initializer
        self.running_mean_std = _RunningStats(self.D, self.device) if self.normalize_input else None
        self.value_mean_std = _RunningStats(1, self.device) if self.normalize_value else None

    def trunk(self, which):
        p = 'a' if which == 'actor' or not self.separate else 'c'
        return [(self.view(f'W{p}{i}'), self.view(f'b{p}{i}')) for i in range(len(self.units))]

    def _param_views(self, arena=None):
        out = []
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
        for pre in (['actor_mlp', 'critic_mlp'] if self.separate else ['actor_mlp']):
            for i in range(len(self.units)):
                names += [f'a2c_network.{pre}.{2 * i}.weight', f'a2c_network.{pre}.{2 * i}.bias']
        names += ['a2c_network.value.weight', 'a2c_network.value.bias']
        if self.head_sizes is None:
            return names + ['a2c_network.logits.weight', 'a2c_network.logits.bias']
        for j in range(len(self.head_sizes)):
            names += [f'a2c_network.logits.{j}.weight', f'a2c_network.logits.{j}.bias']
        return names


class DiscreteA2CAgent(A2CBase):
    # torch_ext.AverageMeter means (float32) for the reward / episode-length summaries
    episode_summary_dtype = np.float32

    # multi-GPU (a2c_common.py:206-220): the per-minibatch gradient exchange is an NCCL all-reduce of the flat gradient in front of the
    # Adam kernel (which applies 1/world), the scheduler sees the rank-mean KL
    def __init__(self, base_name, params):
        super().__init__(base_name, params)
        self.model = DiscreteModel(self.network_params, self.obs_shape[0], self.actions_num, self.device_t, self.normalize_input,
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
        if type(self.observation_space).__name__ == 'Dict' or len(self.observation_space.shape) != 1:
            raise NotImplementedError('only flat Box observations')
        self.obs_shape = self.observation_space.shape
        action_space = self.env_info['action_space']
        kind = type(action_space).__name__          # a2c_common.py:1211-1224
        if kind == 'Discrete':
            self.head_sizes, self.actions_num, self.is_multi_discrete = None, int(action_space.n), False
        elif kind == 'Tuple':
            self.head_sizes = [int(a.n) for a in action_space]
            self.actions_num, self.is_multi_discrete = sum(self.head_sizes), True      # width of the concatenated logits
            if len(self.head_sizes) > 8:
                raise NotImplementedError('more than 8 heads in a multi-discrete space')
        else:
            raise ValueError(f'Unsupported action space type for DiscreteA2CBase: {type(action_space)}')
        self.is_discrete = True
        if max(self.head_sizes or [self.actions_num]) > 64:
            raise NotImplementedError('more than 64 actions in one discrete head')
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
        H, N, D, K, m, mb = self.horizon_length, self.num_rows, self.obs_shape[0], self.actions_num, self.model, self.minibatch_size
        dev = self.device_t
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)   # noqa: E731
        self.obses = f(H, N, D)
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
        L = len(m.units)
        # rollout / training activations of the actor trunk (and the critic trunk when separate), head buffers
        self.r_a = [f(N, u) for u in m.units]
        self.r_c = [f(N, u) for u in m.units] if m.separate else self.r_a
        self.t_a = [f(mb, u) for u in m.units]
        self.t_c = [f(mb, u) for u in m.units] if m.separate else self.t_a
        self.d_a = [f(mb, u) for u in m.units]
        self.d_c = [f(mb, u) for u in m.units] if m.separate else self.d_a
        self.r_head, self.t_head, self.d_head = f(N, 1 + K), f(mb, 1 + K), f(mb, 1 + K)
        self.n_splits = max(1, min(64, mb // 256))
        self.part = f(self.n_splits, m.num_params)
        self.grad = f(m.num_params)
        self.diag_exp_var = f(self.num_minibatches) if self.diag_on else None
        self._diag_clip = []
        self.loss_partials = torch.zeros((mb + 255) // 256, 8, dtype=torch.float64, device=dev)
        self.gae_partials = torch.zeros(max(64, (N + 63) // 64), 8, dtype=torch.float64, device=dev)
        self.inv_counts = f(self.num_minibatches) if self.mask_autoreset_rows else None
        self.mom_scratch = torch.zeros(ops.NUM_SMS * 4 * 2 * D, dtype=torch.float64, device=dev)
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
        assert L >= 1

    # =============================================================================== env plumbing (tensor envs on the device)
    def _to_dev(self, x, dtype=None):
        t = x if torch.is_tensor(x) else torch.as_tensor(np.asarray(x))
        t = t.to(self.device_t)
        return t if dtype is None or t.dtype == dtype else t.to(dtype)

    def env_reset(self):
        o = self.vec_env.reset()
        o = o['obs'] if isinstance(o, dict) else o
        return self._to_dev(o, torch.float32).contiguous()

    def env_step(self, actions):
        o, rewards, dones, infos = self.vec_env.step(actions)
        o = o['obs'] if isinstance(o, dict) else o
        return self._to_dev(o, torch.float32).contiguous(), self._to_dev(rewards, torch.float32), self._to_dev(dones), infos

    # =============================================================================== forward pieces
    def _norm(self):
        r = self.model.running_mean_std
        return (r.mean_f32, r.std_f32) if self.normalize_input else (None, None)

    def _trunk(self, layers, x, acts, M, rows_per_chunk=None, chunk_stride=0):
        nm, ns = self._norm()
        m = self.model
        ops.linear_fwd(x, layers[0][0], layers[0][1], acts[0], m.act_id, rows_per_chunk=rows_per_chunk, chunk_stride=chunk_stride,
                       x_ld=m.D, norm_mean=nm, norm_std=ns, M=M)
        for i in range(1, len(layers)):
            ops.linear_fwd(acts[i - 1], layers[i][0], layers[i][1], acts[i], m.act_id, M=M)

    def _heads(self, a_last, c_last, head, M):
        """head[:, 0] = value, head[:, 1:] = logits (one GEMM when the trunk is shared)"""
        m = self.model
        wh, bh = m.view('W_head'), m.view('b_head')
        if not m.separate:
            ops.linear_fwd(a_last, wh, bh, head, 0, M=M)
            return
        # separate trunks: two skinny GEMMs into strided halves of the same head buffer is not expressible with linear_fwd's dense
        # output, so the value and the logits go to their own dense buffers
        ops.linear_fwd(c_last, wh[:1], bh[:1], self._val_buf(M), 0, M=M)
        ops.linear_fwd(a_last, wh[1:], bh[1:], self._logit_buf(M), 0, M=M)

    def _val_buf(self, M):
        if not hasattr(self, '_vb'):
            self._vb = {}
        return self._vb.setdefault(M, torch.zeros(M, 1, dtype=torch.float32, device=self.device_t))

    def _logit_buf(self, M):
        if not hasattr(self, '_lb'):
            self._lb = {}
        return self._lb.setdefault(M, torch.zeros(M, self.actions_num, dtype=torch.float32, device=self.device_t))

    def _head_views(self, head, M):
        """(logits, ld, value, value_ld) of the forward buffers for M rows"""
        K = self.actions_num
        if self.model.separate:
            return self._logit_buf(M), K, self._val_buf(M), 1
        return head[:, 1:], K + 1, head, K + 1

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
            self._trunk(m.trunk('actor'), obs, self.r_a, N)
            if m.separate:
                self._trunk(m.trunk('critic'), obs, self.r_c, N)
            self._heads(self.r_a[-1], self.r_c[-1], self.r_head, N)
            lg, ld, vl, vld = self._head_views(self.r_head, N)
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
        self._trunk(m.trunk('actor'), self.obs, self.r_a, N)
        if m.separate:
            self._trunk(m.trunk('critic'), self.obs, self.r_c, N)
        self._heads(self.r_a[-1], self.r_c[-1], self.r_head, N)
        lg, ld, vl, vld = self._head_views(self.r_head, N)
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
            ops.moments_update(x, m.D, epm, H, N, r.running_mean, r.running_var, r.count, r.mean_f32, r.std_f32, self.mom_scratch,
                               self.counters[1:2])
        self._trunk(m.trunk('actor'), x, self.t_a, mb, rows_per_chunk=epm, chunk_stride=N)
        if m.separate:
            self._trunk(m.trunk('critic'), x, self.t_c, mb, rows_per_chunk=epm, chunk_stride=N)
        self._heads(self.t_a[-1], self.t_c[-1], self.t_head, mb)
        lg, ld, vl, vld = self._head_views(self.t_head, mb)
        if m.separate:
            d_lg, d_ld, d_vl, d_vld = self._dl_buf(), K, self._dv_buf(), 1
        else:
            d_lg, d_ld, d_vl, d_vld = self.d_head[:, 1:], K + 1, self.d_head, K + 1
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
        # ---- backward through the heads and the trunk(s): split partial gradients, then one reduction ----
        off_wh, _ = m.layout['W_head']
        off_bh, _ = m.layout['b_head']
        nm, ns = self._norm()
        if m.separate:
            Hl = m.Hl
            ops.linear_bwd_weight(d_vl, self.t_c[-1], self.part[0, off_wh:], self.part[0, off_bh:], Hl, 1, S, M=mb, split_stride=P)
            ops.linear_bwd_weight(d_lg, self.t_a[-1], self.part[0, off_wh + Hl:], self.part[0, off_bh + 1:], Hl, K, S, M=mb, split_stride=P)
            wh = m.view('W_head')
            ops.linear_bwd_data(d_vl, wh[:1], self.t_c[-1], self.d_c[-1], m.act_id, M=mb)
            ops.linear_bwd_data(d_lg, wh[1:], self.t_a[-1], self.d_a[-1], m.act_id, M=mb)
            trunks = [('a', self.t_a, self.d_a), ('c', self.t_c, self.d_c)]
        else:
            ops.linear_bwd_weight(self.d_head, self.t_a[-1], self.part[0, off_wh:], self.part[0, off_bh:], m.Hl, 1 + K, S, M=mb,
                                  split_stride=P)
            ops.linear_bwd_data(self.d_head, m.view('W_head'), self.t_a[-1], self.d_a[-1], m.act_id, M=mb)
            trunks = [('a', self.t_a, self.d_a)]
        for p, acts, dacts in trunks:
            for l in range(len(m.units) - 1, -1, -1):
                off_w, shp = m.layout[f'W{p}{l}']
                off_b, _ = m.layout[f'b{p}{l}']
                if l > 0:
                    ops.linear_bwd_weight(dacts[l], acts[l - 1], self.part[0, off_w:], self.part[0, off_b:], shp[1], shp[0], S, M=mb,
                                          split_stride=P)
                    ops.linear_bwd_data(dacts[l], m.view(f'W{p}{l}'), acts[l - 1], dacts[l - 1], m.act_id, M=mb)
                else:
                    ops.linear_bwd_weight(dacts[0], x, self.part[0, off_w:], self.part[0, off_b:], shp[1], shp[0], S, rows_per_chunk=epm,
                                          chunk_stride=N, x_ld=m.D, norm_mean=nm, norm_std=ns, M=mb, split_stride=P)
        ops.reduce_splits(self.part, self.grad, P, S, split_stride=P)
        if self.multi_gpu:          # a2c_common.py:493-509 (the Adam kernel applies the 1/world scale)
            dist.all_reduce(self.grad, op=dist.ReduceOp.SUM)
        ops.adam_step(m.flat, self.grad, m.exp_avg, m.exp_avg_sq, self.opt_state, None, self.opt_cfg, self.adam_stats, self.counters[2:3],
                      n=P)
        return stats

    def _dl_buf(self):
        if not hasattr(self, '_dlb'):
            self._dlb = torch.zeros(self.minibatch_size, self.actions_num, dtype=torch.float32, device=self.device_t)
        return self._dlb

    def _dv_buf(self):
        if not hasattr(self, '_dvb'):
            self._dvb = torch.zeros(self.minibatch_size, 1, dtype=torch.float32, device=self.device_t)
        return self._dvb

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
