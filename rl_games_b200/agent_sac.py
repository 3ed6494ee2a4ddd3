"""SACAgent: the reference's ``rl_games.algos_torch.sac_agent.SACAgent`` on the CUDA path.

Same config surface, summaries, checkpoints and ``restore``; the replay buffer, the sampling, the five MLP passes of an update, the
losses, the three Adam steps and the Polyak update all run as device kernels (csrc/sac.cu, csrc/mlp_simt.cu / gemm_tc.cu,
csrc/adam.cu).  Random draws are device Philox (seed, per-call-site key, a device counter), so an update reads nothing from the host.
With ``b200_cuda_graph`` (default True) the two update shapes -- critic only, critic + actor -- are captured once each as CUDA graphs
and replayed; ``policy_frequency`` parity is known on the host.

Test hook: ``agent.tapes = {'idx': iter, 'noise_next': iter, 'noise_actor': iter, 'noise_roll': iter, 'u': iter}`` replaces each
Philox draw with the next tensor of the matching iterator (replay indices [B], normals [M, A], uniforms [N, A]).
"""
import os
import time
from datetime import datetime

import numpy as np
import torch

from . import ops
from .common import DefaultAlgoObserver, DefaultRewardsShaper, create_vec_env, make_summary_writer
from .model import CompileTolerantModel, resolve_device
from .model_sac import SACModel

MIN_ALPHA = 0.01        # sac_agent.py base_init: the fixed floor of the actor loss's alpha

# every config key the agent reads, plus what launchers and the reference's Runner inject; anything else raises
_KNOWN_KEYS = {
    'name', 'env_name', 'env_config', 'env_info', 'vec_env', 'device', 'features', 'reward_shaper', 'num_actors', 'normalize_input',
    'mixed_precision', 'gamma', 'critic_tau', 'num_steps_per_episode', 'utd_ratio', 'num_updates_per_step', 'num_warmup_frames',
    'num_warmup_steps', 'batch_size', 'init_alpha', 'learnable_temperature', 'replay_buffer_size', 'save_replay_buffer', 'policy_frequency',
    'critic_grad_clip', 'value_bootstrap', 'actor_lr', 'critic_lr', 'alpha_lr', 'actor_betas', 'critic_betas', 'alphas_betas',
    'target_entropy_coef', 'max_epochs', 'max_frames', 'save_frequency', 'save_best_after', 'print_stats', 'train_dir',
    'full_experiment_name', 'games_to_track', 'score_to_win', 'stop_fn', 'multi_gpu', 'capability_manifest', 'weight_decay', 'b200_cuda_graph',
    'population_based_training',
    # read by others, not by the trainer: `player` configures the reference's SACPlayer (inference); `torch_compile` is read by the
    # Runner, whose torch.compile of agent.model is declined with a printed note (CompileTolerantModel)
    'player', 'torch_compile',
}


class SACAgent(CompileTolerantModel):
    def __init__(self, base_name, params):
        self.config = config = params['config']
        self.name = base_name
        unknown = sorted(set(config) - _KNOWN_KEYS)
        if unknown:
            raise NotImplementedError(f'SAC config keys with no implementation here: {unknown}')
        if config.get('multi_gpu', False):
            raise NotImplementedError('multi_gpu: True is not supported by the SAC agent (the reference SAC is single-process too)')
        if config.get('population_based_training', False):
            raise NotImplementedError('population_based_training is not supported by the SAC agent')
        if float(config.get('weight_decay', 0.0)) != 0.0:
            raise NotImplementedError('weight_decay: the reference SAC optimisers take none')
        self.network_params = params['network']
        self.device_str = config.get('device', 'cuda:0')
        self.ppo_device = self.device_str          # the name the reference's Runner reads
        self._require_cuda()
        self.device_t = resolve_device(self.device_str)
        config.setdefault('features', {})
        self.algo_observer = config['features'].get('observer') or DefaultAlgoObserver()

        self.num_actors = config.get('num_actors', 1)
        self.env_name = config['env_name']
        self.env_config = config.get('env_config', {})
        self.env_info = config.get('env_info')
        if self.env_info is None:
            self.vec_env = create_vec_env(self.env_name, self.num_actors, **self.env_config)
            self.env_info = self.vec_env.get_env_info()
        else:
            self.vec_env = config.get('vec_env', None)
        self.num_agents = self.env_info.get('agents', 1)
        if self.num_agents > 1:
            raise NotImplementedError("env_info['agents'] > 1: multi-agent SAC is not supported")
        obs_space, act_space = self.env_info['observation_space'], self.env_info['action_space']
        if isinstance(obs_space, dict) or hasattr(obs_space, 'spaces') or len(getattr(obs_space, 'shape', ()) or ()) != 1:
            raise NotImplementedError('SAC needs a flat Box observation space (CNN / dict observations are not supported)')
        if not hasattr(act_space, 'low') or len(act_space.shape) != 1:
            raise NotImplementedError('SAC supports continuous Box action spaces only (discrete action spaces are not supported)')
        self.autoreset_mode = self.env_info.get('autoreset_mode', 'same_step')

        self.gamma = config.get('gamma', 0.99)
        self.critic_tau = float(config.get('critic_tau', 0.005))
        self.num_steps_per_episode = config.get('num_steps_per_episode', 1)
        utd = config.get('utd_ratio', None)
        self.num_updates_per_step = max(1, round(utd * self.num_actors)) if utd is not None else config.get('num_updates_per_step', 1)
        if config.get('num_warmup_frames', None) is not None:
            self.num_warmup_steps = int(np.ceil(config['num_warmup_frames'] / (self.num_actors * self.num_steps_per_episode)))
        else:
            self.num_warmup_steps = config.get('num_warmup_steps', 1000)
        self.batch_size = config['batch_size']
        self.init_alpha = config['init_alpha']
        self.learnable_temperature = config['learnable_temperature']
        self.replay_buffer_size = config['replay_buffer_size']
        if self.replay_buffer_size < self.num_actors:
            raise NotImplementedError('replay_buffer_size smaller than num_actors (one env step would overwrite itself)')
        self.save_replay_buffer = config.get('save_replay_buffer', False)
        self.normalize_input = config.get('normalize_input', False)
        self.mixed_precision = bool(config.get('mixed_precision', True))      # torch_ext.default_mixed_precision() on a bf16 GPU
        self.policy_frequency = config.get('policy_frequency', 2)
        self.update_counter = 0
        self.critic_grad_clip = config.get('critic_grad_clip', 5.0)
        self.value_bootstrap = config.get('value_bootstrap', True)
        self.target_entropy_coef = config.get('target_entropy_coef', 1.0)
        self.A = act_space.shape[0]
        self.D = obs_space.shape[0]
        self.target_entropy = self.target_entropy_coef * -self.A
        self.num_frames_per_epoch = self.num_actors * self.num_steps_per_episode
        self.save_best_after = config.get('save_best_after', 500)
        self.save_freq = config.get('save_frequency', 0)
        self.print_stats = config.get('print_stats', True)
        self.max_epochs = config.get('max_epochs', -1)
        self.max_frames = config.get('max_frames', -1)
        self.games_to_track = config.get('games_to_track', 100)
        self.stop_fn = config.get('stop_fn', None)
        if self.stop_fn is not None and not callable(self.stop_fn):
            raise ValueError(f"'stop_fn' must be callable, got {type(self.stop_fn).__name__}")
        self.use_graph = bool(config.get('b200_cuda_graph', True))
        rs = config['reward_shaper']
        self.rewards_shaper = rs if not isinstance(rs, dict) else DefaultRewardsShaper(**rs)
        self.lrs = (float(config['actor_lr']), float(config['critic_lr']), float(config['alpha_lr']))
        self.betas = (tuple(config.get('actor_betas', [0.9, 0.999])), tuple(config.get('critic_betas', [0.9, 0.999])),
                      tuple(config.get('alphas_betas', [0.9, 0.999])))

        dev = self.device_t
        self.action_low = torch.tensor(act_space.low, dtype=torch.float32).to(dev)
        self.action_high = torch.tensor(act_space.high, dtype=torch.float32).to(dev)
        self.action_scale = (self.action_high - self.action_low) / 2.0
        self.action_bias = (self.action_high + self.action_low) / 2.0
        lss = torch.log(((torch.tensor(act_space.high, dtype=torch.float32) - torch.tensor(act_space.low, dtype=torch.float32)) / 2.0)
                        .clamp_min(1e-8)).sum()
        self.log_action_scale_sum = float(lss)
        self.act_box = (self.action_scale, self.action_bias, self.action_low, self.action_high)

        self.model = SACModel(self.network_params, self.D, self.A, dev, self.normalize_input, self.init_alpha)
        self.seed = int(params.get('seed', 0) or 0) & 0xFFFFFFFFFFFFFFFF

        self.frame = self.epoch_num = 0
        self.last_mean_rewards = -float('inf')
        self.mean_rewards = -float('inf')
        self.experiment_name = config.get('full_experiment_name') or (config['name'] + datetime.now().strftime('_%d-%H-%M-%S'))
        self.train_dir = config.get('train_dir', 'runs')
        self.experiment_dir = os.path.join(self.train_dir, self.experiment_name)
        self.nn_dir = os.path.join(self.experiment_dir, 'nn')
        self.summaries_dir = os.path.join(self.experiment_dir, 'summaries')
        for d in (self.train_dir, self.experiment_dir, self.nn_dir, self.summaries_dir):
            os.makedirs(d, exist_ok=True)
        self.writer = make_summary_writer(self.summaries_dir)
        self.tapes = None
        self._tb = None
        self.obs = None
        self._tensor_env = True
        self._alloc()
        self._graphs = {}

    # =============================================================================== device state
    def _require_cuda(self):
        """no CPU fallback: the kernels are the product (the host-logic tests replace this hook together with every op)"""
        if not str(self.device_str).startswith('cuda'):
            raise RuntimeError('rl_games_b200 agents run on CUDA only (device=%r): there is no CPU fallback' % self.device_str)
        torch.cuda.set_device(resolve_device(self.device_str))

    @property
    def device(self):
        return self.device_str

    def _alloc(self):
        dev, N, D, A, B, cap = self.device_t, self.num_actors, self.D, self.A, self.batch_size, self.replay_buffer_size
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)       # noqa: E731
        u8 = lambda *s: torch.zeros(*s, dtype=torch.uint8, device=dev)        # noqa: E731
        self.rb = {'obs': f(cap, D), 'act': f(cap, A), 'rew': f(cap), 'next': f(cap, D), 'term': u8(cap), 'trunc': u8(cap),
                   'state': torch.zeros(2, dtype=torch.int64, device=dev)}
        self.slot = torch.zeros(N, dtype=torch.int32, device=dev)
        self.term_s, self.trunc_s, self.prev_dones = u8(N), u8(N), u8(N)
        self.ep_state = f(2 * N)
        self.meter = torch.zeros(3, dtype=torch.float64, device=dev)
        self.rng_ctr = torch.zeros(1, dtype=torch.int64, device=dev)
        self.roll_ctr = torch.zeros(1, dtype=torch.int64, device=dev)
        u = self.model.units
        self.x_cur, self.x_pi, self.x_next = f(B, D + A), f(B, D + A), f(B, D + A)
        self.reward_b, self.not_done_b = f(B), f(B)
        self.acts_a = [f(B, w) for w in u] + [f(B, 2 * A)]               # actor trunk activations + head
        self.acts_q = [[f(B, w) for w in u] + [f(B, 1)] for _ in range(2)]
        self.acts_t = [[f(B, w) for w in u] + [f(B, 1)] for _ in range(2)]
        self.d_act = [f(B, w) for w in u]
        self.d_out = [f(B, 1), f(B, 1)]
        self.d_head = f(B, 2 * A)
        self.dx_in = [f(B, D + A), f(B, D + A)]
        self.eps_pi = f(B, A)
        self.logp_next, self.logp_pi = f(B), f(B)
        self.roll_acts = [f(N, w) for w in u] + [f(N, 2 * A)]
        self.actions = f(N, A)
        self.obs_buf = f(N, D)
        self.n_splits = max(1, min(64, B // 256))
        m = self.model
        self.part_a = f(self.n_splits, m.actor.n)
        self.part_c = f(self.n_splits, m.critic.n)
        self.stats = f(self.num_updates_per_step * self.num_steps_per_episode + 1, 8)
        self.counters = torch.zeros(4, dtype=torch.int32, device=dev)
        self.opt_state = torch.zeros(3, 8, dtype=torch.float64, device=dev)
        for i, lr in enumerate(self.lrs):
            self.opt_state[i, 0] = lr
        self.opt_cfg = [ops.OptCfg(b[0], b[1], 1e-8, 0.0, float(gn), 0.0, 0.0, 0.0, 1.0, 1.0, int(gn > 0), 0)
                        for b, gn in zip(self.betas, (0.0, self.critic_grad_clip, 0.0))]
        if self.normalize_input:
            self.rms_scratch = torch.zeros(ops.NUM_SMS * 2 * D, dtype=torch.float64, device=dev)
            self.rms_counter = torch.zeros(1, dtype=torch.int32, device=dev)
        if self.mixed_precision:
            self._fwd, self._bwd_data, self._bwd_w = ops.linear_fwd_tc, ops.linear_bwd_data_tc, ops.linear_bwd_weight_tc
        else:
            self._fwd, self._bwd_data, self._bwd_w = ops.linear_fwd, ops.linear_bwd_data, ops.linear_bwd_weight

    def init_tensors(self):
        self.ep_state.zero_()
        self.prev_dones.zero_()

    @property
    def alpha(self):
        return self.model.log_alpha.exp()

    # =============================================================================== MLP passes
    def _mlp_fwd(self, layers, x, x_ld, K0, acts, M, norm=None, fp32=False):
        """fp32=True: the fp32 kernels whatever mixed_precision says -- the passes the reference runs outside autocast (the critic target's
        actor and target critics, sac_agent.py update_critic; the rollout's act())"""
        L = len(layers)
        fwd = ops.linear_fwd if fp32 else self._fwd
        for l, (W, b) in enumerate(layers):
            X, ld, K = (x, x_ld, K0) if l == 0 else (acts[l - 1], W.shape[1], W.shape[1])
            nm, ns = norm if (l == 0 and norm is not None) else (None, None)
            fwd(X, W, b, acts[l], self.model.act_id if l < L - 1 else 0, x_ld=ld, norm_mean=nm, norm_std=ns, M=M)

    def _mlp_bwd(self, arena, prefix, layers, x, x_ld, acts, d_top, part, M, dx_out=None, weights=True):
        """gradients of one MLP into `part` (split partials of `arena`) and, with dx_out, dL/d(input) into dx_out"""
        L, act = len(layers), self.model.act_id
        pre = 'trunk.' if prefix == '' else prefix
        dY = d_top
        for l in range(L - 1, -1, -1):
            W, _ = layers[l]
            X, ld = (x, x_ld) if l == 0 else (acts[l - 1], W.shape[1])
            if weights:
                ow, ob = arena.layout[f'{pre}{2 * l}.weight'][0], arena.layout[f'{pre}{2 * l}.bias'][0]
                self._bwd_w(dY, X, part[0, ow:], part[0, ob:], W.shape[1], W.shape[0], self.n_splits, x_ld=ld, M=M, split_stride=arena.n)
            if l > 0:
                self._bwd_data(dY, W, acts[l - 1], self.d_act[l - 1], act, M=M)
                dY = self.d_act[l - 1]
            elif dx_out is not None:
                self._bwd_data(dY, W, None, dx_out, 0, M=M)

    def _adam(self, i, params, grads, m, v, n):
        ops.adam_step(params, grads, m, v, self.opt_state[i], None, self.opt_cfg[i], None, self.counters[i:i + 1], n=n)

    def _tape(self, key):
        if self.tapes is None or key not in self.tapes:
            return None
        return next(self.tapes[key]).to(self.device_t)

    def _fill_update_tapes(self, actor_step):
        """copy this update's tape draws into fixed device buffers, which the eager and the captured update both read"""
        B, A = self.batch_size, self.A
        if self._tb is None:
            self._tb = {'idx': torch.zeros(B, dtype=torch.int64, device=self.device_t), 'noise_next': torch.zeros(B, A, device=self.device_t),
                        'noise_actor': torch.zeros(B, A, device=self.device_t)}
        for k in ('idx', 'noise_next') + (('noise_actor',) if actor_step else ()):
            self._tb[k].copy_(self._tape(k))

    def _tb_get(self, key):
        return None if self.tapes is None else self._tb[key]

    # =============================================================================== one gradient update (sac_agent.py update)
    def _update(self, stats_row, actor_step):
        m, B, D, A = self.model, self.batch_size, self.D, self.A
        ld = D + A
        norm = (m.running_mean_std.mean_f32, m.running_mean_std.std_f32) if self.normalize_input else (None, None)
        ops.sac_replay_sample(self.rb, B, self._tb_get('idx'), self.seed, self.rng_ctr, norm[0], norm[1], self.x_cur, self.x_pi, self.x_next,
                              self.reward_b, self.not_done_b)
        # ---- update_critic: target from the next observations (actor + target critics, no gradients)
        actor_l = m.layers(m.actor)
        self._mlp_fwd(actor_l, self.x_next, ld, D, self.acts_a, B, fp32=True)
        ops.sac_squash_fwd(self.acts_a[-1], B, A, m.log_std_bounds, self._tb_get('noise_next'), self.seed, self.rng_ctr, ops.SAC_SITE_NEXT,
                           self.act_box, self.log_action_scale_sum, dst=self.x_next[:, D:], dst_ld=ld, logp=self.logp_next)
        for k, q in enumerate(('Q1.', 'Q2.')):
            self._mlp_fwd(m.layers(m.critic_target, q), self.x_next, ld, ld, self.acts_t[k], B, fp32=True)
            self._mlp_fwd(m.layers(m.critic, q), self.x_cur, ld, ld, self.acts_q[k], B)
        ops.sac_critic_loss(self.acts_q[0][-1], self.acts_q[1][-1], self.acts_t[0][-1], self.acts_t[1][-1], self.logp_next, self.reward_b,
                            self.not_done_b, m.log_alpha, self.gamma, B, self.d_out[0], self.d_out[1], stats_row)
        for k, q in enumerate(('Q1.', 'Q2.')):
            self._mlp_bwd(m.critic, q, m.layers(m.critic, q), self.x_cur, ld, self.acts_q[k], self.d_out[k], self.part_c, B)
        ops.reduce_splits(self.part_c, m.critic.grad, m.critic.n, self.n_splits)
        self._adam(1, m.critic.flat, m.critic.grad, m.critic.exp_avg, m.critic.exp_avg_sq, m.critic.n)
        # ---- update_actor_and_alpha (every policy_frequency-th update), on the updated critic
        if actor_step:
            self._mlp_fwd(actor_l, self.x_pi, ld, D, self.acts_a, B)
            ops.sac_squash_fwd(self.acts_a[-1], B, A, m.log_std_bounds, self._tb_get('noise_actor'), self.seed, self.rng_ctr, ops.SAC_SITE_ACTOR,
                               self.act_box, self.log_action_scale_sum, dst=self.x_pi[:, D:], dst_ld=ld, eps_out=self.eps_pi,
                               logp=self.logp_pi)
            for k, q in enumerate(('Q1.', 'Q2.')):
                self._mlp_fwd(m.layers(m.critic, q), self.x_pi, ld, ld, self.acts_q[k], B)
            ops.sac_actor_loss(self.acts_q[0][-1], self.acts_q[1][-1], self.logp_pi, m.log_alpha, MIN_ALPHA, self.target_entropy,
                               self.learnable_temperature, B, self.d_out[0], self.d_out[1], m.log_alpha_grad, stats_row)
            for k, q in enumerate(('Q1.', 'Q2.')):       # critic weights get no update from this pass: input gradients only
                self._mlp_bwd(m.critic, q, m.layers(m.critic, q), self.x_pi, ld, self.acts_q[k], self.d_out[k], None, B,
                              dx_out=self.dx_in[k], weights=False)
            ops.sac_squash_bwd(self.acts_a[-1], self.eps_pi, B, A, m.log_std_bounds, self.act_box, self.dx_in[0][:, D:], self.dx_in[1][:, D:],
                               ld, m.log_alpha, MIN_ALPHA, self.d_head)
            self._mlp_bwd(m.actor, '', actor_l, self.x_pi, ld, self.acts_a, self.d_head, self.part_a, B)
            ops.reduce_splits(self.part_a, m.actor.grad, m.actor.n, self.n_splits)
            self._adam(0, m.actor.flat, m.actor.grad, m.actor.exp_avg, m.actor.exp_avg_sq, m.actor.n)
            if self.learnable_temperature:
                self._adam(2, m.log_alpha, m.log_alpha_grad, m.log_alpha_m, m.log_alpha_v, 1)
        # ---- update_target_weights (post-step critic); info/alpha = alpha after this update
        ops.sac_polyak(m.critic_target.flat, m.critic.flat, self.critic_tau, m.log_alpha, stats_row[5:6] if actor_step else None)
        ops.bump_u64(self.rng_ctr)

    def update(self, stats_row):
        self.update_counter += 1
        actor_step = self.update_counter % self.policy_frequency == 0
        if self.tapes is not None:
            self._fill_update_tapes(actor_step)
        if not self.use_graph:
            self._update(stats_row, actor_step)
            return actor_step
        key = (actor_step, self.tapes is not None)
        g = self._graphs.get(key)
        if g is None:
            # capture on a side stream; the captured update writes a fixed stats row that is copied out after each replay
            self._graph_row = self.stats[-1]
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=s):
                    self._update(self._graph_row, actor_step)
            torch.cuda.current_stream().wait_stream(s)
            self._graphs[key] = g
            # capture recorded the launches without running them: run this update for real
        g.replay()
        if actor_step:
            stats_row.copy_(self._graph_row)
        else:
            stats_row[:3].copy_(self._graph_row[:3])      # a critic-only update writes the critic columns only
        return actor_step

    # =============================================================================== env plumbing
    def _to_dev(self, x, dtype=torch.float32):
        if isinstance(x, np.ndarray):
            x = torch.from_numpy(x)
        return x.to(self.device_t, dtype=dtype)

    def _obs(self, obs):
        if isinstance(obs, dict):
            obs = obs['obs']
        return self._to_dev(obs).contiguous()

    def _update_obs_stats(self, obs):
        if not self.normalize_input:
            return
        r = self.model.running_mean_std
        ops.moments_update(obs, self.D, obs.shape[0], 1, 0, r.running_mean, r.running_var, r.count, r.mean_f32, r.std_f32,
                           self.rms_scratch, self.rms_counter)

    def env_reset(self):
        raw = self.vec_env.reset()
        self._tensor_env = isinstance(raw['obs'] if isinstance(raw, dict) else raw, torch.Tensor)
        obs = self._obs(raw)
        self._update_obs_stats(obs)
        self.prev_dones.zero_()
        return obs

    def _act(self, obs, random_exploration):
        m, N = self.model, self.num_actors
        if random_exploration:
            ops.sac_uniform_actions(self.action_low, self.action_high, self._tape('u'), self.seed, self.roll_ctr, self.actions, N, self.A)
        else:
            norm = (m.running_mean_std.mean_f32, m.running_mean_std.std_f32) if self.normalize_input else None
            self._mlp_fwd(m.layers(m.actor), obs, self.D, self.D, self.roll_acts, N, norm=norm, fp32=True)
            ops.sac_squash_fwd(self.roll_acts[-1], N, self.A, m.log_std_bounds, self._tape('noise_roll'), self.seed, self.roll_ctr,
                               ops.SAC_SITE_ROLLOUT, self.act_box, 0.0, dst=self.actions, dst_ld=self.A)
        ops.bump_u64(self.roll_ctr)
        return self.actions

    def _store(self, obs, action, rewards, next_obs, dones, infos):
        """_store_transitions: shaped reward, terminated / truncated split, the replay write and the episode accounting, on the device"""
        shaped = self._to_dev(self.rewards_shaper(self._to_dev(rewards))).reshape(-1).contiguous()
        d8 = self._to_dev(dones, torch.uint8).reshape(-1).contiguous()
        tout = None
        if self.value_bootstrap and isinstance(infos, dict) and 'time_outs' in infos:
            tout = self._to_dev(infos['time_outs']).ne(0).to(torch.uint8).reshape(-1).contiguous()
        # the reference's done_indices: done rows, and under next_step only the live ones (read before the insert moves prev_dones on)
        done_rows = d8.bool() & (self.prev_dones == 0) if self.autoreset_mode == 'next_step' else d8.bool()
        done_idx = done_rows.nonzero(as_tuple=False)
        final = None
        if self.autoreset_mode != 'next_step' and isinstance(infos, dict) and infos.get('final_observation') is not None:
            final = self._to_dev(infos['final_observation']).contiguous()
        ops.sac_replay_insert(obs, action, shaped, next_obs, final, d8, tout, self.value_bootstrap, self.autoreset_mode == 'next_step',
                              self.prev_dones, self.rb, self.slot, self.term_s, self.trunc_s, self.ep_state, self.meter, self.games_to_track)
        return done_idx

    # =============================================================================== epoch (sac_agent.py play_steps / train_epoch)
    def play_steps(self, random_exploration=False):
        t_start = time.perf_counter()
        step_time = update_time = 0.0
        obs = self.obs
        n_upd = 0
        actor_rows = []
        for _ in range(self.num_steps_per_episode):
            action = self._act(obs, random_exploration)
            t0 = time.perf_counter()
            # the env gets a copy: the action buffer is rewritten by the next step's sampler
            env_actions = action.clone() if self._tensor_env else action.cpu().numpy()
            next_obs_raw, rewards, dones, infos = self.vec_env.step(env_actions)
            step_time += time.perf_counter() - t0
            next_obs = self._obs(next_obs_raw)
            self._update_obs_stats(next_obs)
            done_idx = self._store(obs, action, rewards, next_obs, dones, infos)
            self.algo_observer.process_infos(infos, done_idx)
            obs = self.obs = next_obs
            if not random_exploration:
                t1 = time.perf_counter()
                for _ in range(self.num_updates_per_step):
                    if self.update(self.stats[n_upd]):
                        actor_rows.append(n_upd)
                    n_upd += 1
                update_time += time.perf_counter() - t1
        total = time.perf_counter() - t_start
        return step_time, total - update_time, update_time, total, n_upd, actor_rows

    def train_epoch(self):
        random_exploration = self.epoch_num <= self.num_warmup_steps
        return self.play_steps(random_exploration)

    def _epoch_losses(self, n_upd, actor_rows):
        """per-epoch means of the per-update losses (torch_ext.mean_list), one host read"""
        st = self.stats[:n_upd].cpu()
        out = {'c1_loss': float(st[:, 1].mean()), 'c2_loss': float(st[:, 2].mean())}
        if actor_rows:
            a = st[actor_rows]
            out['a_loss'] = float(a[:, 3].mean())
            out['entropy'] = float(a[:, 4].mean())
            if self.learnable_temperature:
                out['alpha_loss'] = float(a[:, 6].mean())
                out['alpha'] = float(a[:, 5].mean())
        return out

    def game_stats(self):
        """(size, mean reward, mean length) of the episode meter"""
        mh = self.meter.cpu().numpy()
        return int(mh[2]), float(mh[0]), float(mh[1])

    def clear_stats(self):
        self.meter.zero_()
        self.mean_rewards = -float('inf')
        self.algo_observer.after_clear_stats()

    def train(self):
        self.init_tensors()
        self.algo_observer.after_init(self)
        total_time = 0
        self.obs = self.env_reset()
        while True:
            self.epoch_num += 1
            step_time, play_time, update_time, epoch_time, n_upd, actor_rows = self.train_epoch()
            total_time += epoch_time
            curr = self.num_frames_per_epoch
            self.frame += curr
            if self.print_stats:
                print(f'fps step: {curr / max(step_time, 1e-9):.0f} fps step and policy inference: {curr / max(play_time, 1e-9):.0f} '
                      f'fps total: {curr / max(epoch_time, 1e-9):.0f} epoch: {self.epoch_num}/{self.max_epochs} frames: {self.frame}')
            w = self.writer
            w.add_scalar('performance/step_inference_rl_update_fps', curr / max(epoch_time, 1e-9), self.frame)
            w.add_scalar('performance/step_inference_fps', curr / max(play_time, 1e-9), self.frame)
            w.add_scalar('performance/step_fps', curr / max(step_time, 1e-9), self.frame)
            w.add_scalar('performance/rl_update_time', update_time, self.frame)
            w.add_scalar('performance/step_inference_time', play_time, self.frame)
            w.add_scalar('performance/step_time', step_time, self.frame)
            if self.epoch_num > self.num_warmup_steps and n_upd > 0:
                ls = self._epoch_losses(n_upd, actor_rows)
                for k in ('a_loss', 'c1_loss', 'c2_loss', 'entropy', 'alpha_loss'):
                    if k in ls:
                        w.add_scalar('losses/' + k, ls[k], self.frame)
                if 'alpha' in ls:
                    w.add_scalar('info/alpha', ls['alpha'], self.frame)
            w.add_scalar('info/epochs', self.epoch_num, self.frame)
            self.algo_observer.after_print_stats(self.frame, self.epoch_num, total_time)
            should_exit = False
            mean_rewards = -np.inf
            size, mr, ml = self.game_stats()
            if size > 0:
                mean_rewards = np.float32(mr)
                w.add_scalar('rewards/step', mr, self.frame)
                w.add_scalar('rewards/time', mr, total_time)
                w.add_scalar('episode_lengths/step', ml, self.frame)
                w.add_scalar('episode_lengths/time', ml, total_time)
                if mean_rewards > self.last_mean_rewards and self.epoch_num >= self.save_best_after:
                    print('saving next best rewards: ', mean_rewards)
                    self.last_mean_rewards = mean_rewards
                    self.save(os.path.join(self.nn_dir, self.config['name']))
                    if self.last_mean_rewards > self.config.get('score_to_win', float('inf')):
                        print('Maximum reward achieved. Network won!')
                        self.save(os.path.join(self.nn_dir, self.config['name'] + '_ep_' + str(self.epoch_num) + '_rew_' + str(mean_rewards)))
                        should_exit = True
            checkpoint_name = self.config['name'] + '_ep_' + str(self.epoch_num) + '_rew_' + str(mean_rewards)
            if self.save_freq > 0 and self.epoch_num % self.save_freq == 0:
                self.save(os.path.join(self.nn_dir, 'last_' + checkpoint_name))
            if self.epoch_num >= self.max_epochs and self.max_epochs != -1:
                self.save(os.path.join(self.nn_dir, 'last_' + self.config['name'] + '_ep_' + str(self.epoch_num)
                                       + '_rew_' + str(mean_rewards).replace('[', '_').replace(']', '_')))
                print('MAX EPOCHS NUM!')
                should_exit = True
            if self.frame >= self.max_frames and self.max_frames != -1:
                self.save(os.path.join(self.nn_dir, 'last_' + self.config['name'] + '_frame_' + str(self.frame)
                                       + '_rew_' + str(mean_rewards).replace('[', '_').replace(']', '_')))
                print('MAX FRAMES NUM!')
                should_exit = True
            if not should_exit and self.stop_fn is not None and self.stop_fn(self):
                self.save(os.path.join(self.nn_dir, 'last_' + self.config['name'] + '_custom_stop_ep_' + str(self.epoch_num)))
                print('Custom stop callback returned True. Stopping training.')
                should_exit = True
            if should_exit:
                return self.last_mean_rewards, self.epoch_num

    # =============================================================================== weights / checkpoints
    def get_weights(self):
        m = self.model
        state = {'actor': m.part_state_dict(m.actor), 'critic': m.part_state_dict(m.critic), 'critic_target': m.part_state_dict(m.critic_target)}
        if self.normalize_input:
            state['running_mean_std'] = m.running_mean_std.state_dict('')
        return state

    def set_weights(self, weights):
        m = self.model
        m.load_part_state_dict(m.actor, weights['actor'])
        m.load_part_state_dict(m.critic, weights['critic'])
        m.load_part_state_dict(m.critic_target, weights['critic_target'])
        if self.normalize_input and 'running_mean_std' in weights:
            m.running_mean_std.load_state_dict(weights['running_mean_std'], '')

    def _opt_steps(self):
        return [int(s) for s in self.opt_state[:, 1].cpu().tolist()]

    def get_full_state_weights(self):
        m = self.model
        state = self.get_weights()
        state['epoch'] = self.epoch_num
        state['frame'] = self.frame
        sa, sc, sl = self._opt_steps()
        state['actor_optimizer'] = m.adam_state_dict(m.actor.views(m.actor.exp_avg), m.actor.views(m.actor.exp_avg_sq), sa, self.lrs[0],
                                                     self.betas[0])
        state['critic_optimizer'] = m.adam_state_dict(m.critic.views(m.critic.exp_avg), m.critic.views(m.critic.exp_avg_sq), sc, self.lrs[1],
                                                      self.betas[1])
        state['log_alpha_optimizer'] = m.adam_state_dict([m.log_alpha_m.reshape(())], [m.log_alpha_v.reshape(())], sl, self.lrs[2],
                                                         self.betas[2])
        state['log_alpha'] = m.log_alpha.detach().reshape(()).cpu().clone()
        state['last_mean_rewards'] = self.last_mean_rewards
        if self.vec_env is not None and hasattr(self.vec_env, 'get_env_state'):
            state['env_state'] = self.vec_env.get_env_state()
        if self.save_replay_buffer:
            st = self.rb['state'].cpu()
            idx, fill = int(st[0]), int(st[1])
            state['replay_buffer'] = {'obses': self.rb['obs'].cpu(), 'next_obses': self.rb['next'].cpu(), 'actions': self.rb['act'].cpu(),
                                      'rewards': self.rb['rew'].cpu().unsqueeze(1), 'dones': self.rb['term'].cpu().bool().unsqueeze(1),
                                      'truncated': self.rb['trunc'].cpu().bool().unsqueeze(1), 'idx': idx,
                                      'full': fill == self.replay_buffer_size}
        cm = self.config.get('capability_manifest')
        if cm is not None:
            state['capability_manifest'] = cm
        return state

    def _load_adam(self, i, ms, vs, osd, lr_default):
        m = self.model
        step = m.load_adam_state_dict(ms, vs, osd)
        b1, b2 = self.betas[i]
        self.opt_state[i].zero_()
        lr = osd['param_groups'][0]['lr'] if osd.get('param_groups') else lr_default
        self.opt_state[i, 0] = float(lr)
        if step > 0:
            self.opt_state[i, 1] = float(step)
            self.opt_state[i, 2] = b1 ** step
            self.opt_state[i, 3] = b2 ** step

    def set_full_state_weights(self, weights, set_epoch=True):
        m = self.model
        self.set_weights(weights)
        if set_epoch:
            self.epoch_num = weights['epoch']
            self.frame = weights['frame']
        self._load_adam(0, m.actor.views(m.actor.exp_avg), m.actor.views(m.actor.exp_avg_sq), weights['actor_optimizer'], self.lrs[0])
        self._load_adam(1, m.critic.views(m.critic.exp_avg), m.critic.views(m.critic.exp_avg_sq), weights['critic_optimizer'], self.lrs[1])
        self._load_adam(2, [m.log_alpha_m.reshape(())], [m.log_alpha_v.reshape(())], weights['log_alpha_optimizer'], self.lrs[2])
        if 'log_alpha' in weights:
            m.log_alpha.copy_(weights['log_alpha'].reshape(1).to(self.device_t))
        self.last_mean_rewards = weights.get('last_mean_rewards', -float('inf'))
        if 'replay_buffer' in weights:
            rb = weights['replay_buffer']
            self.rb['obs'].copy_(rb['obses']); self.rb['next'].copy_(rb['next_obses']); self.rb['act'].copy_(rb['actions'])     # noqa: E702
            self.rb['rew'].copy_(rb['rewards'].reshape(-1)); self.rb['term'].copy_(rb['dones'].reshape(-1))                      # noqa: E702
            self.rb['trunc'].copy_(rb['truncated'].reshape(-1))
            cap = self.replay_buffer_size
            self.rb['state'].copy_(torch.tensor([int(rb['idx']), cap if rb['full'] else int(rb['idx'])], dtype=torch.int64))
        if self.vec_env is not None and hasattr(self.vec_env, 'set_env_state'):
            self.vec_env.set_env_state(weights.get('env_state', None))
        if 'capability_manifest' in weights:
            declared = self.config.get('capability_manifest')
            if declared is not None and declared != weights['capability_manifest']:
                print('WARNING: config capability_manifest differs from the checkpoint one; keeping the config value')
            else:
                self.config['capability_manifest'] = weights['capability_manifest']

    def save(self, fn):
        torch.save(self.get_full_state_weights(), fn + '.pth')

    def restore(self, fn, set_epoch=True):
        if not os.path.exists(fn):
            raise FileNotFoundError(f'Checkpoint file not found: {fn}')
        checkpoint = torch.load(fn, map_location=self.device_t, weights_only=False)
        self.set_full_state_weights(checkpoint, set_epoch=set_epoch)

    def get_param(self, param_name):
        pass

    def set_param(self, param_name, param_value):
        pass

    def set_eval(self):
        pass

    def set_train(self):
        pass
