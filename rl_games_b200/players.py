"""Players: run a trained policy in an env on the CUDA path -- mirror of rl_games.common.player.BasePlayer and
rl_games.algos_torch.players (PpoPlayerContinuous, PpoPlayerDiscrete, SACPlayer).

Same constructor (``Player(params)``), config keys (``player: {games_num, n_game_life, deterministic, print_stats, render,
render_sleep, balance_env_rewards, use_vecenv, env_config}``), ``run()`` loop and printed lines as the reference's players, and the same
checkpoints (``restore(fn)``).  The policy is evaluated by the forward code of the training agents themselves -- ``A2CAgent._policy_step``
/ ``_lstm_step`` / ``_trunk``, ``DiscreteA2CAgent._forward`` / ``_conv_forward``, ``SACAgent._act`` -- run on the player's own buffers
(one step of N = the detected batch rows), so a policy is played in the arithmetic its rollout was trained with: the precision keys
(``mixed_precision``, ``b200_rollout_fp32``) resolve as in the agent.  Deterministic actions are ``mu`` (a zero noise tape through the
Gaussian head kernels, which also apply the clamp and the env rescale), ``tanh(mu)`` rescaled and clamped for SAC (a zero noise tape
through ``sac_squash_fwd``) and the per-head argmax of the masked logits (``categorical_argmax``).  Sampled actions come from the
rollout's Philox streams, keyed as the agents key them (PPO: ``b200_rng_seed``, else ``seed``; SAC: ``seed``) with the player's step
counter as the counter.

With ``b200_cuda_graph`` (default True) one player step -- normalisation, trunk, LSTM step, head, action write, and the zeroing of the
recurrent state rows the previous step finished -- is captured once per batch size and replayed; the observation and the actions live
in static device buffers, and the host-to-device copy of the observations and the device-to-host copy of the actions stay outside the
graph.
"""
import time

import numpy as np
import torch

from . import ops
from .agent import A2CAgent, rollout_precision
from .agent_discrete import DiscreteA2CAgent, DiscreteModel, discrete_spaces
from .agent_sac import SACAgent
from .common import configurations, create_vec_env
from .layerwise import Kernels
from .model import B200Model, _RunningStats, resolve_device
from .model_sac import SACModel


def unsqueeze_obs(obs):
    """tr_helpers.py:71-78"""
    if len(obs.size()) > 1 or obs.size()[0] > 1:
        obs = obs.unsqueeze(0)
    return obs


def _create_env(name, env_config):
    """env_configurations.configurations[name]['env_creator'](**env_config), in this package's registry first, then in the reference's"""
    if name in configurations and 'env_creator' in configurations[name]:
        env = configurations[name]['env_creator'](**env_config)
        return env, _env_info(env)
    try:
        from rl_games.common import env_configurations as reference_configurations
    except ImportError:
        raise KeyError(f"env '{name}' has no 'env_creator' in rl_games_b200.common.configurations and rl_games is not importable to "
                       f"look it up there") from None
    env = reference_configurations.configurations[name]['env_creator'](**env_config)
    return env, reference_configurations.get_env_info(env)


def _env_info(env):
    """env_configurations.get_env_info (env_configurations.py:328-347)"""
    info = {'observation_space': env.observation_space, 'action_space': env.action_space, 'agents': 1, 'value_size': 1}
    if hasattr(env, 'get_number_of_agents'):
        info['agents'] = env.get_number_of_agents()
    if hasattr(env, 'value_size'):
        info['value_size'] = env.value_size
    return info


class BasePlayer:
    """common/player.py BasePlayer: env creation, config keys, the run() loop; the subclasses own the model and the step"""

    def __init__(self, params):
        self.params = params
        self.config = config = params['config']
        self.network_params = params['network']
        self.env_name = config['env_name']
        self.player_config = config.get('player', {})
        self.env_config = config.get('env_config', {})
        self.env_config = self.player_config.get('env_config', self.env_config)
        self.env_info = config.get('env_info')
        self.clip_actions = config.get('clip_actions', True)
        self.env_seed = self.env_config.pop('seed', None)
        self.balance_env_rewards = self.player_config.get('balance_env_rewards', False)
        self.evaluation = self.player_config.get('evaluation', False)
        self.dir_to_monitor = self.player_config.get('dir_to_monitor')
        if self.evaluation and self.dir_to_monitor is not None:
            raise NotImplementedError('player.evaluation with player.dir_to_monitor: the evaluation checkpoint watcher needs the '
                                      '`watchdog` package, which the CUDA players do not use; restore a checkpoint and run() instead')
        if self.env_info is None:
            if self.player_config.get('use_vecenv', False):
                print('[BasePlayer] Creating vecenv: ', self.env_name)
                self.env = create_vec_env(self.env_name, config['num_actors'], **self.env_config)
                self.env_info = self.env.get_env_info()
            else:
                print('[BasePlayer] Creating regular env: ', self.env_name)
                self.env, self.env_info = _create_env(self.env_name, self.env_config)
        else:
            self.env = config.get('vec_env')
        self.num_agents = self.env_info.get('agents', 1)
        self.value_size = self.env_info.get('value_size', 1)
        if self.value_size != 1:
            raise NotImplementedError('value_size > 1 is not supported by the CUDA players')
        self.action_space = self.env_info['action_space']
        self.observation_space = self.env_info['observation_space']
        if type(self.observation_space).__name__ == 'Dict':
            raise NotImplementedError('Dict observation spaces are not supported by the CUDA players')
        self.obs_shape = self.observation_space.shape
        self.is_tensor_obses = False
        self.states = None
        self.batch_size = 1
        self.has_batch_dimension = False
        self.has_central_value = config.get('central_value_config') is not None
        self.device_name = config.get('device_name', 'cuda')
        self._require_cuda()
        self.device = resolve_device(self.device_name)
        self.render_env = self.player_config.get('render', False)
        self.games_num = self.player_config.get('games_num', 1000000000)
        self.is_deterministic = self.player_config.get('deterministic', True)
        self.n_game_life = self.player_config.get('n_game_life', 1)
        self.print_stats = self.player_config.get('print_stats', True)
        self.render_sleep = self.player_config.get('render_sleep', 0.002)
        self.max_steps = 108000 // 4
        self.use_cuda_graph = bool(config.get('b200_cuda_graph', True))
        self.rng_seed = int(config.get('b200_rng_seed', params.get('seed', 0) or 0))
        self.is_rnn = False
        self.num_rows = 0           # rows of the allocated step buffers (the detected batch size)
        self._graphs = {}

    def _require_cuda(self):
        """no CPU fallback: the kernels are the product (the host-logic tests replace this hook together with every op)"""
        if not str(self.device_name).startswith('cuda'):
            raise RuntimeError('rl_games_b200 players run on CUDA only (device_name=%r): there is no CPU fallback' % self.device_name)
        torch.cuda.set_device(resolve_device(self.device_name))

    # ------------------------------------------------------------------------------------------------ env plumbing (player.py)
    def env_step(self, env, actions):
        if not self.is_tensor_obses:
            actions = actions.cpu().numpy()
        obs, rewards, dones, infos = env.step(actions)
        if hasattr(obs, 'dtype') and obs.dtype == np.float64:
            obs = np.float32(obs)
        if self.is_tensor_obses:
            return self.obs_to_torch(obs), rewards.cpu(), dones.cpu(), infos
        if np.isscalar(dones):
            rewards = np.expand_dims(np.asarray(rewards), 0)
            dones = np.expand_dims(np.asarray(dones), 0)
        return self.obs_to_torch(obs), torch.from_numpy(rewards), torch.from_numpy(dones), infos

    def obs_to_torch(self, obs):
        if isinstance(obs, dict) and 'obs' in obs:
            obs = obs['obs']
        if isinstance(obs, dict):
            raise NotImplementedError('Dict observations are not supported by the CUDA players')
        return self.cast_obs(obs)

    def cast_obs(self, obs):
        if isinstance(obs, torch.Tensor):
            self.is_tensor_obses = True
        elif isinstance(obs, np.ndarray):
            assert obs.dtype != np.int8
            obs = torch.from_numpy(obs).to(self.device, torch.uint8 if obs.dtype == np.uint8 else torch.float32)
        elif np.isscalar(obs):
            obs = torch.tensor([obs], dtype=torch.float32, device=self.device)
        return obs

    def env_reset(self, env):
        return self.obs_to_torch(env.reset())

    def get_batch_size(self, obses, batch_size):
        if len(obses.size()) > len(self.obs_shape):
            batch_size = obses.size()[0]
            self.has_batch_dimension = True
        self.batch_size = batch_size
        return batch_size

    def _load_checkpoint(self, fn):
        """torch_ext.load_checkpoint: strips `_orig_mod.` prefixes"""
        checkpoint = torch.load(fn, map_location=self.device, weights_only=False)
        if 'model' in checkpoint:
            checkpoint['model'] = {k.replace('_orig_mod.', ''): v for k, v in checkpoint['model'].items()}
        return checkpoint

    def _restore_env_state(self, checkpoint):
        env_state = checkpoint.get('env_state', None)
        if self.env is not None and env_state is not None:
            self.env.set_env_state(env_state)

    def restore(self, fn):
        checkpoint = self._load_checkpoint(fn)
        self.model.load_state_dict(checkpoint['model'])
        if self.normalize_input and 'running_mean_std' in checkpoint:
            self.model.running_mean_std.load_state_dict(checkpoint['running_mean_std'])
        self._weights_loaded()
        self._restore_env_state(checkpoint)

    def _weights_loaded(self):
        """refresh the device copies derived from the weights"""

    def get_weights(self):
        return {'model': self.model.state_dict()}

    def set_weights(self, weights):
        self.model.load_state_dict(weights['model'])
        if self.normalize_input and 'running_mean_std' in weights:
            self.model.running_mean_std.load_state_dict(weights['running_mean_std'])
        self._weights_loaded()

    def reset(self):
        self.init_rnn()

    def init_rnn(self):
        if self.is_rnn:
            self._ensure_rows(self.batch_size)
            self.rnn_h.zero_()
            self.rnn_c.zero_()
            self.done_dev.zero_()

    # ------------------------------------------------------------------------------------------------ one policy step
    def _ensure_rows(self, N):
        if N != self.num_rows:
            self.num_rows = N
            self._graphs = {}
            self._alloc(N)

    def _alloc(self, N):
        raise NotImplementedError

    def _step_body(self, deterministic):
        raise NotImplementedError

    def _graph_key(self, deterministic):
        return deterministic

    def _mutable(self):
        """the device state a step advances"""
        return [self.rng_epoch]

    def _run_step(self, deterministic):
        """the step on the static buffers: eager, or the replay of its graph (captured at the first step of this key)"""
        if not self.use_cuda_graph:
            self._step_body(deterministic)
            return
        key = self._graph_key(deterministic)
        g = self._graphs.get(key)
        if g is None:
            # one eager run first loads every kernel the step launches (a module load cannot happen inside a capture); the state it
            # advances (Philox counter, recurrent states) is put back, so the first step's result comes from the replay like every later one
            snap = [t.clone() for t in self._mutable()]
            self._step_body(deterministic)
            for t, v in zip(self._mutable(), snap):
                t.copy_(v)
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            g = torch.cuda.CUDAGraph()
            with torch.cuda.stream(s):
                with torch.cuda.graph(g, stream=s):
                    self._step_body(deterministic)
            torch.cuda.current_stream().wait_stream(s)
            self._graphs[key] = g
        g.replay()

    def _prepare_obs(self, obs):
        """the step's observation rows into the static input buffer (outside the graph)"""
        if not self.has_batch_dimension:
            obs = unsqueeze_obs(obs)
        N = obs.shape[0]
        self._ensure_rows(N)
        self.obs_buf.copy_(obs.reshape(N, -1))
        return N

    def _done_rows(self, done):
        """the finished rows of a step, for the recurrent-state zeroing at the start of the next step (on the device)"""
        if self.is_rnn:
            self.done_dev.copy_(done.reshape(-1).to(torch.uint8), non_blocking=True)

    # ------------------------------------------------------------------------------------------------ player.py BasePlayer.run
    def get_action(self, obs, is_deterministic=False):
        raise NotImplementedError('step')

    def get_masked_action(self, obs, mask, is_deterministic=False):
        raise NotImplementedError('step')

    def run(self):
        render = self.render_env
        n_game_life = self.n_game_life
        n_games = self.games_num * n_game_life
        is_deterministic = self.is_deterministic
        sum_rewards = 0
        sum_steps = 0
        sum_game_res = 0
        games_played = 0
        has_masks = False
        has_masks_func = getattr(self.env, 'has_action_mask', None) is not None
        if has_masks_func:
            has_masks = self.env.has_action_mask()
        need_init_rnn = self.is_rnn
        for _ in range(n_games):
            if games_played >= n_games:
                break
            obses = self.env_reset(self.env)
            batch_size = 1
            batch_size = self.get_batch_size(obses, batch_size)
            if need_init_rnn:
                self.init_rnn()
                need_init_rnn = False
            cr = torch.zeros(batch_size, dtype=torch.float32)
            steps = torch.zeros(batch_size, dtype=torch.float32)
            if self.balance_env_rewards:
                per_env_rewards = torch.zeros(batch_size, dtype=torch.float32)
                per_env_steps = torch.zeros(batch_size, dtype=torch.float32)
                per_env_game_res = torch.zeros(batch_size, dtype=torch.float32)
                per_env_games_played = torch.zeros(batch_size, dtype=torch.float32)
            print_game_res = False
            for n in range(self.max_steps):
                if has_masks:
                    masks = self.env.get_action_mask()
                    action = self.get_masked_action(obses, masks, is_deterministic)
                else:
                    action = self.get_action(obses, is_deterministic)
                obses, r, done, info = self.env_step(self.env, action)
                cr += r
                steps += 1
                self._done_rows(done)
                if render:
                    self.env.render(mode='human')
                    time.sleep(self.render_sleep)
                all_done_indices = done.nonzero(as_tuple=False)
                done_indices = all_done_indices[::self.num_agents]
                done_count = len(done_indices)
                games_played += done_count
                if done_count > 0:
                    game_res = 0.0
                    if isinstance(info, dict):
                        if 'battle_won' in info:
                            print_game_res = True
                            game_res = info.get('battle_won', 0.5)
                        if 'scores' in info:
                            print_game_res = True
                            game_res = info.get('scores', 0.5)
                    if self.balance_env_rewards:
                        per_env_rewards[done_indices] += cr[done_indices]
                        per_env_steps[done_indices] += steps[done_indices]
                        per_env_games_played[done_indices] += 1
                        if print_game_res:
                            per_env_game_res[done_indices] += game_res
                        cr[done_indices] = 0
                        steps[done_indices] = 0
                    else:
                        cur_rewards = cr[done_indices].sum().item()
                        cur_steps = steps[done_indices].sum().item()
                        cr = cr * (1.0 - done.float())
                        steps = steps * (1.0 - done.float())
                        sum_rewards += cur_rewards
                        sum_steps += cur_steps
                        sum_game_res += game_res
                        if self.print_stats:
                            cur_rewards_done = cur_rewards / done_count
                            cur_steps_done = cur_steps / done_count
                            if print_game_res:
                                print(f'reward: {cur_rewards_done:.2f} steps: {cur_steps_done:.1f} w: {game_res}')
                            else:
                                print(f'reward: {cur_rewards_done:.2f} steps: {cur_steps_done:.1f}')
                    if batch_size // self.num_agents == 1 or games_played >= n_games:
                        break
        if self.balance_env_rewards:
            valid_envs = per_env_games_played > 0
            per_env_avg_rewards = torch.zeros(batch_size, dtype=torch.float32)
            per_env_avg_steps = torch.zeros(batch_size, dtype=torch.float32)
            per_env_avg_game_res = torch.zeros(batch_size, dtype=torch.float32)
            per_env_avg_rewards[valid_envs] = per_env_rewards[valid_envs] / per_env_games_played[valid_envs]
            per_env_avg_steps[valid_envs] = per_env_steps[valid_envs] / per_env_games_played[valid_envs]
            overall_avg_reward = per_env_avg_rewards[valid_envs].mean().item()
            overall_avg_steps = per_env_avg_steps[valid_envs].mean().item()
            if print_game_res:
                per_env_avg_game_res[valid_envs] = per_env_game_res[valid_envs] / per_env_games_played[valid_envs]
                overall_winrate = per_env_avg_game_res[valid_envs].mean().item()
                print('av reward:', overall_avg_reward * n_game_life, 'av steps:', overall_avg_steps * n_game_life,
                      'winrate:', overall_winrate * n_game_life)
            else:
                print('av reward:', overall_avg_reward * n_game_life, 'av steps:', overall_avg_steps * n_game_life)
        else:
            print(sum_rewards)
            if print_game_res:
                print('av reward:', sum_rewards / games_played * n_game_life, 'av steps:', sum_steps / games_played * n_game_life,
                      'winrate:', sum_game_res / games_played * n_game_life)
            else:
                print('av reward:', sum_rewards / games_played * n_game_life, 'av steps:', sum_steps / games_played * n_game_life)


class PpoPlayerContinuous(BasePlayer):
    """algos_torch/players.py PpoPlayerContinuous on A2CAgent's rollout forward"""
    _trunk = A2CAgent._trunk
    _lstm_step = A2CAgent._lstm_step
    _policy_step = A2CAgent._policy_step
    _repack = A2CAgent._repack

    def __init__(self, params):
        super().__init__(params)
        config = self.config
        model_name = params.get('model', {}).get('name', 'continuous_a2c_logstd')
        if model_name != 'continuous_a2c_logstd':
            raise NotImplementedError(f"model '{model_name}': only continuous_a2c_logstd is on the B200 hot path")
        if len(self.obs_shape) != 1:
            raise NotImplementedError('only flat observations are on the B200 hot path')
        self.actions_num = self.action_space.shape[0]
        self.actions_low = torch.from_numpy(np.asarray(self.action_space.low).copy()).float().to(self.device)
        self.actions_high = torch.from_numpy(np.asarray(self.action_space.high).copy()).float().to(self.device)
        self.normalize_input = config['normalize_input']
        self.normalize_value = config.get('normalize_value', False)
        self.model = B200Model(self.network_params, self.obs_shape[0], self.actions_num, self.device, self.normalize_input,
                               self.normalize_value, self.value_size)
        self.is_rnn = self.model.is_rnn()
        if self.is_rnn and not config.get('zero_rnn_on_done', True):
            raise NotImplementedError('zero_rnn_on_done: False is not on the B200 hot path')
        _, self.use_tc, self.gemm_tc, self.rollout_fp32 = rollout_precision(self.model, self.actions_num, config)
        self.obs_norm = _RunningStats.f32_pair(self.model.running_mean_std)
        self.mlp_norm = (None, None) if (self.is_rnn and self.model.rnn_before_mlp) else self.obs_norm
        self.tc_wide = self.use_tc and ops.tc_kind(self.model.D, self.model.units, self.actions_num) == 2
        dev, m = self.device, self.model
        self.wbf = torch.empty(m.num_params, dtype=torch.bfloat16, device=dev) if self.gemm_tc else None
        self.kernels = Kernels(tc=self.gemm_tc, bf16_arena=(m.flat, self.wbf) if self.gemm_tc else None)
        self.wpack = torch.zeros(ops.tc_pack_bytes(m.D, m.units, self.actions_num), dtype=torch.uint8, device=dev) if self.use_tc else None
        self.rng_epoch = torch.zeros(1, dtype=torch.int64, device=dev)        # the Philox counter: one per player step
        self.prev_dones, self.valid = None, None
        self._tensors_ready = True
        self._weights_loaded()

    def _weights_loaded(self):
        self.model.refresh_sigma_floor()
        self._repack()

    def run(self):
        self._weights_loaded()          # the runner's `sigma` override writes the raw parameter after restore()
        super().run()

    def _alloc(self, N):
        """A2CAgent.init_tensors' rollout buffers for one step of N rows (arena time index 0)"""
        dev, m, A = self.device, self.model, self.actions_num
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)   # noqa: E731
        self.obs_buf = f(N, m.D)
        self.actions, self.mus, self.sigmas = f(1, N, A), f(1, N, A), f(1, N, A)
        self.neglogpacs, self.values = f(1, N), f(1, N)
        self.env_actions = f(N, A)
        self.dones = torch.zeros(N, dtype=torch.uint8, device=dev)
        self.dones_buf = torch.zeros(1, N, dtype=torch.uint8, device=dev)
        self.zero_noise = f(N, A)
        self.noise = None           # [N, A] normal tape for sampled actions (tests); None: the Philox stream
        self.ra = [f(N, u) for u in m.units] if (self.rollout_fp32 or not self.use_tc) else []
        self.tc_l1_scratch = (torch.zeros((N + 127) // 128 * ops.tc_tile_bytes(m.D, m.units, A)[0], dtype=torch.uint8, device=dev)
                              if self.tc_wide else None)
        if self.is_rnn:
            Hd = m.rnn_units
            self.rnn_h, self.rnn_c, self.r_gates = f(N, Hd), f(N, Hd), f(N, 4 * Hd)
            self.r_y = f(N, Hd) if m.rnn_layer_norm else None
            self.done_dev = torch.zeros(N, dtype=torch.uint8, device=dev)

    def _graph_key(self, deterministic):
        return deterministic, None if self.noise is None else self.noise.data_ptr()

    def _mutable(self):
        return [self.rng_epoch] + ([self.rnn_h, self.rnn_c] if self.is_rnn else [])

    def _step_body(self, deterministic):
        N = self.num_rows
        if self.is_rnn:     # the rows the previous step finished start from zero states (player.py run(): states[:, done] = 0)
            ops.rnn_mask_rows(self.rnn_h, N, 0, self.rnn_h, N, self.model.rnn_units, done=self.done_dev, done_rpc=N)
            ops.rnn_mask_rows(self.rnn_c, N, 0, self.rnn_c, N, self.model.rnn_units, done=self.done_dev, done_rpc=N)
        self._policy_step(self.obs_buf, 0, self.zero_noise if deterministic else self.noise)
        ops.bump_u64(self.rng_epoch)

    def get_action(self, obs, is_deterministic=False):
        self._prepare_obs(obs)
        self._run_step(is_deterministic)
        if self.is_rnn:
            self.states = [self.rnn_h.unsqueeze(0), self.rnn_c.unsqueeze(0)]
        current_action = self.env_actions
        if not self.has_batch_dimension:
            current_action = torch.squeeze(current_action)
        return current_action.clone()


class PpoPlayerDiscrete(BasePlayer):
    """algos_torch/players.py PpoPlayerDiscrete on DiscreteA2CAgent's forward"""
    _conv_out = staticmethod(DiscreteA2CAgent._conv_out)
    _conv_forward = DiscreteA2CAgent._conv_forward
    _forward = DiscreteA2CAgent._forward
    _repack = DiscreteA2CAgent._repack

    def __init__(self, params):
        super().__init__(params)
        config = self.config
        if self.has_central_value:
            raise NotImplementedError('central_value_config')
        (_, self.obs_dtype, self.head_sizes, self.actions_num, self.is_multi_discrete,
         self.mixed_precision) = discrete_spaces(self.observation_space, self.action_space, self.network_params, config)
        self.normalize_input = config['normalize_input']
        self.normalize_value = config.get('normalize_value', False)
        self.model = DiscreteModel(self.network_params, self.obs_shape, self.actions_num, self.device, self.normalize_input,
                                   self.normalize_value, head_sizes=self.head_sizes)
        self.is_rnn = False
        m = self.model
        self.wbf = torch.empty(m.num_params, dtype=torch.bfloat16, device=self.device) if self.mixed_precision else None
        self.kernels = Kernels(tc=True, bf16_arena=(m.flat, self.wbf)) if self.mixed_precision else Kernels()
        self.obs_norm = _RunningStats.f32_pair(m.running_mean_std)
        self.rng_epoch = torch.zeros(1, dtype=torch.int64, device=self.device)
        self._weights_loaded()

    def _weights_loaded(self):
        self._repack()

    def _alloc(self, N):
        """DiscreteA2CAgent.init_tensors' rollout buffers for one step of N rows"""
        dev, m, K = self.device, self.model, self.actions_num
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)   # noqa: E731
        self.obs_buf = torch.zeros(N, m.D, dtype=self.obs_dtype, device=dev)
        self.mask_buf = torch.ones(N, K, dtype=torch.uint8, device=dev)
        nh = len(self.head_sizes) if self.head_sizes else 1
        self.actions_out = torch.zeros(N, nh, dtype=torch.int64, device=dev)
        self.neglogp, self.values = f(N), f(N)
        self.u = None               # [n_heads, N] uniform tape for sampled actions (tests); None: the Philox stream
        self.r_a = [f(N, u) for u in m.units] + [f(N, K if m.separate else 1 + K)]
        if m.separate:
            self.r_c = [f(N, u) for u in m.units] + [f(N, 1)]
            self.r_out = (self.r_a[-1], K, self.r_c[-1], 1)
        else:
            self.r_c = None
            self.r_out = (self.r_a[-1][:, 1:], K + 1, self.r_a[-1], K + 1)
        if m.cnn:
            conv_bufs = lambda: [f(N, shp[0], *self._conv_out(g, shp)) for shp, g in m.cnn.layers]   # noqa: E731
            self.r_ka = conv_bufs()
            self.r_kc = conv_bufs() if m.separate else None
        else:
            self.r_ka = self.r_kc = None

    def _graph_key(self, deterministic):
        return deterministic, self._masked, None if self.u is None else self.u.data_ptr()

    def _step_body(self, deterministic):
        N, K, m = self.num_rows, self.actions_num, self.model
        self._forward(self.obs_buf, self.r_a, self.r_c, N, conv=(self.r_ka, self.r_kc))
        lg, ld, vl, vld = self.r_out
        masks = self.mask_buf if self._masked else None
        if deterministic:
            ops.categorical_argmax(lg, ld, K, masks, self.actions_out, N, head_sizes=self.head_sizes)
        else:
            vm = m.value_mean_std
            ops.categorical_sample(lg, ld, K, vl, vld, masks, self.u, self.rng_seed, self.rng_epoch, 0,
                                   None if vm is None else vm.running_mean, None if vm is None else vm.running_var, self.normalize_value,
                                   self.actions_out, self.neglogp, self.values, None, None, None, None, N, head_sizes=self.head_sizes)
        ops.bump_u64(self.rng_epoch)

    def _act(self, obs, action_masks, is_deterministic):
        N = self._prepare_obs(obs)
        self._masked = action_masks is not None
        if self._masked:
            self.mask_buf.copy_(torch.as_tensor(np.asarray(action_masks) if not torch.is_tensor(action_masks) else action_masks)
                                .reshape(N, -1).to(self.device, torch.uint8))
        self._run_step(is_deterministic)
        a = self.actions_out if self.is_multi_discrete else self.actions_out[:, 0]
        return a.squeeze().clone()

    def get_masked_action(self, obs, action_masks, is_deterministic=True):
        return self._act(obs, action_masks, is_deterministic)

    def get_action(self, obs, is_deterministic=False):
        return self._act(obs, None, is_deterministic)


class SACPlayer(BasePlayer):
    """algos_torch/players.py SACPlayer on SACAgent's rollout forward (fp32 kernels, as the agent's rollout)"""
    _act = SACAgent._act

    def __init__(self, params):
        super().__init__(params)
        if self.num_agents > 1:
            raise NotImplementedError("env_info['agents'] > 1: multi-agent SAC is not supported")
        if len(getattr(self.observation_space, 'shape', ()) or ()) != 1:
            raise NotImplementedError('SAC needs a flat Box observation space (CNN / dict observations are not supported)')
        if not hasattr(self.action_space, 'low') or len(self.action_space.shape) != 1:
            raise NotImplementedError('SAC supports continuous Box action spaces only (discrete action spaces are not supported)')
        self.actions_num = self.A = self.action_space.shape[0]
        self.D = self.obs_shape[0]
        dev = self.device
        self.action_low = torch.tensor(self.action_space.low, dtype=torch.float32).to(dev)
        self.action_high = torch.tensor(self.action_space.high, dtype=torch.float32).to(dev)
        self.action_scale = (self.action_high - self.action_low) / 2.0
        self.action_bias = (self.action_high + self.action_low) / 2.0
        self.act_box = (self.action_scale, self.action_bias, self.action_low, self.action_high)
        self.normalize_input = self.config.get('normalize_input', False)
        self.model = SACModel(self.network_params, self.D, self.A, dev, self.normalize_input, self.config.get('init_alpha', 1.0))
        self.seed = int(params.get('seed', 0) or 0) & 0xFFFFFFFFFFFFFFFF      # the agent's rollout stream key
        self.k32 = Kernels()
        self.obs_norm = _RunningStats.f32_pair(self.model.running_mean_std)
        self.roll_ctr = torch.zeros(1, dtype=torch.int64, device=dev)

    def restore(self, fn):
        checkpoint = self._load_checkpoint(fn)
        m = self.model
        m.load_part_state_dict(m.actor, checkpoint['actor'])
        m.load_part_state_dict(m.critic, checkpoint['critic'])
        m.load_part_state_dict(m.critic_target, checkpoint['critic_target'])
        if self.normalize_input and 'running_mean_std' in checkpoint:
            m.running_mean_std.load_state_dict(checkpoint['running_mean_std'])
        self._restore_env_state(checkpoint)

    def _alloc(self, N):
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.device)   # noqa: E731
        self.num_actors = N
        self.obs_buf = f(N, self.D)
        self.roll_acts = [f(N, w) for w in self.model.units] + [f(N, 2 * self.A)]
        self.actions = f(N, self.A)
        self.zero_noise = f(N, self.A)
        self.noise = None           # [N, A] normal tape for sampled actions (tests); None: the Philox stream
        self._deterministic = True

    def _tape(self, key):
        return self.zero_noise if self._deterministic else self.noise

    def _graph_key(self, deterministic):
        return deterministic, None if self.noise is None else self.noise.data_ptr()

    def _mutable(self):
        return [self.roll_ctr]

    def _step_body(self, deterministic):
        self._deterministic = deterministic
        self._act(self.obs_buf, False)

    def get_action(self, obs, is_deterministic=False):
        self._prepare_obs(obs)
        self._run_step(is_deterministic)
        actions = self.actions
        if not self.has_batch_dimension:
            actions = torch.squeeze(actions)
        return actions.clone()

    def reset(self):
        pass


def player_builders():
    """(algo name, builder) of every player: the reference's names for the three players"""
    return (('a2c_continuous', lambda **kwargs: PpoPlayerContinuous(**kwargs)),
            ('a2c_discrete', lambda **kwargs: PpoPlayerDiscrete(**kwargs)),
            ('sac', lambda **kwargs: SACPlayer(**kwargs)))
