"""Synthetic measurement environments (SURVEY.md 8d) behind the reference's IVecEnv contract
(common/ivecenv.py): step(actions) -> (obs, rewards, dones, infos), reset() -> obs, get_env_info().

The reference has no on-GPU synthetic env (its `test_env` is a CPU numpy gym env behind Ray), so these
are new fixtures, registered through the same registries a stock YAML would name:

    env_name: b200_synthetic          (vecenv_type B200_SYNTHETIC)      -- on-GPU, same_step autoreset
    env_name: b200_synthetic_host     (vecenv_type B200_SYNTHETIC_HOST) -- numpy/pinned-host edition used for
                                                                          the end-to-end (H2D/D2H) bench leg

obs ~ N(0,1) (Philox4x32-10), reward = -||a||^2, done = (t >= max_len) | Bernoulli(p_done),
infos['time_outs'] = (t >= max_len) & ~terminated.
"""
import numpy as np
import torch

from . import ops
from .common import IVecEnv, Box, register_vecenv, register_env


class SyntheticGPUEnv(IVecEnv):
    """Tensor env: everything stays on the training device, one kernel launch per step, static output
    buffers (so a whole rollout is CUDA-graph capturable: `cuda_graph_capturable = True`)."""
    cuda_graph_capturable = True

    def __init__(self, config_name, num_actors, obs_dim=60, act_dim=8, max_len=100, p_done=0.01, seed=5,
                 device='cuda:0', autoreset_mode='same_step', agents=1, **kwargs):
        # agents > 1: a multi-agent env of num_actors envs whose rows are num_actors * agents independent agent rows
        self.agents = int(agents)
        self.N, self.D, self.A = int(num_actors) * self.agents, int(obs_dim), int(act_dim)
        self.max_len, self.p_done, self._seed = int(max_len), float(p_done), int(seed)
        self.device = torch.device(device)
        self.autoreset_mode = autoreset_mode
        dev = self.device
        self.obs = torch.empty(self.N, self.D, device=dev)
        self.rewards = torch.empty(self.N, device=dev)
        self.dones = torch.zeros(self.N, dtype=torch.uint8, device=dev)
        self.time_outs = torch.zeros(self.N, dtype=torch.uint8, device=dev)
        self.ep_t = torch.zeros(self.N, dtype=torch.int32, device=dev)
        self.rng_epoch = torch.zeros(1, dtype=torch.int64, device=dev)
        self.step_index = 0
        self.infos = {'time_outs': self.time_outs}

    def seed(self, seed):
        self._seed = int(seed)

    def reset(self):
        self.ep_t.zero_()
        ops.synth_env_step(None, self.obs, self.rewards, self.dones, self.time_outs, self.ep_t, self.N, self.D, self.A,
                           1 << 30, 0.0, self._seed, self.rng_epoch, 1023)
        self.ep_t.zero_()
        self.step_index = 0
        return self.obs

    def begin_rollout(self):
        """Called by the agent at the start of every rollout: step indices restart (they are baked into
        captured graphs), the epoch counter (device memory) advances instead."""
        self.step_index = 0

    def end_rollout(self):
        ops.bump_u64(self.rng_epoch)

    def step(self, actions):
        ops.synth_env_step(actions, self.obs, self.rewards, self.dones, self.time_outs, self.ep_t, self.N, self.D, self.A,
                           self.max_len, self.p_done, self._seed, self.rng_epoch, self.step_index)
        self.step_index += 1
        return self.obs, self.rewards, self.dones, self.infos

    def get_env_info(self):
        info = {'observation_space': Box(-np.inf, np.inf, (self.D,)), 'action_space': Box(-1.0, 1.0, (self.A,))}
        if self.autoreset_mode != 'same_step':
            info['autoreset_mode'] = self.autoreset_mode
        if self.agents > 1:
            info['agents'] = self.agents
        return info


class SyntheticHostEnv(IVecEnv):
    """numpy edition (obs/rewards/dones live in HOST memory like envpool / gymnasium vector envs): every
    step costs an H2D copy of obs/rewards/dones and a D2H copy of the actions -- the end-to-end leg.
    The observation stream is pre-generated into a ring so host RNG speed does not enter the measurement."""

    def __init__(self, config_name, num_actors, obs_dim=60, act_dim=8, max_len=100, p_done=0.01, seed=5, ring=32,
                 **kwargs):
        self.N, self.D, self.A = int(num_actors), int(obs_dim), int(act_dim)
        self.max_len, self.p_done = int(max_len), float(p_done)
        rng = np.random.default_rng(seed)
        # page-locked ring (like envpool's output buffers): numpy views of pinned torch storage, so H2D copies need no staging
        self._ring_t = []
        self.ring = []
        for _ in range(ring):
            t = torch.empty(self.N, self.D, dtype=torch.float32)
            try:
                t = t.pin_memory()
            except Exception:
                pass
            t.copy_(torch.from_numpy(rng.standard_normal((self.N, self.D), dtype=np.float32)))
            self._ring_t.append(t)
            self.ring.append(t.numpy())
        self.term = [(rng.random(self.N) < self.p_done) for _ in range(ring)]
        self.i = 0
        self.t = np.zeros(self.N, dtype=np.int32)

    def reset(self):
        self.t[:] = 0
        self.i = 0
        return self.ring[0]

    def step(self, actions):
        rew = -np.einsum('ij,ij->i', actions, actions).astype(np.float32)
        self.i = (self.i + 1) % len(self.ring)
        self.t += 1
        to = self.t >= self.max_len
        term = self.term[self.i]
        done = to | term
        self.t[done] = 0
        return self.ring[self.i], rew, done.astype(np.uint8), {'time_outs': (to & ~term)}

    def get_env_info(self):
        return {'observation_space': Box(-np.inf, np.inf, (self.D,)), 'action_space': Box(-1.0, 1.0, (self.A,))}


register_vecenv('B200_SYNTHETIC', lambda config_name, num_actors, **kw: SyntheticGPUEnv(config_name, num_actors, **kw))
register_vecenv('B200_SYNTHETIC_HOST', lambda config_name, num_actors, **kw: SyntheticHostEnv(config_name, num_actors, **kw))
register_env('b200_synthetic', {'vecenv_type': 'B200_SYNTHETIC'})
register_env('b200_synthetic_host', {'vecenv_type': 'B200_SYNTHETIC_HOST'})
