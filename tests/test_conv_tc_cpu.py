"""The discrete agent's ``mixed_precision: True`` path (bf16 tensor-core convs and layer-wise GEMMs) on CPU, without the CUDA kernels:
- which C-ABI entry points the rollout and the update call, every call header-checked (tests/test_abi_calls_cpu.py's recorder): all conv
  and linear layers on the ``_tc`` entry points with ``True``; with ``False`` or no key, the call sequence the fp32 agent made before
  the tensor-core path existed (tests/golden/discrete_cnn_abi_seq.json, recorded at that commit by ``python tests/test_conv_tc_cpu.py``);
- the bf16 twin of the parameter arena after every point that changes the arena: an update, set_weights, a checkpoint restore;
- checkpoints in both directions between a tensor-core and an fp32 agent;
- the golden reference runs replayed through the kernel-faithful stand-ins of tests/_torch_ops_conv_tc.py;
- the reference's Pong YAML with ``mixed_precision: True`` through the reference's own Runner."""
import json
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import test_abi_calls_cpu as ABI  # noqa: E402
import test_cnn_cpu as CNN  # noqa: E402
import test_reference_runner_cpu as RR  # noqa: E402

GOLDENS = CNN.GOLDENS
SEQ_FILE = os.path.join(HERE, 'golden', 'discrete_cnn_abi_seq.json')
CONV_LINEAR = ('conv2d_fwd', 'conv2d_bwd_data', 'conv2d_bwd_weight', 'linear_fwd', 'linear_bwd_data', 'linear_bwd_weight')


def _make(monkeypatch, tmp_path, g, over=None, install=None):
    """the golden run's agent (tests/test_cnn_cpu.py) with the config overrides `over`; install(monkeypatch) replaces the ops"""
    from rl_games_b200.runner import Runner
    from rl_games_b200 import agent_discrete
    if install is not None:
        install(monkeypatch)
    monkeypatch.setattr(agent_discrete.DiscreteA2CAgent, '_require_cuda', lambda self: None)
    monkeypatch.setattr(agent_discrete.DiscreteA2CAgent, '_sync', staticmethod(lambda: None))
    env = CNN._FrameEnv(g)
    config = {k: v for k, v in g['config'].items() if k not in ('device', 'torch_compile', 'mixed_precision')}
    config.update({'device': 'cpu', 'env_info': env.get_env_info(), 'vec_env': env, 'reward_shaper': {'scale_value': 0.1},
                   'train_dir': str(tmp_path), 'lr_schedule': None})
    config.update(over or {})
    r = Runner()
    r.load({'params': {'seed': 1, 'algo': {'name': 'a2c_discrete'}, 'model': {'name': 'discrete_a2c'}, 'network': g['network'],
                       'config': config}})
    r.params['config']['vec_env'] = env
    agent = r.algo_factory.create(r.algo_name, base_name='cnn_tc', params=r.params)
    agent.model.load_state_dict(g['init_state'])
    agent.init_tensors()
    agent.obs = agent.env_reset()
    return agent


def _tc_stand_ins(monkeypatch):
    import _torch_ops_conv_tc
    _torch_ops_conv_tc.install_conv_tc(monkeypatch)


class _SeqRecorder(ABI._Recorder):
    """the header-checking recorder, keeping the order of the calls"""

    def __init__(self, real):
        super().__init__(real)
        self.seq = []

    def __getattr__(self, name):
        call = super().__getattr__(name)
        if name in ABI.HOST_ONLY:
            return call

        def rec(*args):
            self.seq.append(name)
            return call(*args)
        return rec


def _abi_sequence(monkeypatch, tmp_path, name, over):
    """the C-ABI calls of one train_epoch (rollout + update) of golden run `name` with config overrides `over`"""
    from rl_games_b200 import ops, _lib
    g = CNN._golden(name)
    rec = _SeqRecorder(_lib.lib)
    ABI._patch(monkeypatch)
    monkeypatch.setattr(ops, 'lib', rec)
    agent = _make(monkeypatch, tmp_path, g, over)
    rec.seq.clear()
    agent.epoch_num += 1
    agent.train_epoch()
    return agent, rec.seq


def _count(seq, name):
    return sum(1 for s in seq if s == name)


@pytest.mark.parametrize('name', GOLDENS)
def test_mixed_precision_true_runs_every_conv_and_linear_layer_on_the_tensor_cores(name, monkeypatch, tmp_path):
    agent, seq = _abi_sequence(monkeypatch, tmp_path, name, {'mixed_precision': True})
    g, m = CNN._golden(name), agent.model
    assert agent.mixed_precision and agent.wbf is not None and agent.wbf.dtype == torch.bfloat16 and agent.wbf.numel() == m.num_params
    for op in CONV_LINEAR:
        assert _count(seq, f'b200rl_{op}_f32') == 0, op
    H, trunks, n_conv = g['H'], 2 if g['separate'] else 1, len(g['network']['cnn']['convs'])
    n_upd = g['config']['mini_epochs'] * (g['N'] * H // g['mb'])
    n_lin = len(g['units']) + 1          # hidden layers + the head layer of each trunk
    assert _count(seq, 'b200rl_conv2d_fwd_tc') == trunks * n_conv * (H + 1 + n_upd)
    assert _count(seq, 'b200rl_conv2d_bwd_weight_tc') == trunks * n_conv * n_upd
    assert _count(seq, 'b200rl_conv2d_bwd_data_tc') == trunks * (n_conv - 1) * n_upd
    assert _count(seq, 'b200rl_linear_fwd_tc') == trunks * n_lin * (H + 1 + n_upd)
    assert _count(seq, 'b200rl_linear_bwd_weight_tc') == trunks * n_lin * n_upd
    assert _count(seq, 'b200rl_linear_bwd_data_tc') == trunks * n_lin * n_upd        # the first layer's lands in the conv gradient
    # the twin follows every optimiser step
    adam = [i for i, s in enumerate(seq) if s.startswith('b200rl_adam_step')]
    assert len(adam) == n_upd
    for i in adam:
        assert seq[i + 1] == 'b200rl_cast_bf16', seq[i:i + 2]
    assert _count(seq, 'b200rl_cast_bf16') == n_upd


def _record_parent_sequences(monkeypatch, tmp_path):
    return {f'{name}|{key}': _abi_sequence(monkeypatch, tmp_path, name, over)[1]
            for name in GOLDENS for key, over in (('absent', {}), ('false', {'mixed_precision': False}))}


@pytest.mark.parametrize('name', GOLDENS)
@pytest.mark.parametrize('key,over', [('absent', {}), ('false', {'mixed_precision': False})])
def test_mixed_precision_false_or_absent_makes_the_fp32_agents_calls(name, key, over, monkeypatch, tmp_path):
    agent, seq = _abi_sequence(monkeypatch, tmp_path, name, over)
    assert not agent.mixed_precision and agent.wbf is None
    assert not any(s.endswith('_tc') or s == 'b200rl_cast_bf16' for s in seq)
    with open(SEQ_FILE) as f:
        assert seq == json.load(f)[f'{name}|{key}']


def _twin_ok(agent):
    return torch.equal(agent.wbf, agent.model.flat.to(torch.bfloat16))


@pytest.mark.parametrize('name', GOLDENS)
def test_the_twin_follows_every_update_weight_load_and_restore(name, monkeypatch, tmp_path):
    g = CNN._golden(name)
    a = _make(monkeypatch, tmp_path, g, {'mixed_precision': True}, install=_tc_stand_ins)
    assert _twin_ok(a)                                    # built with the agent
    flat0 = a.model.flat.clone()
    a.epoch_num += 1
    a.train_epoch(u=g['u'][0])
    assert not torch.equal(a.model.flat, flat0) and _twin_ok(a)       # after the last update
    # every update: the twin the next minibatch reads is the arena after the previous step
    seen = []
    orig = a._minibatch_update

    def spy(i):
        assert _twin_ok(a)
        seen.append(i)
        return orig(i)
    monkeypatch.setattr(a, '_minibatch_update', spy)
    a.epoch_num += 1
    a.train_epoch(u=g['u'][1])
    assert len(seen) == a.mini_epochs_num * a.num_minibatches and _twin_ok(a)
    ckpt = str(tmp_path / 'tc')
    a.save(ckpt)
    # set_weights: a different state
    sd = {k: v + 0.01 if k.startswith('a2c_network.') else v for k, v in a.model.state_dict().items()}
    a.set_weights({'model': sd})
    assert _twin_ok(a) and torch.equal(a.model.state_dict()['a2c_network.value.weight'], sd['a2c_network.value.weight'])
    # a checkpoint restore, into this agent and into a fresh one
    a.restore(ckpt + '.pth')
    assert _twin_ok(a) and not torch.equal(a.model.state_dict()['a2c_network.value.weight'], sd['a2c_network.value.weight'])
    b = _make(monkeypatch, tmp_path, g, {'mixed_precision': True}, install=_tc_stand_ins)
    b.restore(ckpt + '.pth')
    assert _twin_ok(b) and torch.equal(b.model.flat, a.model.flat)


@pytest.mark.parametrize('name', GOLDENS)
def test_checkpoints_are_compatible_both_ways_with_the_fp32_agent(name, monkeypatch, tmp_path):
    g = CNN._golden(name)
    for src_over, dst_over in (({'mixed_precision': True}, {}), ({}, {'mixed_precision': True})):
        src = _make(monkeypatch, tmp_path, g, src_over, install=_tc_stand_ins)
        src.epoch_num += 1
        src.train_epoch(u=g['u'][0])
        ckpt = str(tmp_path / 'ck')
        src.save(ckpt)
        state = torch.load(ckpt + '.pth', weights_only=False)
        dst = _make(monkeypatch, tmp_path, g, dst_over, install=_tc_stand_ins)
        dst.restore(ckpt + '.pth')
        back = dst.get_full_state_weights()
        assert list(back['model']) == list(state['model'])
        for k, v in state['model'].items():
            assert back['model'][k].dtype == v.dtype and torch.equal(back['model'][k], v), k
        assert back['optimizer']['state'].keys() == state['optimizer']['state'].keys()
        for i, st in state['optimizer']['state'].items():
            for k, v in st.items():
                assert torch.equal(torch.as_tensor(back['optimizer']['state'][i][k]), torch.as_tensor(v)), (i, k)
        assert (back['epoch'], back['frame']) == (state['epoch'], state['frame'])
        if dst.mixed_precision:
            assert _twin_ok(dst)


# the tensor-core run against the recorded fp32 reference: each bf16 operand is off by up to 2^-9 relative, through three convs and the
# MLP; every compared quantity stays within LOOSE of the reference's largest magnitude of that quantity (max-norm), the sampled actions
# are the reference's exactly on these tapes
LOOSE = {'rewards': 2e-2, 'values': 2e-2, 'advantages': 5e-2, 'old_logp_actions': 1e-2, 'a_losses': 5e-2, 'c_losses': 5e-2,
         'entropies': 1e-2, 'state': 2e-2}


def max_norm_err(got, ref):
    return (got.double() - ref.double()).abs().max().item() / (ref.double().abs().max().item() + 1e-12)


def check_against_fp32_golden(agent, g, res, ep, cpu=lambda t: t):
    ref = g['epochs_out'][ep]
    fl = lambda t: t.transpose(0, 1).reshape(-1, *t.shape[2:])    # noqa: E731
    assert torch.equal(cpu(agent.actions), ref['mb_actions'])
    got = {'rewards': (cpu(agent.rewards).unsqueeze(2), ref['mb_rewards']), 'values': (cpu(agent.values).unsqueeze(2), ref['mb_values']),
           'advantages': (cpu(fl(agent.advs_n)), ref['advantages']), 'old_logp_actions': (cpu(fl(agent.neglogpacs)), ref['old_logp_actions'])}
    for i, key in ((4, 'a_losses'), (5, 'c_losses'), (6, 'entropies')):
        got[key] = (cpu(torch.stack(res[i])), ref[key])
    for key, (a, r) in got.items():
        assert max_norm_err(a, r) <= LOOSE[key], (key, max_norm_err(a, r))
    sd = agent.model.state_dict()
    for k, v in ref['state'].items():
        assert max_norm_err(cpu(sd[k]).reshape(v.shape), v) <= LOOSE['state'], (k, max_norm_err(cpu(sd[k]).reshape(v.shape), v))


@pytest.mark.parametrize('name', GOLDENS)
def test_kernel_faithful_model_stays_near_the_fp32_reference_golden(name, monkeypatch, tmp_path):
    """the stand-ins that round like the kernels, over both recorded epochs: the bound the GPU run is held to as well"""
    g = CNN._golden(name)
    agent = _make(monkeypatch, tmp_path, g, {'mixed_precision': True}, install=_tc_stand_ins)
    for ep in range(len(g['epochs_out'])):
        agent.epoch_num += 1
        res = agent.train_epoch(u=g['u'][ep])
        check_against_fp32_golden(agent, g, res, ep)


@pytest.mark.skipif(RR.REF is None, reason='reference rl_games not present (oracle/_ref)')
def test_pong_yaml_with_mixed_precision_trains_through_the_reference_runner(monkeypatch, tmp_path):
    """configs/atari/ppo_pong.yaml unchanged but for mixed_precision: True and what a launcher injects (uint8 frames at 36 x 36, one
    epoch): every conv and linear call on the tensor-core entry points, every call header-checked"""
    import yaml
    CNN._ref_path()
    from rl_games.torch_runner import Runner
    import rl_games_b200
    from rl_games_b200 import agent_discrete
    rec = ABI._patch(monkeypatch)
    monkeypatch.setattr(agent_discrete.DiscreteA2CAgent, '_require_cuda', lambda self: None)
    monkeypatch.setattr(agent_discrete.DiscreteA2CAgent, '_sync', staticmethod(lambda: None))
    cfg = yaml.safe_load(open(os.path.join(RR.REF, 'rl_games', 'configs', 'atari', 'ppo_pong.yaml')))
    c, net = cfg['params']['config'], cfg['params']['network']
    nhwc = net['cnn'].get('permute_input', True)
    shape = (CNN._FRAME, CNN._FRAME, 4) if nhwc else (4, CNN._FRAME, CNN._FRAME)
    env = CNN._ImageEnv(c['num_actors'], shape, 6)
    c.update({'env_info': env.get_env_info(), 'vec_env': env, 'device': 'cpu', 'max_epochs': 1, 'train_dir': str(tmp_path),
              'multi_gpu': False, 'mixed_precision': True})
    c.pop('max_frames', None)
    runner = Runner()
    rl_games_b200.register(runner)
    runner.load(cfg)
    runner.params['config']['vec_env'] = env
    made = []
    orig_create = runner.algo_factory.create
    monkeypatch.setattr(runner.algo_factory, 'create', lambda name, **kw: (made.append(orig_create(name, **kw)), made[-1])[1])
    runner.run({'train': True, 'play': False, 'checkpoint': None, 'sigma': None})
    agent, = made
    assert type(agent) is agent_discrete.DiscreteA2CAgent and agent.epoch_num == 1 and agent.mixed_precision
    n_conv = len(net['cnn']['convs'])
    n_upd = c['mini_epochs'] * (c['num_actors'] * c['horizon_length'] // c['minibatch_size'])
    trunks = 2 if net.get('separate') else 1
    assert rec.calls['b200rl_conv2d_fwd_tc'] == trunks * n_conv * (c['horizon_length'] + 1 + n_upd)
    assert rec.calls['b200rl_conv2d_bwd_weight_tc'] == trunks * n_conv * n_upd
    assert rec.calls['b200rl_conv2d_bwd_data_tc'] == trunks * (n_conv - 1) * n_upd
    assert rec.calls['b200rl_linear_fwd_tc'] > 0 and rec.calls['b200rl_linear_bwd_weight_tc'] > 0
    assert rec.calls['b200rl_cast_bf16'] == n_upd + 1
    for op in CONV_LINEAR:
        assert rec.calls.get(f'b200rl_{op}_f32', 0) == 0, op


if __name__ == '__main__':           # records the fp32 agent's call sequences (run at the commit whose sequence is to be kept)
    import tempfile
    mp = pytest.MonkeyPatch()
    with tempfile.TemporaryDirectory() as d:
        seqs = _record_parent_sequences(mp, __import__('pathlib').Path(d))
    mp.undo()
    with open(SEQ_FILE, 'w') as f:
        json.dump(seqs, f, separators=(',', ':'))
    print({k: len(v) for k, v in seqs.items()})
