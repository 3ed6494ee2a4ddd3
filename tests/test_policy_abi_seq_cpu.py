"""The ordered C-ABI launch sequence of the trainers and the players, pinned on the CPU: every call of one training epoch of each agent
family and of a few steps of each player goes through the header-checking recorder of tests/test_abi_calls_cpu.py, which keeps the
call's name, its scalar arguments verbatim and, for each pointer argument, only whether it is NULL.  tests/golden/policy_abi_seq.json
holds, per run, the number of calls, the count of each entry point and the SHA-256 of the whole sequence, so a change to how the
policies' forward code is shared between the trainers and the players cannot move, add, drop or re-argument a launch on any path -- the
fused wgmma rollout and the wide-observation rollout included, which no CPU stand-in computes.  Regenerate with
``python tests/test_policy_abi_seq_cpu.py`` at a commit whose sequences are to be kept."""
import collections
import ctypes
import hashlib
import json
import os
import sys
import tempfile

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, 'golden'))
import test_abi_calls_cpu as ABI  # noqa: E402
import test_players_cpu as TP  # noqa: E402

SEQ_FILE = os.path.join(HERE, 'golden', 'policy_abi_seq.json')


class _ArgRecorder(ABI._Recorder):
    """the header-checking recorder, keeping every call in order: [name, scalar arguments, pointer arguments as 1 (set) / None (NULL)]"""

    def __init__(self, real):
        super().__init__(real)
        self.seq = []

    def __getattr__(self, name):
        call = super().__getattr__(name)
        if name in ABI.HOST_ONLY:
            return call
        sig = self.real.protos[name]

        def rec(*args):
            rc = call(*args)
            row = [name[len('b200rl_'):]]
            for a, (_, t) in zip(args, sig):
                if t is ctypes.c_void_p:
                    row.append(None if a is None or (isinstance(a, int) and a == 0) else 1)
                else:
                    row.append(a.item() if hasattr(a, 'item') else a)
            self.seq.append(row)
            return rc
        return rec


def _epoch(agent, **kw):
    agent.epoch_num += 1
    agent.train_epoch(**kw)


# --------------------------------------------------------------------------------------------------- trainers
def _continuous(case, fixed_sigma=True):
    def run(mp, tmp):
        if not fixed_sigma:         # the same agent with a state-dependent sigma head
            from rl_games_b200.runner import Runner
            load = Runner.load

            def load_sd(self, conf):
                conf['params']['network']['space']['continuous']['fixed_sigma'] = False
                return load(self, conf)
            mp.setattr(Runner, 'load', load_sd)
        _epoch(ABI._agent(tmp, **ABI.CASES[case]))
    return run


def _central_value(mp, tmp):
    import test_agent_cv_host_cpu as HC
    from gen_layer_census import _KeepOps
    g = torch.load(os.path.join(HERE, 'golden', 'agent_cv.pt'), weights_only=False)
    _epoch(HC._build_cv(_KeepOps(mp), tmp, g))


def _discrete(name):
    def run(mp, tmp):
        import test_discrete_host_cpu as HD
        g = torch.load(os.path.join(HERE, 'golden', name), weights_only=False)
        _epoch(HD._build(mp, tmp, g, stand_ins=False))
    return run


def _cnn(name, mixed):
    def run(mp, tmp):
        import test_cnn_cpu as CNN
        import test_conv_tc_cpu as CT
        _epoch(CT._make(mp, tmp, CNN._golden(name), {'mixed_precision': mixed}))
    return run


def _sac(mp, tmp):
    import _sac_golden as SG
    import test_agent_host_cpu as H
    g = SG.load('sac_box_norm_same_step')
    SG.run(SG.make_agent(g, H._CudaLookingStr('cpu'), tmp), g)      # warm-up epochs, then epochs with updates


# --------------------------------------------------------------------------------------------------- players
def _player(cls_name, make, steps):
    """`steps` of (deterministic, rows the step finished or None) through the player that make(cls) builds"""
    def run(mp, tmp):
        from rl_games_b200 import players
        mp.setattr(players.BasePlayer, '_require_cuda', lambda self: None)
        p, env = make(getattr(players, cls_name))
        o = env.reset()
        p.get_batch_size(o, 1)
        p.init_rnn()
        for det, done in steps:
            if env.masks is not None:
                p.get_masked_action(o, env.masks, det)
            else:
                p.get_action(o, det)
            if done is not None:
                p._done_rows(torch.tensor(done, dtype=torch.uint8))
    return run


def _cont(net, over=None, D=4, tape=False):
    def make(cls):
        from rl_games_b200.common import Box
        env = TP._Env(3, D, Box(-np.ones(2), np.ones(2), (2,)))
        p = cls(TP._params('a2c_continuous', env, net, over))
        if tape:        # sampled actions from a noise tape instead of the Philox stream
            p._ensure_rows(3)
            p.noise = torch.zeros(3, 2)
        return p, env
    return make


def _disc(space='discrete', cnn=False, over=None):
    def make(cls):
        from rl_games_b200.common import Box, Discrete, Tuple
        act, K = (Tuple([Discrete(3), Discrete(4)]), 7) if space == 'multi_discrete' else (Discrete(5), 5)
        net = dict(TP.DISCRETE, space={space: None})
        obs_space = None
        if cnn:
            obs_space = Box(0, 255, (12, 12, 4), np.uint8)
            net['cnn'] = {'type': 'conv2d', 'activation': 'relu', 'initializer': {'name': 'default'},
                          'convs': [{'filters': 4, 'kernel_size': 3, 'strides': 2, 'padding': 0},
                                    {'filters': 8, 'kernel_size': 3, 'strides': 1, 'padding': 1}]}
        env = TP._Env(3, 4, act, obs_space=obs_space, masks=None if cnn else np.ones((3, K), np.uint8))
        params = TP._params('a2c_discrete', env, net, over)
        params['model']['name'] = 'multi_discrete_a2c' if space == 'multi_discrete' else 'discrete_a2c'
        return cls(params), env
    return make


def _sac_player(cls):
    from rl_games_b200.common import Box
    env = TP._Env(3, 4, Box(np.array([-2.0, 0.0]), np.array([2.0, 1.0]), (2,)))
    return cls(TP._params('sac', env, TP.SAC_NET, {'normalize_input': True})), env


def _net(units=(32, 16, 8), fixed_sigma=True, rnn=None):
    net = json.loads(json.dumps(TP.MLP))
    net['mlp']['units'] = list(units)
    net['space']['continuous']['fixed_sigma'] = fixed_sigma
    if rnn:
        net['rnn'] = rnn
    return net


def _lstm(before, ln=False):
    return _net((16, 8), rnn={'name': 'lstm', 'units': 8, 'layers': 1, 'before_mlp': before, 'layer_norm': ln})


_STEPS = [(True, None), (False, None), (True, None), (False, None)]
_LSTM_STEPS = [(True, [0, 1, 0]), (False, [1, 0, 1]), (True, None), (False, [0, 0, 1]), (True, None)]

RUNS = {f'ppo {case}': _continuous(case) for case in ABI.CASES}
RUNS.update({
    'ppo state-dependent sigma': _continuous('fp32', fixed_sigma=False),
    'ppo state-dependent sigma on the tensor cores': _continuous('mlp [512,256,128] on the tensor cores (layer-wise GEMMs)', fixed_sigma=False),
    'central value': _central_value,
    'discrete': _discrete('agent_discrete.pt'),
    'discrete masked': _discrete('agent_discrete_masked.pt'),
    'multi-discrete': _discrete('agent_multidiscrete.pt'),
    'cnn shared fp32': _cnn('agent_cnn_shared.pt', False),
    'cnn shared tc': _cnn('agent_cnn_shared.pt', True),
    'cnn separate fp32': _cnn('agent_cnn_separate.pt', False),
    'cnn separate tc': _cnn('agent_cnn_separate.pt', True),
    'sac': _sac,
    'player fp32': _player('PpoPlayerContinuous', _cont(_net((16, 8)), {'mixed_precision': False}), _STEPS),
    'player fp32 noise tape': _player('PpoPlayerContinuous', _cont(_net((16, 8)), {'mixed_precision': False}, tape=True), _STEPS),
    'player fused': _player('PpoPlayerContinuous', _cont(_net()), _STEPS),
    'player fused, rollout fp32': _player('PpoPlayerContinuous', _cont(_net(), {'b200_rollout_fp32': True}), _STEPS),
    'player fused, wide observations': _player('PpoPlayerContinuous', _cont(_net(), {'mixed_precision': True}, D=128), _STEPS),
    'player layer-wise tensor cores': _player('PpoPlayerContinuous', _cont(_net((512, 256, 128)), {'mixed_precision': True}), _STEPS),
    'player state-dependent sigma': _player('PpoPlayerContinuous', _cont(_net(fixed_sigma=False)), _STEPS),
    'player lstm before the mlp': _player('PpoPlayerContinuous', _cont(_lstm(True), {'mixed_precision': False}), _LSTM_STEPS),
    'player lstm after the mlp': _player('PpoPlayerContinuous', _cont(_lstm(False), {'mixed_precision': False}), _LSTM_STEPS),
    'player lstm+ln on the tensor cores': _player('PpoPlayerContinuous', _cont(_lstm(True, True), {'mixed_precision': True}), _LSTM_STEPS),
    'player discrete masked': _player('PpoPlayerDiscrete', _disc(), _STEPS),
    'player discrete masked on the tensor cores': _player('PpoPlayerDiscrete', _disc(over={'mixed_precision': True}), _STEPS),
    'player multi-discrete masked': _player('PpoPlayerDiscrete', _disc('multi_discrete'), _STEPS),
    'player cnn': _player('PpoPlayerDiscrete', _disc(cnn=True), _STEPS),
    'player cnn on the tensor cores': _player('PpoPlayerDiscrete', _disc(cnn=True, over={'mixed_precision': True}), _STEPS),
    'player sac': _player('SACPlayer', _sac_player, _STEPS),
})


def _record(run, mp, tmp):
    """the calls one run makes, in order"""
    from rl_games_b200 import ops, _lib
    rec = _ArgRecorder(_lib.lib)
    ABI._patch(mp)
    mp.setattr(ops, 'lib', rec)
    torch.manual_seed(0)
    run(mp, tmp)
    return rec.seq


def _summary(seq):
    """what the fixture keeps of a sequence: its length, the calls per entry point and the digest of the sequence itself"""
    text = json.dumps(seq, separators=(',', ':'))
    return {'calls': len(seq), 'launches': dict(sorted(collections.Counter(row[0] for row in seq).items())),
            'sha256': hashlib.sha256(text.encode()).hexdigest()}


def _fixture():
    with open(SEQ_FILE) as f:
        return json.load(f)


def test_the_fixture_holds_every_run():
    assert list(_fixture()) == list(RUNS)


@pytest.mark.parametrize('name', list(RUNS))
def test_launch_sequence_is_the_recorded_one(name, monkeypatch, tmp_path):
    got, want = _summary(_record(RUNS[name], monkeypatch, tmp_path)), _fixture()[name]
    assert got['launches'] == want['launches']          # which entry points were added or dropped
    assert got == want                                  # then the order and every scalar argument


if __name__ == '__main__':           # records the sequences (run at the commit whose sequences are to be kept)
    import pathlib
    out = {}
    for name, run in RUNS.items():
        mp = pytest.MonkeyPatch()
        try:
            with tempfile.TemporaryDirectory() as d:
                out[name] = _summary(_record(run, mp, pathlib.Path(d)))
        finally:
            mp.undo()
    with open(SEQ_FILE, 'w') as f:
        f.write('{\n' + ',\n'.join(f' {json.dumps(k)}: {json.dumps(v)}' for k, v in out.items()) + '\n}\n')
    print({k: v['calls'] for k, v in out.items()})
