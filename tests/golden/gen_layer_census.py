"""Records the census of layer GEMM and convolution calls the agents make: tests/golden/layer_census.json.

Each agent family runs one train_epoch (rollout + update) with the C ABI replaced by the header-checking recorder of
tests/test_abi_calls_cpu.py (no GPU, nothing computed).  For every call of the linear / conv2d entry points and of reduce_splits, the
census keeps the scalar arguments verbatim and the pointer facts the layout depends on, taken relative to the buffer each pointer points
into (never a raw address):
- which optional pointers are set (normaliser, bias, A_prev, db, W_bf16);
- the element offset of W / W_bf16 in its arena, mod 8, and the byte offset of X, mod 16;
- for a weight gradient: the element offset of dW in its split row and the offset of db from dW.
Identical calls are merged; each entry lists the configurations that made it.  Two parts: ``golden`` (the configurations of the
golden replays, always reproducible) and ``yaml`` (every shipped reference YAML that trains in the Runner sweeps, needs oracle/_ref).

tests/test_layer_census_cpu.py checks that the agents still make exactly these calls; tests/test_layer_census_gpu.py replays each
entry on the H100 against fp64.  Regenerate with ``python tests/golden/gen_layer_census.py`` after a change that alters the calls."""
import ctypes
import json
import os
import sys
import tempfile

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
ROOT = os.path.dirname(TESTS)
sys.path.insert(0, TESTS)
sys.path.insert(0, ROOT)
import test_abi_calls_cpu as ABI  # noqa: E402

OUT = os.path.join(HERE, 'layer_census.json')
FNS = tuple(f'b200rl_{op}_{p}' for op in ('linear_fwd', 'linear_bwd_data', 'linear_bwd_weight', 'conv2d_fwd', 'conv2d_bwd_data',
                                          'conv2d_bwd_weight') for p in ('f32', 'tc')) + ('b200rl_reduce_splits_f32',)
# optional pointer arguments -> the census flag that says whether the call passed one
OPTIONAL = {'norm_mean': 'norm', 'b': 'bias', 'A_prev': 'A_prev', 'db_part': 'db', 'W_bf16': 'W_bf16'}


class CensusRecorder(ABI._Recorder):
    """the header-checking recorder, keeping the scalar arguments and the relative pointer facts of the census entry points"""

    def __init__(self, real):
        super().__init__(real)
        self.entries = []
        self.bufs = {}           # address -> (buffer base address, element size): what ptr() / the bf16 twin lookup saw in this call

    def note(self, t):
        if isinstance(t, torch.Tensor):
            base = t.untyped_storage().data_ptr()
            self.bufs[t.data_ptr()] = (base, t.element_size())

    def _rel(self, p):
        base, es = self.bufs[p]
        return (p - base) // es, (p - base)

    def __getattr__(self, name):
        call = super().__getattr__(name)
        if name not in FNS:
            return call
        sig = self.real.protos[name]

        def rec(*args):
            rc = call(*args)
            e = {'fn': name[len('b200rl_'):], 'args': {}, 'ptr': {}}
            for a, (an, t) in zip(args, sig):
                if an == 'stream':
                    continue
                if t is ctypes.c_void_p:
                    if an in OPTIONAL:
                        e['ptr'][OPTIONAL[an]] = a is not None and a != 0
                else:
                    e['args'][an] = a
            v = dict(zip((an for an, _ in sig), args))
            if 'W' in v and v['W']:
                e['ptr']['w_mod8'] = self._rel(v['W'])[0] % 8
            if v.get('W_bf16'):
                e['ptr']['wb_mod8'] = self._rel(v['W_bf16'])[0] % 8
            if 'X' in v:
                e['ptr']['x_align16'] = self._rel(v['X'])[1] % 16
            if 'dW_part' in v:
                w_off = self._rel(v['dW_part'])[0]
                e['ptr']['dw_off'] = w_off % v['split_stride'] if v['split_stride'] > 0 else w_off
                if v.get('db_part'):
                    e['ptr']['db_rel'] = self._rel(v['db_part'])[0] - w_off
            self.entries.append(e)
            self.bufs = {}
            return rc
        return rec


class _KeepOps:
    """a monkeypatch for the CPU builders that install torch stand-ins: everything but the stand-ins on `ops` is applied, so the real
    wrappers (and the recorder behind them) are what runs"""

    def __init__(self, mp):
        self.mp = mp

    def setattr(self, target, name, value=None, raising=True):
        from rl_games_b200 import ops
        if target is not ops:
            self.mp.setattr(target, name, value, raising=raising)

    def __getattr__(self, name):
        return getattr(self.mp, name)


def _install(mp):
    """the recorder behind ops.lib; ops.ptr / ops._bf16_view_ptr note which buffer each pointer of the current call points into"""
    from rl_games_b200 import ops, _lib
    ABI._patch(mp)
    rec = CensusRecorder(_lib.lib)
    mp.setattr(ops, 'lib', rec)
    real_ptr, real_view = ops.ptr, ops._bf16_view_ptr

    def ptr(t):
        rec.note(t)
        return real_ptr(t)

    def view(W, bf16_arena):
        p = real_view(W, bf16_arena)
        if p is not None:
            fb = bf16_arena[1]
            rec.bufs[p] = (fb.untyped_storage().data_ptr(), 2)
        return p
    mp.setattr(ops, 'ptr', ptr)
    mp.setattr(ops, '_bf16_view_ptr', view)
    return rec


def _epoch(agent, **kw):
    agent.epoch_num += 1
    agent.train_epoch(**kw)


# --------------------------------------------------------------------------------------------------- the golden configurations
def _continuous(case):
    def run(mp, tmp):
        _epoch(ABI._agent(tmp, **ABI.CASES[case]))
    return run


def _discrete(name):
    def run(mp, tmp):
        import test_discrete_host_cpu as HD
        g = torch.load(os.path.join(HERE, name), weights_only=False)
        _epoch(HD._build(mp, tmp, g, stand_ins=False))
    return run


def _cnn(name, mixed):
    def run(mp, tmp):
        import test_cnn_cpu as CNN
        import test_conv_tc_cpu as CT
        _epoch(CT._make(mp, tmp, CNN._golden(name), {'mixed_precision': mixed}))
    return run


def _central_value(mp, tmp):
    import test_agent_cv_host_cpu as HC
    g = torch.load(os.path.join(HERE, 'agent_cv.pt'), weights_only=False)
    _epoch(HC._build_cv(_KeepOps(mp), tmp, g))


def _lstm_ln(name, mixed):
    def run(mp, tmp):
        import test_lstm_ln_cpu as LN
        g = torch.load(os.path.join(HERE, name), weights_only=False)
        _epoch(LN._host_agent(g, _KeepOps(mp), tmp, mixed), noise=g['noise'][0])
    return run


def _multi_agent(mp, tmp):
    import test_multiagent_cpu as MA
    g = torch.load(os.path.join(HERE, 'agent_ma.pt'), weights_only=False)
    agent, _ = MA._build(_KeepOps(mp), tmp, g)
    agent.init_tensors()
    agent.obs = agent.env_reset()
    _epoch(agent)


def _sac(fixture):
    def run(mp, tmp):
        import _sac_golden as SG
        import test_agent_host_cpu as H
        g = SG.load(fixture)
        SG.run(SG.make_agent(g, H._CudaLookingStr('cpu'), tmp), g)      # every recorded epoch: the first ones only fill the replay buffer
    return run


GOLDEN_CONFIGS = {
    'ppo fp32': _continuous('fp32'),
    'ppo fp32 masked': _continuous('fp32 masked, rms advantage, standard schedule'),
    'ppo [512,256,128] tc': _continuous('mlp [512,256,128] on the tensor cores (layer-wise GEMMs)'),
    'ppo lstm before the mlp': _continuous('lstm before the mlp'),
    'ppo lstm after the mlp': _continuous('lstm after the mlp'),
    'ppo lstm after the mlp tc': _continuous('lstm after the mlp on the tensor cores (layer-wise GEMMs)'),
    'ppo lstm+ln': _lstm_ln('agent_lstm_ln.pt', False),
    'ppo lstm+ln tc': _lstm_ln('agent_lstm_ln.pt', True),
    'ppo lstm+ln after the mlp tc': _lstm_ln('agent_lstm_ln_after.pt', True),
    'discrete': _discrete('agent_discrete.pt'),
    'discrete masked': _discrete('agent_discrete_masked.pt'),
    'multi-discrete': _discrete('agent_multidiscrete.pt'),
    'cnn shared fp32': _cnn('agent_cnn_shared.pt', False),
    'cnn shared tc': _cnn('agent_cnn_shared.pt', True),
    'cnn separate fp32': _cnn('agent_cnn_separate.pt', False),
    'cnn separate tc': _cnn('agent_cnn_separate.pt', True),
    'central value': _central_value,
    'multi-agent': _multi_agent,
    'sac box norm': _sac('sac_box_norm_same_step'),
    'sac fixed alpha': _sac('sac_fixed_alpha_next_step'),
}


# --------------------------------------------------------------------------------------------------- the shipped YAMLs
def _yaml_configs():
    """every shipped YAML the Runner sweeps train (the refused ones make no kernel call), run the way those sweeps run them"""
    import test_cnn_cpu as CNN
    import test_conv_tc_cpu as CT
    import test_reference_runner_cpu as RR
    import test_sac_cpu as SAC
    out = {}
    for rel in RR._shipped_ppo_yamls():
        if rel not in RR._REFUSED:
            out[f'yaml {rel}'] = (RR.test_every_shipped_ppo_yaml_of_the_in_scope_families_runs_through_the_reference_runner, rel)
    for rel in CNN._image_yamls():
        out[f'yaml {rel}'] = (CNN.test_every_atari_and_minigrid_yaml_trains_or_gives_its_reason, rel)
    out['yaml atari/ppo_pong.yaml mixed_precision'] = (lambda rel, monkeypatch, tmp_path:
                                                       CT.test_pong_yaml_with_mixed_precision_trains_through_the_reference_runner(monkeypatch, tmp_path), None)
    for rel in SAC._shipped_sac_yamls():
        if rel not in SAC._SAC_REFUSED:
            out[f'yaml {rel}'] = (SAC.test_every_shipped_sac_yaml_runs_through_the_reference_runner, rel)
    return out


def _run_yaml(entry):
    fn, rel = entry

    def run(mp, tmp):
        import test_cnn_cpu as CNN
        mp.setattr(CNN, '_FRAME', 84)           # the image YAMLs at the frame size of their envs: the Nature CNN's 3136 -> 512 flatten
        fn(rel=rel, monkeypatch=mp, tmp_path=tmp)
    return run


def _record(run):
    """the census calls one configuration makes"""
    import pathlib
    from rl_games_b200 import ops
    mp = pytest.MonkeyPatch()
    try:
        rec = _install(mp)
        # the Runner sweeps patch ABI._patch's recorder in themselves: keep ours behind ops.lib
        mp.setattr(ABI, '_patch', lambda m: (_patch_keep(m, rec), rec)[1])
        with tempfile.TemporaryDirectory() as d:
            torch.manual_seed(0)
            run(mp, pathlib.Path(d))
        assert ops.lib is rec
        return rec.entries
    finally:
        mp.undo()


def _patch_keep(m, rec):
    from rl_games_b200 import ops
    m.setattr(torch.cuda, 'set_device', lambda d: None)
    m.setattr(torch.cuda, 'Event', ABI.H._Event)
    m.setattr(torch.cuda, 'current_stream', lambda *a: ABI.H._Stream())
    m.setattr(torch.Tensor, 'pin_memory', lambda self: self)
    m.setattr(ops, 'lib', rec)


def _key(e):
    return json.dumps({k: e[k] for k in ('fn', 'args', 'ptr')}, sort_keys=True)


def census(configs):
    """{entry key: entry} over the configurations, each entry tagged with the configurations that made it"""
    merged = {}
    for name, run in configs.items():
        for e in _record(run):
            k = _key(e)
            merged.setdefault(k, dict(e, configs=[]))
            if name not in merged[k]['configs']:
                merged[k]['configs'].append(name)
    return [merged[k] for k in sorted(merged)]


def golden_part():
    return census(GOLDEN_CONFIGS)


def yaml_part():
    return census({k: _run_yaml(v) for k, v in _yaml_configs().items()})


def have_reference():
    return os.path.isdir(os.path.join(ROOT, 'oracle', '_ref', 'rl_games'))


def dumps(c):
    """one entry per line: diffs of the fixture read as the calls that changed"""
    parts = []
    for part in ('golden', 'yaml'):
        lines = ',\n'.join('  ' + json.dumps(e, sort_keys=True) for e in c[part])
        parts.append(f' "{part}": [\n{lines}\n ]')
    return '{\n' + ',\n'.join(parts) + '\n}\n'


if __name__ == '__main__':
    if not have_reference():
        sys.exit('oracle/_ref is missing: run __graft_entry__.build() first (the yaml part needs the reference)')
    c = {'golden': golden_part(), 'yaml': yaml_part()}
    with open(OUT, 'w') as f:
        f.write(dumps(c))
    print({part: len(v) for part, v in c.items()})
