"""The census of layer GEMM and convolution calls (tests/golden/layer_census.json, written by tests/golden/gen_layer_census.py) is the
list of calls tests/test_layer_census_gpu.py replays against fp64 on the GPU.  Here, without a GPU:
- the agents still make exactly the recorded calls: a change that issues a new geometry, argument or buffer layout fails until the
  fixture is regenerated, which brings the new call under the GPU replay;
- every entry obeys the argument rules of include/b200rl.h, so a hand-edited fixture cannot replay calls no agent could make;
- the calls the replay exists for are in it."""
import json
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'golden'))
import gen_layer_census as G  # noqa: E402

with open(G.OUT) as _f:
    FIXTURE = json.load(_f)
ENTRIES = FIXTURE['golden'] + FIXTURE['yaml']


def _strip(entries):
    return [json.loads(json.dumps(e)) for e in entries]


def test_golden_configurations_make_the_recorded_calls():
    assert _strip(G.golden_part()) == FIXTURE['golden']


@pytest.mark.skipif(not G.have_reference(), reason='reference rl_games not present (oracle/_ref)')
def test_shipped_yamls_make_the_recorded_calls():
    assert _strip(G.yaml_part()) == FIXTURE['yaml']


def test_the_fixture_is_written_as_the_generator_writes_it():
    with open(G.OUT) as f:
        assert f.read() == G.dumps(FIXTURE)


def _rows_per_split(fn, P, S):
    """the weight-gradient kernels' split rule: ceil(P / S) rows, rounded up to the reduction slab"""
    slab = 64 if fn.endswith('_tc') else 16
    rps = -(-P // S)
    return -(-rps // slab) * slab


def _header_rules(e):
    """include/b200rl.h's argument rules for one entry (the kernels return B200RL_EINVAL otherwise) and the layout facts the replay
    relies on"""
    fn, a, p = e['fn'], e['args'], e['ptr']
    assert fn in {n[len('b200rl_'):] for n in G.FNS}
    assert e['configs'] and all(isinstance(c, str) for c in e['configs'])
    if fn == 'reduce_splits_f32':
        assert a['n'] > 0 and a['n_splits'] > 0 and a['split_stride'] >= a['n']
        return
    assert a['M'] > 0
    if fn.startswith('linear'):
        assert a['K'] > 0 and a['Nout'] > 0
        n_w, n_b, D = a['Nout'] * a['K'], a['Nout'], a['K']
    else:
        for k in ('C', 'H', 'Wd', 'Cout', 'KH', 'KW', 'stride'):
            assert a[k] > 0, k
        assert a['pad'] >= 0 and a['H'] + 2 * a['pad'] >= a['KH'] and a['Wd'] + 2 * a['pad'] >= a['KW']
        n_w, n_b, D = a['Cout'] * a['C'] * a['KH'] * a['KW'], a['Cout'], a['C'] * a['H'] * a['Wd']
        if fn.endswith('_tc') and 'bwd_weight' not in fn:
            assert p.get('W_bf16') is True and 'wb_mod8' in p, 'the tensor-core convolutions read the bf16 twin only'
    if 'W_bf16' in p and p['W_bf16']:
        assert fn.endswith('_tc') and p['wb_mod8'] == p.get('w_mod8', p['wb_mod8']), 'the twin has the arena offsets'
    if 'rows_per_chunk' in a:                                   # the first-layer readers: chunked arena rows
        assert a['rows_per_chunk'] > 0 and a['x_ld'] >= D and 0 <= p['x_align16'] < 16
        if a['rows_per_chunk'] < a['M']:
            assert a['chunk_stride'] >= a['rows_per_chunk']
    if 'act' in a:
        assert a['act'] in (0, 1, 2, 3)
    if 'act_prev' in a:
        assert a['act_prev'] in (0, 1, 2, 3)
    if 'bwd_weight' in fn:
        S, ss = a['n_splits'], a['split_stride']
        assert 1 <= S <= 65535
        assert 0 <= p['dw_off'] and p['dw_off'] + n_w <= ss, 'dW inside one split row'
        if p['db']:
            db = p['dw_off'] + p['db_rel']
            assert 0 <= db and db + n_b <= ss and (db + n_b <= p['dw_off'] or db >= p['dw_off'] + n_w), 'db inside the row, apart from dW'


@pytest.mark.parametrize('part', ['golden', 'yaml'])
def test_every_entry_obeys_the_header_rules(part):
    if part == 'yaml' and not FIXTURE['yaml']:
        pytest.skip('no yaml part')
    for e in FIXTURE[part]:
        try:
            _header_rules(e)
        except AssertionError as ex:
            raise AssertionError(f'{e}: {ex}') from None


def test_the_census_holds_the_calls_the_replay_exists_for():
    def have(pred, entries=ENTRIES):
        return any(pred(e['fn'], e['args'], e['ptr']) for e in entries)
    # SAC's critic reads [obs | action] rows (K = D + A); its actor reads the obs columns of the same rows: K = D, row stride D + A
    sac = [e for e in ENTRIES if any(c.startswith('sac') or '/sac_' in c for c in e['configs'])]
    assert have(lambda f, a, p: f.startswith('linear_fwd') and a['x_ld'] > a['K'], sac)
    assert have(lambda f, a, p: f.startswith('linear_bwd_weight') and a['x_ld'] > a['K'], sac)
    # a value head
    assert have(lambda f, a, p: f.startswith('linear') and a['Nout'] == 1)
    # SAC on the tensor cores: no twin, its fp32 weights are rounded as they are staged
    assert have(lambda f, a, p: f == 'linear_fwd_tc' and not p['W_bf16'])
    assert have(lambda f, a, p: f == 'linear_bwd_data_tc' and not p['W_bf16'])
    # a weight gradient whose trailing splits are empty
    def pixels(f, a):
        if f.startswith('linear'):
            return a['M']
        return a['M'] * ((a['H'] + 2 * a['pad'] - a['KH']) // a['stride'] + 1) * ((a['Wd'] + 2 * a['pad'] - a['KW']) // a['stride'] + 1)
    assert have(lambda f, a, p: 'bwd_weight' in f and _rows_per_split(f, pixels(f, a), a['n_splits']) * (a['n_splits'] - 1) >= pixels(f, a))
    if G.have_reference():
        # the Nature CNN's flatten at minibatch 2048, fp32 and tensor cores, and a [512, 256, 128] MLP
        for f in ('linear_fwd_f32', 'linear_fwd_tc', 'linear_bwd_weight_f32', 'linear_bwd_weight_tc'):
            assert have(lambda fn, a, p: fn == f and a['K'] == 3136 and a['Nout'] == 512 and a['M'] == 2048), f
        assert have(lambda f, a, p: f == 'linear_fwd_tc' and a['K'] == 512 and a['Nout'] == 256)

