"""Discrete action spaces wider than the narrow categorical kernels (more than 8 heads, or a head of more than 64 actions) on CPU, without
the CUDA kernels:
- the oracle against the reference's golden runs on Discrete(362) with masks and on a Tuple of 10 heads with per-head masks
  (tests/golden/gen_golden_cat_wide.py);
- the agent's host logic on torch stand-ins against the same runs;
- one epoch per precision with every C-ABI call header-checked: the wide entry points, never the narrow ones;
- the choice of kernels from the layout, the refusals, the memory check before allocation;
- the model's state-dict keys and index-keyed Adam order at the microrts layout (1792 heads);
- the wide sampler's Philox counters against their host reference (tests/_cat_wide_ref.py)."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import test_abi_calls_cpu as ABI  # noqa: E402
import test_discrete_host_cpu as DH  # noqa: E402
import test_oracle_vs_golden as TOV  # noqa: E402

GOLDEN = os.path.join(HERE, 'golden')
WIDE_GOLDENS = ['agent_discrete_wide362.pt', 'agent_multidiscrete_wide.pt']
MICRORTS_HEADS = [6, 4, 4, 4, 4, 7, 49] * 256          # gym-microrts unit commands on a 16 x 16 map: 1792 heads, 19968 logits


def _golden(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


@pytest.mark.parametrize('name', WIDE_GOLDENS)
def test_oracle_matches_the_reference_on_wide_spaces(name):
    TOV.test_discrete_train_epochs_match_reference_agent(name)


@pytest.mark.parametrize('name', WIDE_GOLDENS)
def test_agent_host_logic_matches_the_reference_on_wide_spaces(name, monkeypatch, tmp_path):
    DH.test_discrete_agent_host_logic_matches_reference_golden(name, False, monkeypatch, tmp_path)


@pytest.mark.parametrize('mixed_precision', [False, True])
@pytest.mark.parametrize('name', WIDE_GOLDENS)
def test_one_epoch_makes_header_checked_wide_calls(name, mixed_precision, monkeypatch, tmp_path):
    g = _golden(name)
    rec = ABI._patch(monkeypatch)
    agent = DH._build(monkeypatch, tmp_path, g, stand_ins=False, over={'mixed_precision': mixed_precision})
    agent.epoch_num += 1
    agent.train_epoch(u=g['u'][0])
    n_upd = g['config']['mini_epochs'] * (g['N'] * g['H'] // g['mb'])
    assert rec.calls['b200rl_categorical_sample_wide_f32'] == g['H']
    assert rec.calls['b200rl_categorical_sample_f32'] == 1                  # the values-only bootstrap forward serves every layout
    assert rec.calls['b200rl_categorical_loss_wide_f32'] == n_upd
    assert rec.calls.get('b200rl_categorical_loss_f32', 0) == 0
    lin = 'tc' if mixed_precision else 'f32'
    assert rec.calls[f'b200rl_linear_fwd_{lin}'] > 0
    assert rec.calls.get('b200rl_linear_fwd_' + ('f32' if mixed_precision else 'tc'), 0) == 0
    assert agent.loss_partials.shape == (g['mb'], 8)                         # one partial row per minibatch row


def test_kernel_choice_follows_the_layout():
    from rl_games_b200 import ops
    assert not ops.categorical_is_wide(64) and ops.categorical_is_wide(65) and ops.categorical_is_wide(362)
    assert not ops.categorical_is_wide(8 * 64, [64] * 8)
    assert ops.categorical_is_wide(9 * 2, [2] * 9) and ops.categorical_is_wide(65 + 3, [3, 65])
    assert ops.categorical_is_wide(sum(MICRORTS_HEADS), MICRORTS_HEADS)
    assert ops.categorical_loss_partial_rows(1000, 64) == 4 and ops.categorical_loss_partial_rows(1000, 362) == 1000


def _spaces(action_space, units=(64, 32)):
    from rl_games_b200.agent_discrete import discrete_spaces
    from rl_games_b200.common import Box
    return discrete_spaces(Box(-np.inf, np.inf, (8,)), action_space, {'mlp': {'units': list(units)}}, {})


def test_wide_layouts_are_accepted_and_unrunnable_ones_refused():
    from rl_games_b200.agent_discrete import HEAD_MAX_OUTPUTS
    from rl_games_b200.common import Discrete, Tuple
    assert _spaces(Discrete(4672))[2:5] == (None, 4672, False)
    sizes, K, multi = _spaces(Tuple([Discrete(k) for k in MICRORTS_HEADS]))[2:5]
    assert sizes == MICRORTS_HEADS and K == 19968 and multi
    with pytest.raises(ValueError, match='head of 0 actions'):
        _spaces(Tuple([Discrete(3), Discrete(0)]))
    with pytest.raises(ValueError, match='head of 0 actions'):
        _spaces(Discrete(0))
    with pytest.raises(NotImplementedError, match=f'at most {HEAD_MAX_OUTPUTS} outputs'):
        _spaces(Discrete(HEAD_MAX_OUTPUTS))
    _spaces(Discrete(HEAD_MAX_OUTPUTS - 1), units=(16,))
    with pytest.raises(NotImplementedError, match='32-bit parameter index'):
        _spaces(Discrete(2 ** 21), units=(1024,))


def test_microrts_model_keys_and_optimizer_order():
    """DiscreteModel at 1792 heads: logits.{j} keys in ModuleList order, head j's rows of the fused head, and the index-keyed Adam state
    in the reference's model.parameters() order"""
    from rl_games_b200.agent_discrete import DiscreteModel
    K = sum(MICRORTS_HEADS)
    m = DiscreteModel({'mlp': {'units': [32, 16], 'activation': 'relu'}}, 8, K, 'cpu', False, False, head_sizes=MICRORTS_HEADS)
    names = m.param_names()
    nh = len(MICRORTS_HEADS)
    assert names[-2 * nh:] == [f'a2c_network.logits.{j}.{w}' for j in range(nh) for w in ('weight', 'bias')]
    assert names[:6] == ['a2c_network.actor_mlp.0.weight', 'a2c_network.actor_mlp.0.bias', 'a2c_network.actor_mlp.2.weight',
                         'a2c_network.actor_mlp.2.bias', 'a2c_network.value.weight', 'a2c_network.value.bias']
    m.flat.copy_(torch.arange(m.num_params, dtype=torch.float32))
    sd = m.state_dict()
    wh = m.view('W_head')
    off = 1
    for j, k in enumerate(MICRORTS_HEADS):
        assert sd[f'a2c_network.logits.{j}.weight'].shape == (k, 16)
        assert torch.equal(sd[f'a2c_network.logits.{j}.weight'], wh[off:off + k])
        off += k
    assert off == 1 + K
    st = m.optimizer_state_dict(1e-3, 1.0, 0.0)
    assert sorted(st['state']) == list(range(len(names)))
    assert st['state'][len(names) - 1]['exp_avg'].shape == (MICRORTS_HEADS[-1],)
    m2 = DiscreteModel({'mlp': {'units': [32, 16], 'activation': 'relu'}}, 8, K, 'cpu', False, False, head_sizes=MICRORTS_HEADS)
    m2.load_state_dict(sd, strict=False)
    assert torch.equal(m2.flat, m.flat)


def test_wide_policy_refused_before_allocation_when_the_device_is_short(monkeypatch, tmp_path):
    """a wide-head agent on a device whose free memory is below init_tensors_bytes plus the epoch's transient allowance: RuntimeError
    naming the bytes, nothing allocated"""
    from rl_games_b200 import agent_discrete
    g = _golden('agent_multidiscrete_wide.pt')
    agent = DH._build(monkeypatch, tmp_path, g)
    need = agent.init_tensors_bytes() + agent.TRANSIENT_BYTES
    # the wide layout's buffers are in the count: [H, N, K] masks, [H, N, heads] actions, one loss partial row per minibatch row
    H, N, K, mb = g['H'], g['N'], sum(g['K']), g['mb']
    assert agent.init_tensors_bytes() > H * N * (K + 8 * len(g['K'])) + 8 * 8 * mb
    agent._tensors_ready = False
    for name in ('obses', 'part', 'r_a', 't_a', 'd_a', 'grad', 'loss_partials'):
        delattr(agent, name)
    agent.device_t = torch.device('cuda', 0)           # the check only runs on a CUDA device; the device is never touched
    monkeypatch.setattr(torch.cuda, 'mem_get_info', lambda dev=None: (need - 1, 80 * 2 ** 30))
    allocs = []
    monkeypatch.setattr(agent_discrete.torch, 'zeros', lambda *a, **k: allocs.append(a))
    with pytest.raises(RuntimeError, match=f'this wide-head policy needs {need} bytes of device memory'):
        agent.init_tensors()
    assert allocs == [] and not hasattr(agent, 'obses')
    monkeypatch.setattr(torch.cuda, 'mem_get_info', lambda dev=None: (need, 80 * 2 ** 30))
    agent._check_memory()


def test_wide_philox_layout_extends_the_narrow_one_without_collisions():
    import _cat_wide_ref as W
    import _philox_ref as P
    seed, rows = 0x1234ABCD, 257
    for epoch, step in ((0, 0), (3, 17)):
        np.testing.assert_array_equal(W.categorical_uniforms_wide(seed, rows, 8, epoch, step)[:8],
                                      P.categorical_uniforms(seed, rows, 8, epoch, step))
    # counters of heads 0..99 at a few steps, and the Gaussian sampler's (q < 8): all distinct
    r = np.arange(rows, dtype=np.uint64)
    seen = set()
    n = 0
    for step in (0, 1, 5):
        for j in range(100):
            lo, hi = W.wide_counters(r, j, 2, step)
            seen.update(zip(lo.tolist(), [hi] * rows))
            n += rows
        for q in range(P.GAUSS_Q_MAX):
            seen.update(zip(r.tolist(), [P.policy_counter(2, step, q)] * rows))
            n += rows
    assert len(seen) == n
    u = W.categorical_uniforms_wide(seed, rows, 100, 2, 5)
    assert ((u >= 0) & (u < 1)).all() and len(np.unique(u)) > 0.99 * u.size


def test_wide_cdf_order_matches_a_sequential_sum_closely_and_picks_legal_actions():
    import _cat_wide_ref as W
    rng = np.random.default_rng(0)
    z = rng.normal(size=(64, 362)).astype(np.float32) * 2
    mask = rng.random((64, 362)) < 0.3
    z = np.where(mask, z, -1e8).astype(np.float32)
    p = np.exp(z - z.max(1, keepdims=True))
    p = (p / p.sum(1, keepdims=True)).astype(np.float32)
    np.testing.assert_allclose(W.wide_cdf(p), np.cumsum(p.astype(np.float64), 1), atol=1e-5)
    a, _ = W.wide_inverse_cdf(p, rng.random(64).astype(np.float32))
    assert (p[np.arange(64), a] > 0).all()
