"""The fused tensor-core forward kernels (mlp_fwd_tc_kernel<train | rollout>, narrow observations) at sizes where persistent CTAs run
more than one tile: the training forward at 140 tiles (70 CTAs x 2 tiles, last tile partial) and the rollout at N = 16384, in each of
the three activation units.  Against the fp32 CUDA-core kernels with the tolerances of tests/test_mlp_tc_gpu.py, and launch against
launch: the same inputs must give the same bytes (tiles, loss partials, rewritten old_mu / old_sigma, rollout outputs)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_mlp_tc_gpu import A, D, UNITS, cosine, decode_tiles, make_net, rel_l2  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = 'cuda'
ACTS = [1, 2, 3]       # elu, relu, tanh: one translation unit each


@pytest.mark.parametrize('act', ACTS)
def test_tc_fwd_train_two_tiles_per_cta(act):
    from rl_games_b200 import ops
    from rl_games_b200.ops import LossCfg
    g = torch.Generator().manual_seed(20 + act)
    W, b, Wh, bh, logstd = make_net(g)
    M = 140 * 128 - 37
    n_tiles = (M + 127) // 128
    obs = (torch.randn(M, D, generator=g) * 2 + 0.5).to(DEV)
    nm = (torch.randn(D, generator=g) * 0.3).to(DEV); ns = (torch.rand(D, generator=g) + 0.7).to(DEV)
    actions = torch.randn(M, A, generator=g).to(DEV)
    old_mu = (torch.randn(M, A, generator=g) * 0.5).to(DEV); old_sigma = (torch.rand(M, A, generator=g) + 0.5).to(DEV)
    old_v = torch.randn(M, generator=g).to(DEV); ret = torch.randn(M, generator=g).to(DEV)
    old_nlp = (torch.randn(M, generator=g) * 0.3 + 9.0).to(DEV); adv = torch.randn(M, generator=g).to(DEV)
    cfg = LossCfg(0.2, 2.0, 0.0, 1, 2, 1, 1, 1)
    ec = torch.tensor([0.0], device=DEV)
    stride = ops.loss_partial_stride()
    # ---- fp32 reference ----
    ta = [torch.empty(M, u, device=DEV) for u in UNITS]
    ops.linear_fwd(obs, W[0], b[0], ta[0], act, norm_mean=nm, norm_std=ns)
    ops.linear_fwd(ta[0], W[1], b[1], ta[1], act)
    ops.linear_fwd(ta[1], W[2], b[2], ta[2], act)
    mu_r, sg_r = old_mu.clone(), old_sigma.clone()
    d_head = torch.empty(M, A + 1, device=DEV); d_a3 = torch.empty(M, UNITS[2], device=DEV)
    partials = torch.zeros(n_tiles, stride, dtype=torch.float64, device=DEV)
    nb = ops.ppo_head_loss(ta[2], Wh, bh, logstd, actions, mu_r, sg_r, old_v, ret, old_nlp, adv, None, M, 0, M, A, cfg, None,
                           d_head, d_a3, act, partials)
    stats_r = torch.zeros(16, device=DEV); dls_r = torch.empty(A, device=DEV)
    ops.ppo_loss_finalize(partials, nb, A, ec, stats_r, dls_r)
    # ---- two launches of the tensor-core forward on the same inputs ----
    tb = ops.tc_tile_bytes(D, UNITS, A)
    wpack = torch.zeros(ops.tc_pack_bytes(D, UNITS, A), dtype=torch.uint8, device=DEV)
    ops.tc_pack_weights(W[0], W[1], W[2], Wh, D, UNITS, A, wpack)
    runs = []
    for _ in range(2):
        r = dict(act=[torch.full((n_tiles * tb[i],), 0xA5, dtype=torch.uint8, device=DEV) for i in range(3)],
                 dhead=torch.full((n_tiles * tb[3],), 0xA5, dtype=torch.uint8, device=DEV),
                 xt=torch.full((n_tiles * ops.tc_xtile_bytes(D, UNITS, A),), 0xA5, dtype=torch.uint8, device=DEV),
                 partials=torch.zeros(132, stride, dtype=torch.float64, device=DEV), mu=old_mu.clone(), sg=old_sigma.clone())
        r['nb'] = ops.tc_mlp_fwd_train(obs, M, 0, D, nm, ns, wpack, b, bh, logstd, UNITS, M, A, actions, r['mu'], r['sg'], old_v, ret,
                                       old_nlp, adv, None, cfg, None, r['act'], r['dhead'], r['partials'], xtile=r['xt'], activation=act)
        runs.append(r)
    torch.cuda.synchronize()
    t, u = runs
    assert t['nb'] == 70 and u['nb'] == 70
    for i in range(3):
        assert torch.equal(t['act'][i], u['act'][i]), i
    for k in ('dhead', 'xt', 'partials', 'mu', 'sg'):
        assert torch.equal(t[k], u[k]), k
    # ---- against the fp32 kernels ----
    for i, C in enumerate(UNITS):
        got = decode_tiles(t['act'][i], n_tiles, C)[:M]
        assert rel_l2(got, ta[i]) < 1.5e-2, (i, rel_l2(got, ta[i]))
    torch.testing.assert_close(t['mu'], mu_r, rtol=0, atol=4e-2)
    assert torch.equal(t['sg'], sg_r)
    stats_t = torch.zeros(16, device=DEV); dls_t = torch.empty(A, device=DEV)
    ops.ppo_loss_finalize(t['partials'], t['nb'], A, ec, stats_t, dls_t)
    for k in (0, 1, 2, 3, 4):
        assert float(stats_t[k]) == pytest.approx(float(stats_r[k]), rel=4e-2, abs=2e-3), (k, stats_t[:8], stats_r[:8])
    assert float(stats_t[5]) == float(stats_r[5])
    dh = decode_tiles(t['dhead'], n_tiles, 16)
    assert torch.equal(dh[M:], torch.zeros_like(dh[M:]))       # padded rows of the partial tile contribute nothing
    dh = dh[:M, :A + 1]
    assert rel_l2(dh, d_head) < 6e-2 and cosine(dh, d_head) > 0.998, (rel_l2(dh, d_head), cosine(dh, d_head))
    assert rel_l2(dls_t, dls_r) < 5e-2


@pytest.mark.parametrize('act', ACTS)
def test_tc_rollout_16384(act):
    from rl_games_b200 import ops
    N = 16384
    g = torch.Generator().manual_seed(40 + act)
    W, b, Wh, bh, logstd = make_net(g)
    obs = (torch.randn(N, D, generator=g) * 2).to(DEV)
    nm = (torch.randn(D, generator=g) * 0.3).to(DEV); ns = (torch.rand(D, generator=g) + 0.7).to(DEV)
    noise = torch.randn(N, A, generator=g).to(DEV)
    vm, vv = torch.tensor([1.5], dtype=torch.float64, device=DEV), torch.tensor([4.0], dtype=torch.float64, device=DEV)
    lo, hi = torch.full((A,), -1.0, device=DEV), torch.full((A,), 1.0, device=DEV)
    dones_cur = (torch.rand(N, generator=g) < 0.3).to(torch.uint8).to(DEV)

    def outs():
        return dict(a=torch.empty(N, A, device=DEV), m=torch.empty(N, A, device=DEV), s=torch.empty(N, A, device=DEV),
                    nl=torch.empty(N, device=DEV), v=torch.empty(N, device=DEV), e=torch.empty(N, A, device=DEV),
                    d=torch.zeros(N, dtype=torch.uint8, device=DEV), vo=torch.empty(N, device=DEV))
    ra = [torch.empty(N, u, device=DEV) for u in UNITS]
    ops.linear_fwd(obs, W[0], b[0], ra[0], act, norm_mean=nm, norm_std=ns)
    ops.linear_fwd(ra[0], W[1], b[1], ra[1], act); ops.linear_fwd(ra[1], W[2], b[2], ra[2], act)
    r = outs()
    ops.policy_head_sample(ra[2], Wh, bh, logstd, vm, vv, True, noise, 1, None, 0, r['a'], r['m'], r['s'], r['nl'], r['v'], r['e'], True,
                           lo, hi, dones_cur, r['d'], None, None, N, A)
    wpack = torch.zeros(ops.tc_pack_bytes(D, UNITS, A), dtype=torch.uint8, device=DEV)
    ops.tc_pack_weights(W[0], W[1], W[2], Wh, D, UNITS, A, wpack)
    runs = []
    for _ in range(2):
        t = outs()
        ops.tc_mlp_fwd_rollout(obs, D, nm, ns, wpack, b, bh, logstd, UNITS, N, A, vm, vv, True, noise, 1, None, 0, t['a'], t['m'],
                               t['s'], t['nl'], t['v'], t['e'], True, lo, hi, dones_cur, t['d'], None, None, activation=act)
        ops.tc_mlp_fwd_rollout(obs, D, nm, ns, wpack, b, bh, logstd, UNITS, N, A, vm, vv, True, None, 0, None, 0, None, None, None, None,
                               t['vo'], None, False, None, None, None, None, None, None, values_only=True, activation=act)
        runs.append(t)
    torch.cuda.synchronize()
    t, u = runs
    for k in t:
        assert torch.equal(t[k], u[k]), k
    assert torch.equal(t['vo'], t['v'])
    torch.testing.assert_close(t['m'], r['m'], rtol=0, atol=4e-2)
    torch.testing.assert_close(t['a'], r['a'], rtol=0, atol=4e-2)
    torch.testing.assert_close(t['v'], r['v'], rtol=0, atol=8e-2)
    assert torch.equal(t['s'], r['s']) and torch.equal(t['d'], r['d'])
    torch.testing.assert_close(t['nl'], r['nl'], rtol=1e-5, atol=1e-4)
    torch.testing.assert_close(t['e'], torch.clamp(t['a'], -1, 1), rtol=0, atol=1e-6)
