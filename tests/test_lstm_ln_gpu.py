"""Layer-normed LSTM policies (rnn.layer_norm: True) on the GPU: the two LSTM-cell + LayerNorm kernels against autograd of a torch
restatement, the fp32 agent against the reference's golden runs (eager and CUDA graph), the layer-wise tensor-core agent against the
fp32 agent, and the c4 geometry with the option against the CPU oracle."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _lstm_ln_oracle as LO  # noqa: E402
from oracle import ppo_oracle as O  # noqa: E402
from test_agent_gpu import DEV, TapeEnvGPU, _check_epoch, make_agent  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _rnn(units, before_mlp):
    return {'rnn': {'name': 'lstm', 'units': units, 'layers': 1, 'before_mlp': before_mlp, 'layer_norm': True}}


def _scatter_rows(S, rpc, stride):
    s = torch.arange(S)
    return (s // rpc) * stride + s % rpc


def _cell_ln_ref(G, cin, w, b, m):
    """torch restatement: pre-activations G [S,4Hd] and masked c_{t-1} -> (y, h, c, h*m, c*m)"""
    i, f, g, o = G.chunk(4, dim=1)
    c = torch.sigmoid(f) * cin + torch.sigmoid(i) * torch.tanh(g)
    h = torch.sigmoid(o) * torch.tanh(c)
    y = F.layer_norm(h, (h.shape[1],), w, b, 1e-5)
    return y, h, c, h * m, c * m


def _inputs(S, Hd, rpc, seed):
    g = torch.Generator().manual_seed(seed)
    G = torch.randn(S, 4 * Hd, generator=g) * 1.5
    cin = torch.randn(S, Hd, generator=g)
    w, b = 1.0 + 0.3 * torch.randn(Hd, generator=g), 0.2 * torch.randn(Hd, generator=g)
    # done flags of the next step, chunk-mapped like the arena's: row s -> (s / rpc) * (rpc + 3) + s % rpc
    dstride = rpc + 3
    done = (torch.rand(((S + rpc - 1) // rpc) * dstride, generator=g) < 0.3).to(torch.uint8)
    m = 1.0 - done[_scatter_rows(S, rpc, dstride)].float().unsqueeze(1)
    return G, cin, w, b, done, dstride, m


@pytest.mark.parametrize('Hd', [12, 64, 256, 1024])
def test_cell_ln_forward_matches_torch(Hd):
    """a partial last CTA of rows (S = 37), scattered output rows, done-masked carries; y dense and scattered"""
    S, rpc, sstride = 37, 5, 9
    G, cin, w, b, done, dstride, m = _inputs(S, Hd, rpc, seed=Hd)
    y_ref, h_ref, c_ref, hn_ref, cn_ref = _cell_ln_ref(G.double(), cin.double(), w.double(), b.double(), m.double())
    d = lambda t: t.to(DEV).contiguous()     # noqa: E731
    gates, cin_d, w_d, b_d, done_d = d(G), d(cin), d(w), d(b), d(done)
    c_out, h_out, y_out = (torch.zeros(S, Hd, device=DEV) for _ in range(3))
    nrows = int(_scatter_rows(S, rpc, sstride).max()) + 1
    y_sc = torch.full((nrows, Hd), 7.0, device=DEV)
    hin_n, cin_n = torch.zeros(S, Hd, device=DEV), torch.zeros(S, Hd, device=DEV)
    mean, rstd = torch.zeros(S, device=DEV), torch.zeros(S, device=DEV)
    from rl_games_b200 import ops
    ops.lstm_cell_ln_fwd(gates, cin_d, c_out, h_out, w_d, b_d, S, Hd, y_out=y_out, y_scatter=y_sc, scatter_rpc=rpc, scatter_stride=sstride,
                         hin_next=hin_n, cin_next=cin_n, done_next=done_d, done_rpc=rpc, done_stride=dstride, mean=mean, rstd=rstd)
    torch.cuda.synchronize()
    tol = dict(rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(c_out.cpu().double(), c_ref, **tol)
    torch.testing.assert_close(h_out.cpu().double(), h_ref, **tol)
    torch.testing.assert_close(y_out.cpu().double(), y_ref, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(hin_n.cpu().double(), hn_ref, **tol)
    torch.testing.assert_close(cin_n.cpu().double(), cn_ref, **tol)
    rows = _scatter_rows(S, rpc, sstride)
    torch.testing.assert_close(y_sc.cpu()[rows], y_out.cpu(), rtol=0, atol=0)
    untouched = torch.ones(nrows, dtype=torch.bool)
    untouched[rows] = False
    assert (y_sc.cpu()[untouched] == 7.0).all()
    torch.testing.assert_close(mean.cpu().double(), h_ref.mean(1), **tol)
    torch.testing.assert_close(rstd.cpu().double(), 1.0 / torch.sqrt(h_ref.var(1, unbiased=False) + 1e-5), rtol=1e-4, atol=1e-4)
    acts = torch.cat([torch.sigmoid(G[:, :2 * Hd]), torch.tanh(G[:, 2 * Hd:3 * Hd]), torch.sigmoid(G[:, 3 * Hd:])], 1)
    torch.testing.assert_close(gates.cpu(), acts, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize('Hd', [12, 64, 256, 1024])
def test_cell_ln_backward_matches_autograd(Hd):
    """dgates / dcin / dgamma / dbeta against autograd of the restatement: dy through a scattered buffer, recurrent dh / dc of the next
    step through done-masked carries, dgamma / dbeta as split partials summed by reduce_splits; bit-reproducible"""
    from rl_games_b200 import ops
    S, rpc, sstride, n_splits, P = 37, 5, 9, 6, Hd + 40
    G, cin, w, b, done, dstride, m = _inputs(S, Hd, rpc, seed=100 + Hd)
    g = torch.Generator().manual_seed(200 + Hd)
    nrows = int(_scatter_rows(S, rpc, sstride).max()) + 1
    dY_full = torch.randn(nrows, Hd, generator=g)
    dhn, dcn = torch.randn(S, Hd, generator=g), torch.randn(S, Hd, generator=g)
    rows = _scatter_rows(S, rpc, sstride)
    Gr, cr, wr, br = (t.double().clone().requires_grad_(True) for t in (G, cin, w, b))
    y, _, _, hn, cn = _cell_ln_ref(Gr, cr, wr, br, m.double())
    ((y * dY_full[rows].double()).sum() + (hn * dhn.double()).sum() + (cn * dcn.double()).sum()).backward()
    d = lambda t: t.to(DEV).contiguous()     # noqa: E731
    gates, cin_d, w_d, b_d, done_d = d(G), d(cin), d(w), d(b), d(done)
    c_t, h_t = torch.zeros(S, Hd, device=DEV), torch.zeros(S, Hd, device=DEV)
    y_d, mean, rstd = torch.zeros(S, Hd, device=DEV), torch.zeros(S, device=DEV), torch.zeros(S, device=DEV)
    ops.lstm_cell_ln_fwd(gates, cin_d, c_t, h_t, w_d, b_d, S, Hd, y_out=y_d, mean=mean, rstd=rstd)
    outs = []
    for _ in range(2):
        dgates, dcin = torch.zeros(S, 4 * Hd, device=DEV), torch.zeros(S, Hd, device=DEV)
        pw, pb = torch.full((n_splits, P), float('nan'), device=DEV), torch.full((n_splits, P), float('nan'), device=DEV)
        ops.lstm_cell_ln_bwd(gates, c_t, cin_d, d(dY_full), w_d, mean, rstd, pw, pb, n_splits, dgates, dcin, S, Hd,
                             scatter_rpc=rpc, scatter_stride=sstride, dhin_next=d(dhn), dcin_next=d(dcn), done_next=done_d, done_rpc=rpc,
                             done_stride=dstride, split_stride=P)
        dgamma, dbeta = torch.zeros(Hd, device=DEV), torch.zeros(Hd, device=DEV)
        ops.reduce_splits(pw, dgamma, Hd, n_splits, split_stride=P)
        ops.reduce_splits(pb, dbeta, Hd, n_splits, split_stride=P)
        torch.cuda.synchronize()
        outs.append((dgates.cpu(), dcin.cpu(), dgamma.cpu(), dbeta.cpu(), pw.cpu(), pb.cpu()))
    for a, b_ in zip(outs[0], outs[1]):
        assert torch.equal(a.nan_to_num(0.0), b_.nan_to_num(0.0))
    dgates, dcin, dgamma, dbeta, pw, pb = outs[0]
    assert not pw[:, :Hd].isnan().any() and pw[:, Hd:].isnan().all()      # every split row written, nothing past Hd
    tol = dict(rtol=1e-4, atol=3e-5)
    torch.testing.assert_close(dgates.double(), Gr.grad, **tol)
    torch.testing.assert_close(dcin.double(), cr.grad, **tol)
    torch.testing.assert_close(dgamma.double(), wr.grad, **tol)
    torch.testing.assert_close(dbeta.double(), br.grad, **tol)


def test_cell_ln_backward_split_partials_at_separate_offsets():
    """the agent's layout: gamma and beta at their own 8-aligned offsets of a [n_splits, P] partial arena, every split row written"""
    from rl_games_b200 import ops
    S, Hd, n_splits = 300, 64, 16
    o_w, o_b, P = 8, 8 + 64, 200
    G, cin, w, b, _, _, _ = _inputs(S, Hd, 7, seed=5)
    g = torch.Generator().manual_seed(6)
    dY = torch.randn(S, Hd, generator=g)
    Gr, cr, wr, br = (t.double().clone().requires_grad_(True) for t in (G, cin, w, b))
    y, *_ = _cell_ln_ref(Gr, cr, wr, br, torch.ones(S, 1, dtype=torch.float64))
    (y * dY.double()).sum().backward()
    d = lambda t: t.to(DEV).contiguous()     # noqa: E731
    gates, cin_d, w_d, b_d = d(G), d(cin), d(w), d(b)
    c_t, h_t = torch.zeros(S, Hd, device=DEV), torch.zeros(S, Hd, device=DEV)
    y_d, mean, rstd = torch.zeros(S, Hd, device=DEV), torch.zeros(S, device=DEV), torch.zeros(S, device=DEV)
    ops.lstm_cell_ln_fwd(gates, cin_d, c_t, h_t, w_d, b_d, S, Hd, y_out=y_d, mean=mean, rstd=rstd)
    part = torch.full((n_splits, P), float('nan'), device=DEV)
    dgates, dcin = torch.zeros(S, 4 * Hd, device=DEV), torch.zeros(S, Hd, device=DEV)
    ops.lstm_cell_ln_bwd(gates, c_t, cin_d, d(dY), w_d, mean, rstd, part[0, o_w:], part[0, o_b:], n_splits, dgates, dcin, S, Hd,
                         split_stride=P)
    out = torch.zeros(P, device=DEV)
    ops.reduce_splits(part[0, o_w:], out[o_w:], 2 * Hd, n_splits, split_stride=P)
    torch.cuda.synchronize()
    assert not part[:, o_w:o_b + Hd].isnan().any()
    assert part[:, :o_w].isnan().all() and part[:, o_b + Hd:].isnan().all()
    torch.testing.assert_close(out[o_w:o_w + Hd].cpu().double(), wr.grad, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(out[o_b:o_b + Hd].cpu().double(), br.grad, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(dgates.cpu().double(), Gr.grad, rtol=1e-4, atol=1e-5)


def _golden_run(name, graph):
    g = torch.load(os.path.join(GOLDEN, name), weights_only=False)
    assert g['rnn_layer_norm']
    cfgk = g['config']
    over = {k: cfgk[k] for k in ('clip_value', 'use_smooth_clamp', 'bound_loss_type', 'bounds_loss_coef', 'entropy_coef', 'truncate_grads',
                                 'value_bootstrap', 'mini_epochs', 'lr_schedule', 'critic_coef', 'seq_length', 'learning_rate',
                                 'kl_threshold', 'max_epochs', 'normalize_input', 'normalize_value', 'normalize_advantage', 'e_clip', 'tau',
                                 'gamma') if k in cfgk}
    over.setdefault('lr_schedule', None)
    over['b200_cuda_graph'] = graph
    env = TapeEnvGPU(g['obs_tape'], g['done_tape'], g['timeout_tape'], g['A'], g['autoreset'])
    agent = make_agent(over, g['N'], g['H'], g['D'], g['A'], g['units'], g['mb'], env, g['init_state'],
                       network_over=_rnn(g['rnn_units'], g['rnn_before_mlp']))
    assert agent.is_rnn and agent.model.rnn_layer_norm and not agent.use_tc
    for ep, ref in enumerate(g['epochs_out']):
        agent.epoch_num += 1
        agent.train_epoch(noise=g['noise'][ep].to(DEV))
        assert torch.equal(agent.dones_buf.cpu(), ref['mb_dones'])
        torch.testing.assert_close(agent.values.cpu().unsqueeze(2), ref['mb_values'], rtol=1e-4, atol=1e-5)
        nmb = agent.num_minibatches
        st = agent.last_stats
        torch.testing.assert_close(torch.stack([st[e * nmb:(e + 1) * nmb, 4].mean() for e in range(agent.mini_epochs_num)]),
                                   ref['kls'], rtol=2e-3, atol=2e-6)
        _check_epoch(agent, ref['state'], ref['dataset'], {'a': ref['a_losses'], 'c': ref['c_losses'], 'e': ref['entropies']},
                     ref['last_lr'], g['units'], lstm=True)
        sd = agent.model.state_dict()
        for k in LO.LN_NAMES:
            torch.testing.assert_close(sd[k].cpu(), ref['state'][k], rtol=1e-3, atol=2e-5, msg=lambda m: k + ': ' + m)
    return agent


@pytest.mark.parametrize('name', ['agent_lstm_ln.pt', 'agent_lstm_ln_after.pt', 'agent_lstm_ln_after_masked.pt'])
@pytest.mark.parametrize('graph', [False, True])
def test_layer_normed_lstm_agent_matches_reference_golden(name, graph):
    _golden_run(name, graph)


@pytest.mark.parametrize('before', [True, False])
def test_layerwise_tensor_core_path_tracks_fp32_agent(before):
    """mixed_precision: True on a layer-normed LSTM policy: the gate GEMMs on the tensor cores, the LayerNorm in fp32 on both paths; bf16
    tolerance class against the fp32 agent (as tests/test_agent_gpu.py::test_layerwise_tensor_core_path_tracks_fp32_agent)"""
    N, H, D, A, mb, units, rnn = 256, 8, 44, 5, 1024, [64, 32], 32
    obs_tape, done_tape, tout_tape = O.make_tapes(H + 1, N, D, seed=52, p_done=0.08)
    params = LO.init_params(D, units, A, seed=7, rnn_units=rnn, rnn_before_mlp=before, ln_seed=3)
    g = torch.Generator().manual_seed(17)
    noise = torch.randn(H, N, A, generator=g).to(DEV)
    agents = []
    for mp in (False, True):
        a = make_agent({'mixed_precision': mp, 'mini_epochs': 2, 'b200_cuda_graph': False, 'seq_length': 4}, N, H, D, A, units, mb,
                       TapeEnvGPU(obs_tape, done_tape, tout_tape, A), params, network_over=_rnn(rnn, before))
        assert a.gemm_tc == mp and not a.use_tc and a.model.rnn_layer_norm
        a.epoch_num += 1
        a.train_epoch(noise=noise)
        agents.append(a)
    f, t = agents
    torch.testing.assert_close(t.values, f.values, rtol=0, atol=6e-2)
    torch.testing.assert_close(t.mus, f.mus, rtol=0, atol=6e-2)
    sf, st = f.last_stats, t.last_stats
    torch.testing.assert_close(st[:, 0], sf[:, 0], rtol=0.1, atol=2e-2)
    torch.testing.assert_close(st[:, 1], sf[:, 1], rtol=0.1, atol=2e-2)
    sdf, sdt = f.model.state_dict(), t.model.state_dict()
    for k in LO.param_names(len(units)):
        if k.endswith('weight') or 'weight_' in k:
            du_f = (sdf[k].cpu() - params[k]).flatten()
            du_t = (sdt[k].cpu() - params[k]).flatten()
            cos = float(du_f @ du_t / (du_f.norm() * du_t.norm() + 1e-20))
            assert cos > 0.8, (k, cos)


def test_lstm_ln_c4_geometry_full_width_vs_oracle():
    """the c4 geometry (tests/test_agent_gpu.py::test_lstm_c4_geometry_full_width_vs_oracle: 8192 envs, obs 348, 17 actions, LSTM 256 before
    the MLP [512, 256, 128], seq_length 4, horizon 8, one mini-epoch of 4 minibatches) with rnn.layer_norm, fp32 kernels vs the oracle"""
    N, H, D, A, units, mb, hid = 8192, 8, 348, 17, [512, 256, 128], 16384, 256
    g = torch.Generator().manual_seed(42)
    obs_tape = torch.randn(H + 1, N, D, generator=g) * 1.5 + 0.3
    done_tape = (torch.rand(H + 1, N, generator=g) < 0.05).to(torch.uint8)
    tout_tape = (torch.rand(H + 1, N, generator=g) < 0.3) & done_tape.bool()
    params = LO.init_params(D, units, A, seed=9, rnn_units=hid, ln_seed=4)
    noise = torch.randn(H, N, A, generator=g)
    cfg = {'mini_epochs': 1, 'rnn_units': hid, 'seq_length': 4}
    oag = LO.make_agent(O.TapeEnv(obs_tape, done_tape, tout_tape), params, D, A, units, N, H, mb, cfg)
    oag.obs = oag.env_reset()
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    out = oag.train_epoch(noise)
    agent = make_agent({'mini_epochs': 1, 'seq_length': 4}, N, H, D, A, units, mb, TapeEnvGPU(obs_tape, done_tape, tout_tape, A), params,
                       network_over=_rnn(hid, True))
    assert agent.is_rnn and not agent.use_tc and agent.model.rnn_layer_norm and agent.model.rnn_units == hid
    agent.epoch_num += 1
    agent.train_epoch(noise=noise.to(DEV))
    st = agent.last_stats
    torch.testing.assert_close(agent.values.cpu(), oag.buf['values'].squeeze(2), rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(agent.rnn_h.cpu(), oag.rnn_states[0][0], rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(st[:, 0], torch.stack(out['a_loss']), rtol=5e-3, atol=1e-5)
    torch.testing.assert_close(st[:, 1], torch.stack(out['c_loss']), rtol=5e-3, atol=1e-5)
    torch.testing.assert_close(st[:, 4], torch.stack(out['kl']), rtol=1e-2, atol=1e-6)
    assert agent.last_lr == pytest.approx(oag.last_lr, rel=1e-12)
    sd = agent.model.state_dict()
    for k in LO.param_names(3):
        torch.testing.assert_close(sd[k].cpu(), oag.model.p[k].detach(), rtol=1e-3, atol=5e-5, msg=lambda m: k + ': ' + m)
