"""The LSTM policy's backward on the GPU against fp64 references, not only through Adam.

(a) The plain cell kernels (csrc/rnn.cu: lstm_cell_fwd, lstm_cell_bwd, rnn_mask_rows) against fp64 torch, with every optional argument
the agent passes: scattered MLP-order output rows, next-step carries masked by chunk-mapped done flags, the recurrent dh / dc of the next
step, the in-place state zeroing of the rollout; saturating pre-activations; outputs filled with NaN beforehand, so a row that is not
written, or written where it must not be, shows.  Refused argument combinations write nothing.
Measured on an H100 SXM (80 GB, 700 W): worst error 4.0e-7 (forward) and 2.4e-7 (backward) of the output's max |value|; the bound is
1e-6 of that scale (about 3x), plus rtol 1e-5.

(b) The reduced flat gradient of one CUDA minibatch update (agent._minibatch_update; gv['grad'], which the optimiser kernel reads as const
and clips on the fly, so it holds the unclipped gradient even with truncate_grads and a grad_norm far below the gradient's norm) against
the fp64 autograd gradient of the same minibatch (tests/_lstm_grad_ref.py), per parameter tensor: max |g - g_ref| / max |g_ref| and the
norm ratio |g| / |g_ref|.  Adam's first step is lr * sign(g) and the clip rescales the whole gradient, so the agent tests that compare
weights after training can not be relied on to see a gradient of the wrong size; these can.  The layer-wise tensor-core path is held to
the same reference with the operands of its GEMMs rounded to bf16 (its heads run in fp32 as well): against the plain fp64 gradient one of
its minibatches here is off by 0.47 of scale -- and so is the bf16-operand reference, which agrees with the kernels to 3e-3 -- a
minibatch whose gradient is that sensitive to bf16 rounding, not a kernel error.
Measured on an H100 SXM (80 GB, 700 W), worst over every case, minibatch and tensor: fp32 kernels relative error 3.0e-5, norm ratio
within 2.5e-5 of 1; tensor-core kernels relative error 1.0e-2, norm ratio within 7.5e-3 of 1.  Bounds (about 3x): fp32 1e-4 / 1e-4,
tensor cores 3e-2 / 2.5e-2.
"""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _lstm_grad_ref as GR  # noqa: E402
import _lstm_ln_oracle as LO  # noqa: E402
from oracle import ppo_oracle as O  # noqa: E402
from rl_games_b200._lib import B200RLError  # noqa: E402
from test_agent_gpu import DEV, TapeEnvGPU  # noqa: E402

pytestmark = pytest.mark.gpu

CELL_RTOL, CELL_ATOL = 1e-5, 1e-6          # atol x the output's max |value|
GRAD_TOL = {False: (1e-4, 1e-4), True: (3e-2, 2.5e-2)}      # mixed_precision -> (relative error, |norm ratio - 1|)
NAN = float('nan')


# ------------------------------------------------------------------------------------------------------------------- (a) cell kernels
def _chunk_rows(S, rpc, stride):
    s = torch.arange(S)
    return (s // rpc) * stride + s % rpc


def _cell_fwd_ref(G, cin):
    """fp64: pre-activations G [S, 4Hd], masked c_{t-1} -> activations (i, f, g, o), c, h"""
    i, f, g, o = G.chunk(4, dim=1)
    i, f, g, o = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)
    c = f * cin + i * g
    return torch.cat([i, f, g, o], 1), c, o * torch.tanh(c)


def _pre_activations(S, Hd, gen):
    """N(0, 1.5) pre-activations with every 7th entry pushed to a saturating |x| in [10, 30]"""
    G = torch.randn(S, 4 * Hd, generator=gen, dtype=torch.float64) * 1.5
    sat = torch.rand(S, 4 * Hd, generator=gen) < 1.0 / 7
    G[sat] = torch.sign(G[sat]) * (10.0 + 20.0 * torch.rand(int(sat.sum()), generator=gen, dtype=torch.float64))
    return G.float()


class _Layout:
    """The agent's BPTT window layout: S = sequences of epm envs x J windows, step t; arena done flags [J*T, N] read for step t+1 at
    dn[t + 1, e0:] with (done_rpc = epm, done_stride = T*N); MLP-order rows t_hmlp[t*epm:] with (scatter_rpc = epm, scatter_stride = T*epm)"""

    def __init__(self, S, gen, epm=5, T=3, t=1):
        self.epm, self.T, self.t = min(epm, S), T, t
        self.J = (S + self.epm - 1) // self.epm
        self.N, self.e0 = 2 * self.epm + 1, self.epm
        self.dn = (torch.rand(self.J * T, self.N, generator=gen) < 0.3).to(torch.uint8)
        self.mlp_rows = self.J * T * self.epm
        self.sc_rows = _chunk_rows(S, self.epm, T * self.epm) + t * self.epm       # rows of the MLP-order buffer
        d = self.dn.reshape(-1)
        self.m_next = 1.0 - d[_chunk_rows(S, self.epm, T * self.N) + (t + 1) * self.N + self.e0].double().unsqueeze(1)

    def done_next(self):
        return self.dn.to(DEV)[self.t + 1, self.e0:]


def _max_err(out, ref):
    out, ref = out.double().cpu(), ref.double().cpu()
    return float((out - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)


def _close(out, ref, what):
    out, ref = out.double().cpu(), ref.double().cpu()
    assert not out.isnan().any(), f'{what}: unwritten (NaN) elements'
    torch.testing.assert_close(out, ref, rtol=CELL_RTOL, atol=CELL_ATOL * max(float(ref.abs().max()), 1e-30), msg=lambda m: f'{what}: {m}')


CELL_HD = [1, 7, 32, 33, 256, 1024]
CELL_S = [1, 255, 4097]


@pytest.mark.parametrize('S', CELL_S)
@pytest.mark.parametrize('Hd', CELL_HD)
def test_lstm_cell_fwd_matches_fp64(Hd, S):
    from rl_games_b200 import ops
    gen = torch.Generator().manual_seed(1000 * Hd + S)
    G = _pre_activations(S, Hd, gen)
    cin = torch.randn(S, Hd, generator=gen) * 2.0
    L = _Layout(S, gen)
    acts, c_ref, h_ref = _cell_fwd_ref(G.double(), cin.double())
    worst = 0.0
    for variant in ('bare', 'scatter_carries_dones', 'carries'):
        gates = G.to(DEV)
        c_out, h_out = torch.full((S, Hd), NAN, device=DEV), torch.full((S, Hd), NAN, device=DEV)
        hmlp = torch.full((L.mlp_rows, Hd), NAN, device=DEV)
        hin_n, cin_n = torch.full((S, Hd), NAN, device=DEV), torch.full((S, Hd), NAN, device=DEV)
        kw = {}
        if variant == 'scatter_carries_dones':
            kw = dict(h_scatter=hmlp[L.t * L.epm:], scatter_rpc=L.epm, scatter_stride=L.T * L.epm, hin_next=hin_n, cin_next=cin_n,
                      done_next=L.done_next(), done_rpc=L.epm, done_stride=L.T * L.N)
        elif variant == 'carries':
            kw = dict(hin_next=hin_n, cin_next=cin_n)
        ops.lstm_cell_fwd(gates, cin.to(DEV), c_out, h_out, S, Hd, **kw)
        torch.cuda.synchronize()
        _close(gates, acts, f'{variant} gates (activations in place)')
        _close(c_out, c_ref, f'{variant} c')
        _close(h_out, h_ref, f'{variant} h')
        worst = max(worst, _max_err(gates, acts), _max_err(c_out, c_ref), _max_err(h_out, h_ref))
        hm = hmlp.cpu()
        if variant == 'scatter_carries_dones':
            assert torch.equal(hm[L.sc_rows], h_out.cpu()), 'scattered rows differ from the dense h'
            untouched = torch.ones(L.mlp_rows, dtype=torch.bool)
            untouched[L.sc_rows] = False
            assert hm[untouched].isnan().all(), 'rows outside the scatter pattern were written'
            _close(hin_n, h_ref * L.m_next, 'hin_next')
            _close(cin_n, c_ref * L.m_next, 'cin_next')
            assert (L.m_next == 0).any() or S < 4
        elif variant == 'carries':
            assert torch.equal(hin_n.cpu(), h_out.cpu()) and torch.equal(cin_n.cpu(), c_out.cpu())
            assert hm.isnan().all()
        else:
            assert hm.isnan().all() and hin_n.isnan().all().item() and cin_n.isnan().all().item()
    print(f'lstm_cell_fwd Hd={Hd} S={S}: worst relative error {worst:.2e}')


@pytest.mark.parametrize('S', CELL_S)
@pytest.mark.parametrize('Hd', CELL_HD)
def test_lstm_cell_bwd_matches_fp64_autograd(Hd, S):
    """dgates / dcin against autograd of the fp64 forward: dh from the scattered MLP-order gradient rows, dh / dc of the next step through the
    done-masked carries, each present and absent"""
    from rl_games_b200 import ops
    gen = torch.Generator().manual_seed(7000 * Hd + S)
    G = _pre_activations(S, Hd, gen)
    cin = torch.randn(S, Hd, generator=gen) * 2.0
    L = _Layout(S, gen)
    dH_full = torch.randn(L.mlp_rows, Hd, generator=gen, dtype=torch.float64)
    dhn, dcn = torch.randn(S, Hd, generator=gen, dtype=torch.float64), torch.randn(S, Hd, generator=gen, dtype=torch.float64)
    # the forward the backward reads: activations and c_t from the kernel itself
    gates, c_t, h_t = G.to(DEV), torch.empty(S, Hd, device=DEV), torch.empty(S, Hd, device=DEV)
    ops.lstm_cell_fwd(gates, cin.to(DEV), c_t, h_t, S, Hd)
    worst = 0.0
    for variant in ('dH_next_dones', 'dH', 'next_dones', 'next'):
        use_dH, use_next, use_done = 'dH' in variant, 'next' in variant, 'dones' in variant
        Gr, cr = G.double().requires_grad_(True), cin.double().requires_grad_(True)
        _, c, h = _cell_fwd_ref(Gr, cr)
        m = L.m_next if use_done else torch.ones(S, 1, dtype=torch.float64)
        loss = torch.zeros((), dtype=torch.float64)
        if use_dH:
            loss = loss + (h * dH_full[L.sc_rows]).sum()
        if use_next:
            loss = loss + (h * m * dhn).sum() + (c * m * dcn).sum()
        loss.backward()
        dgates, dcin = torch.full((S, 4 * Hd), NAN, device=DEV), torch.full((S, Hd), NAN, device=DEV)
        kw = {}
        if use_dH:
            kw.update(dH=dH_full.float().to(DEV)[L.t * L.epm:], scatter_rpc=L.epm, scatter_stride=L.T * L.epm)
        if use_next:
            kw.update(dhin_next=dhn.float().to(DEV), dcin_next=dcn.float().to(DEV))
        if use_done:
            kw.update(done_next=L.done_next(), done_rpc=L.epm, done_stride=L.T * L.N)
        ops.lstm_cell_bwd(gates, c_t, cin.to(DEV), dgates, dcin, S, Hd, **kw)
        torch.cuda.synchronize()
        _close(dgates, Gr.grad, f'{variant} dgates')
        _close(dcin, cr.grad, f'{variant} dcin')
        worst = max(worst, _max_err(dgates, Gr.grad), _max_err(dcin, cr.grad))
    print(f'lstm_cell_bwd Hd={Hd} S={S}: worst relative error {worst:.2e}')


@pytest.mark.parametrize('S', CELL_S)
@pytest.mark.parametrize('Hd', CELL_HD)
def test_rnn_mask_rows_matches_torch(Hd, S):
    """the window-initial states (rows of rnn_h0[0, e0:] gathered with (in_rpc = epm, in_stride = N), masked by chunk-mapped done flags), a
    plain gather, and the rollout's in-place zeroing of done rows; rows past S are never written"""
    from rl_games_b200 import ops
    gen = torch.Generator().manual_seed(500 * Hd + S)
    L = _Layout(S, gen)
    h0 = torch.randn(L.J, L.N, Hd, generator=gen)
    rows = _chunk_rows(S, L.epm, L.N) + L.e0
    src = h0.reshape(-1, Hd)[rows]
    dn0 = L.dn.reshape(-1)[_chunk_rows(S, L.epm, L.T * L.N) + L.e0]
    for done in (True, False):
        out = torch.full((S + 3, Hd), NAN, device=DEV)
        kw = dict(done=L.dn.to(DEV)[0, L.e0:], done_rpc=L.epm, done_stride=L.T * L.N) if done else {}
        ops.rnn_mask_rows(h0.to(DEV)[0, L.e0:], L.epm, L.N, out, S, Hd, **kw)
        torch.cuda.synchronize()
        ref = src * (1.0 - dn0.float().unsqueeze(1)) if done else src
        assert torch.equal(out[:S].cpu(), ref) and out[S:].isnan().all().item()
    # in place, as the rollout zeroes the states of finished episodes: (in_rpc = N, in_stride = 0, done_rpc = N)
    h = torch.randn(S, Hd, generator=gen)
    dones = (torch.rand(S, generator=gen) < 0.3).to(torch.uint8)
    hd = h.to(DEV)
    ops.rnn_mask_rows(hd, S, 0, hd, S, Hd, done=dones.to(DEV), done_rpc=S)
    torch.cuda.synchronize()
    assert torch.equal(hd.cpu(), h * (1.0 - dones.float().unsqueeze(1)))


def _refused(fn, *a, **kw):
    try:
        fn(*a, **kw)
    except B200RLError:
        return True
    return False


def test_cell_kernels_refuse_incomplete_arguments_and_write_nothing():
    from rl_games_b200 import ops
    S, Hd = 40, 16
    gen = torch.Generator().manual_seed(3)
    G = torch.randn(S, 4 * Hd, generator=gen).to(DEV)
    cin = torch.randn(S, Hd, generator=gen).to(DEV)
    done = torch.ones(S, dtype=torch.uint8, device=DEV)
    nan = lambda *s: torch.full(s, NAN, device=DEV)     # noqa: E731
    gates = G.clone()
    c_out, h_out, hn, cn, hsc = nan(S, Hd), nan(S, Hd), nan(S, Hd), nan(S, Hd), nan(S, Hd)
    fwd = [dict(hin_next=hn), dict(cin_next=cn), dict(h_scatter=hsc, scatter_rpc=0), dict(hin_next=hn, cin_next=cn, done_next=done, done_rpc=0)]
    for kw in fwd:
        assert _refused(ops.lstm_cell_fwd, gates, cin, c_out, h_out, S, Hd, **kw), kw
    assert _refused(ops.lstm_cell_fwd, gates, cin, c_out, h_out, 0, Hd)
    dg, dc = nan(S, 4 * Hd), nan(S, Hd)
    dh = torch.randn(S, Hd, device=DEV)
    bwd = [dict(dhin_next=dh), dict(dcin_next=dh), dict(dH=dh, scatter_rpc=0), dict(dhin_next=dh, dcin_next=dh, done_next=done, done_rpc=0)]
    for kw in bwd:
        assert _refused(ops.lstm_cell_bwd, G, cin, cin, dg, dc, S, Hd, **kw), kw
    out = nan(S, Hd)
    assert _refused(ops.rnn_mask_rows, cin, 0, 0, out, S, Hd)
    assert _refused(ops.rnn_mask_rows, cin, S, 0, out, S, Hd, done=done, done_rpc=0)
    torch.cuda.synchronize()
    assert torch.equal(gates, G), 'a refused forward activated the gates'
    for t in (c_out, h_out, hn, cn, hsc, dg, dc, out):
        assert t.isnan().all().item(), 'a refused call wrote an output'


# ----------------------------------------------------------------------------------------------------------- (b) minibatch gradient
def make_agent(cfg_over, N, H, D, A, units, mb, env, init_state, hid, before, layer_norm):
    """tests/test_agent_gpu.py::make_agent with an LSTM (optionally layer-normed) network"""
    from rl_games_b200.runner import Runner
    network = {'name': 'actor_critic', 'separate': False,
               'space': {'continuous': {'mu_activation': 'None', 'sigma_activation': 'None', 'mu_init': {'name': 'default'},
                                        'sigma_init': {'name': 'const_initializer', 'val': 0}, 'fixed_sigma': True}},
               'mlp': {'units': list(units), 'activation': 'elu', 'initializer': {'name': 'default'}},
               'rnn': {'name': 'lstm', 'units': hid, 'layers': 1, 'before_mlp': before, 'layer_norm': layer_norm}}
    config = {'name': 'lstm_grad', 'env_name': 'unused', 'reward_shaper': {'scale_value': 1.0}, 'device': DEV,
              'multi_gpu': False, 'mixed_precision': False, 'normalize_input': True, 'normalize_value': True,
              'value_bootstrap': True, 'normalize_advantage': True, 'gamma': 0.99, 'tau': 0.95, 'learning_rate': 3e-4,
              'lr_schedule': 'adaptive', 'kl_threshold': 0.008, 'grad_norm': 1e-3, 'entropy_coef': 0.01, 'truncate_grads': True,
              'e_clip': 0.2, 'clip_value': True, 'use_smooth_clamp': True, 'bound_loss_type': 'regularisation',
              'bounds_loss_coef': 1e-3, 'max_epochs': 100, 'num_actors': N, 'horizon_length': H, 'minibatch_size': mb,
              'mini_epochs': 1, 'critic_coef': 2, 'print_stats': False, 'train_dir': '/tmp/b200_lstm_grad_runs', 'b200_cuda_graph': False}
    config.update(cfg_over)
    config['env_info'] = env.get_env_info()
    config['vec_env'] = env
    params = {'seed': 7, 'algo': {'name': 'a2c_continuous'}, 'model': {'name': 'continuous_a2c_logstd'}, 'network': network,
              'config': config}
    r = Runner()
    r.load({'params': params})
    r.params['config']['vec_env'] = env
    agent = r.algo_factory.create(r.algo_name, base_name='lstm_grad', params=r.params)
    agent.model.load_state_dict({k: v.to(DEV) for k, v in init_state.items()}, strict=False)
    agent.init_tensors()
    agent._repack()
    agent.obs = agent.env_reset()
    return agent


def _snapshot(agent):
    """what the fp64 reference reads, copied to the host before an update"""
    dn = agent.rnn_dones_buf if agent.rnn_dones_buf is not None else agent.dones_buf
    b = {'obses': agent.obses, 'actions': agent.actions, 'neglogpacs': agent.neglogpacs, 'old_values': agent.old_values_n,
         'returns': agent.returns_n, 'advantages': agent.advs_n, 'valid': agent.valid, 'rnn_h0': agent.rnn_h0, 'rnn_c0': agent.rnn_c0,
         'dones': dn}
    b = {k: (None if v is None else v.cpu().clone()) for k, v in b.items()}
    rms = agent.model.running_mean_std
    stats = None if rms is None else (rms.running_mean.cpu().clone(), rms.running_var.cpu().clone(), rms.count.cpu().clone())
    sd = agent.model.state_dict()
    params = {n: sd[n].cpu().clone() for n in agent.model.param_names()}
    return b, stats, params


def _check_update(agent, i, u, units, before, layer_norm, case, min_done_positions=True):
    m = agent.model
    T, epm = agent.seq_length, agent.envs_per_mb
    b, stats, params = _snapshot(agent)
    if min_done_positions:
        assert GR.window_done_positions(b['dones'], i, epm, T) == list(range(T)), 'a window position without a reset flag'
    # the update merges its own minibatch's obs moments at its start on the first update of an epoch (or on every update without
    # precomputed minibatch moments); later ones were merged by the previous update's optimiser tail, so the snapshot already has them
    merge = agent.normalize_input and (not agent.use_mb_moments or u == 0)
    agent._minibatch_update(i, u)
    torch.cuda.synchronize()
    g = agent._gv[u & 1]['grad'].clone().cpu()
    loss_ref, g_ref = GR.minibatch_loss_and_grads(params, b, i, epm, T, units, agent.config, rnn_before_mlp=before, layer_norm=layer_norm,
                                                  activation=m.activation, obs_stats=stats if agent.normalize_input else None,
                                                  merge_obs_stats=merge, gemm_operands=torch.bfloat16 if agent.gemm_tc else None)
    tol_err, tol_ratio = GRAD_TOL[bool(agent.gemm_tc)]
    total = sum(float(v.double().norm()) ** 2 for v in g_ref.values()) ** 0.5
    assert total > 10 * float(agent.grad_norm), 'the clip would not act: the test could not tell a clipped gradient'
    out = []
    for n, v in zip(m.param_names(), m._param_views(g)):
        err, ratio = GR.grad_errors(v, g_ref[n])
        out.append((n, err, ratio))
        assert err < tol_err and abs(ratio - 1.0) < tol_ratio, (case, i, u, n, err, ratio)
    w = max(out, key=lambda r: max(r[1] / tol_err, abs(r[2] - 1) / tol_ratio))
    print(f'lstm grad {case} mb {i} update {u}: worst {w[0]}; max err {max(r[1] for r in out):.2e} '
          f'max |ratio-1| {max(abs(r[2] - 1) for r in out):.2e}')
    return out


def _grad_case(mp, before, layer_norm, autoreset, hid, T, normalize_input=True, N=64, H=8, D=44, A=5, units=(64, 32), mb=128, seed=0,
               p_done=0.2):
    units = list(units)
    obs_tape, done_tape, tout_tape = O.make_tapes(H + 1, N, D, seed=60 + seed, p_done=p_done)
    if layer_norm:
        params = LO.init_params(D, units, A, seed=seed, rnn_units=hid, rnn_before_mlp=before, ln_seed=seed + 1)
    else:
        params = O.init_params(D, units, A, seed=seed, rnn_units=hid, rnn_before_mlp=before)
    gen = torch.Generator().manual_seed(70 + seed)
    for k in params:           # non-zero biases and log-std
        if k.endswith('bias') or k.endswith('sigma') or 'bias_' in k:
            params[k] = params[k] + torch.randn(params[k].shape, generator=gen) * 0.05
    noise = torch.randn(H, N, A, generator=gen).to(DEV)
    env = TapeEnvGPU(obs_tape, done_tape, tout_tape, A, autoreset)
    agent = make_agent({'mixed_precision': mp, 'seq_length': T, 'normalize_input': normalize_input}, N, H, D, A, units, mb, env, params,
                       hid, before, layer_norm)
    assert agent.is_rnn and not agent.use_tc and agent.gemm_tc == mp and agent.model.rnn_layer_norm == layer_norm
    assert (agent.rnn_dones_buf is not None) == (autoreset == 'next_step')
    agent._rollout(noise)          # a first rollout: the window-initial states of the second are not all zero
    agent._rollout(noise)
    agent._gae_and_prepare()
    agent.set_train()
    return agent, units


def _run_updates(agent, units, before, layer_norm, case):
    """minibatch 0, a middle one and the last one, as updates 0, 1, 2 on the same buffers (the later ones on the scratch of the earlier)"""
    nmb = agent.num_minibatches
    for u, i in enumerate(dict.fromkeys([0, nmb // 2, nmb - 1])):
        _check_update(agent, i, u, units, before, layer_norm, case)


@pytest.mark.parametrize('autoreset', ['same_step', 'next_step'])
@pytest.mark.parametrize('layer_norm', [False, True], ids=['plain', 'layer_norm'])
@pytest.mark.parametrize('before', [True, False], ids=['lstm_before_mlp', 'lstm_after_mlp'])
@pytest.mark.parametrize('mp', [False, True], ids=['fp32', 'gemm_tc'])
def test_minibatch_gradient_matches_fp64(mp, before, layer_norm, autoreset):
    """Hd 33, seq_length 4, horizon 8 (two windows per env), 4 minibatches of 16 envs"""
    agent, units = _grad_case(mp, before, layer_norm, autoreset, hid=33, T=4, seed=1)
    _run_updates(agent, units, before, layer_norm, f'{mp}-{before}-{layer_norm}-{autoreset}')


@pytest.mark.parametrize('T', [1, 4, 8], ids=['seq1', 'seq4', 'seq_horizon'])
@pytest.mark.parametrize('hid', [8, 33, 256])
@pytest.mark.parametrize('mp', [False, True], ids=['fp32', 'gemm_tc'])
def test_minibatch_gradient_matches_fp64_hidden_and_window_sizes(mp, hid, T):
    """LSTM 8 / 33 / 256 units, windows of 1 step, 4 steps and the whole horizon (8); LSTM before the MLP on seq_length 1 and the whole
    horizon, after it on 4"""
    before = T != 4
    agent, units = _grad_case(mp, before, False, 'same_step', hid=hid, T=T, seed=5 + hid)
    _run_updates(agent, units, before, False, f'{mp}-hid{hid}-T{T}')


@pytest.mark.parametrize('mp', [False, True], ids=['fp32', 'gemm_tc'])
def test_minibatch_gradient_matches_fp64_without_input_normalisation(mp):
    agent, units = _grad_case(mp, True, False, 'next_step', hid=33, T=4, normalize_input=False, seed=3)
    assert agent.model.running_mean_std is None
    _run_updates(agent, units, True, False, f'{mp}-no-norm')


@pytest.mark.parametrize('mp', [False, True], ids=['fp32', 'gemm_tc'])
def test_minibatch_gradient_matches_fp64_c4_geometry(mp):
    """BASELINE configs[3] at full width: 8192 envs, obs 348, 17 actions, LSTM 256 before the MLP [512, 256, 128], minibatch 16384,
    seq_length 4 (horizon 8: 4 minibatches of 2048 envs)"""
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    agent, units = _grad_case(mp, True, False, 'same_step', hid=256, T=4, N=8192, H=8, D=348, A=17, units=(512, 256, 128), mb=16384,
                              seed=4)
    _run_updates(agent, units, True, False, f'{mp}-c4')
