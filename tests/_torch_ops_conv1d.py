"""Torch (CPU) stand-ins for the conv1d trunk's entry points (conv1d_fwd, conv1d_bwd_data, conv1d_bwd_weight) -- TEST INFRASTRUCTURE
ONLY, in addition to tests/_torch_ops.py (whose stand-ins are used unchanged for everything else).  They restate each kernel's contract
on torch's F.conv1d and its autograd: arena rows through (rows_per_chunk, chunk_stride), fp32 [C, L] rows, the normaliser over the flat
observation, split partials at the layer's flat offsets (all of the sum in split 0, the others zero)."""
import torch
import torch.nn.functional as F

import _torch_ops as T


def _input(X, geo, M, rows_per_chunk, chunk_stride, x_ld, norm_mean, norm_std):
    C, L, _, _ = geo
    x = T._rows(X, M, C * L, rows_per_chunk, chunk_stride, C * L if x_ld is None else x_ld)
    return T._norm(x, norm_mean, norm_std).view(M, C, L)


def conv1d_fwd(X, W, b, Y, geo, act, M, rows_per_chunk=None, chunk_stride=0, x_ld=None, norm_mean=None, norm_std=None):
    x = _input(X, geo, M, rows_per_chunk, chunk_stride, x_ld, norm_mean, norm_std)
    Y[:M] = T.ACT[act](F.conv1d(x, W, b, stride=geo[2], padding=geo[3]))


def conv1d_bwd_data(dY, W, A_prev, dX, geo, act_prev, M):
    C, L, st, pad = geo
    g = torch.nn.grad.conv1d_input((M, C, L), W, dY[:M], stride=st, padding=pad)
    dX[:M] = g if A_prev is None else g * T._act_grad_from_out(A_prev[:M], act_prev)


def conv1d_bwd_weight(dY, X, dW_part, db_part, W_shape, geo, n_splits, M, split_stride, rows_per_chunk=None, chunk_stride=0, x_ld=None,
                      norm_mean=None, norm_std=None):
    x = _input(X, geo, M, rows_per_chunk, chunk_stride, x_ld, norm_mean, norm_std)
    dW = torch.nn.grad.conv1d_weight(x, tuple(W_shape), dY[:M], stride=geo[2], padding=geo[3])
    db = dY[:M].sum((0, 2))
    n, Cout = dW.numel(), W_shape[0]
    fw, fb = T._flat(dW_part), T._flat(db_part)
    for s in range(n_splits):
        fw[s * split_stride:s * split_stride + n] = dW.reshape(-1) if s == 0 else 0.0
        fb[s * split_stride:s * split_stride + Cout] = db if s == 0 else 0.0


def install_conv1d(monkeypatch):
    """_torch_ops.install, the multi-agent post-step's stand-ins and the conv1d trunk's"""
    import _torch_ops_ma
    from rl_games_b200 import ops
    T.install(monkeypatch)
    _torch_ops_ma.install(monkeypatch)
    for name in ('conv1d_fwd', 'conv1d_bwd_data', 'conv1d_bwd_weight'):
        monkeypatch.setattr(ops, name, globals()[name])
