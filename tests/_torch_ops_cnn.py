"""Torch (CPU) stand-ins for the conv trunk's entry points (conv2d_fwd, conv2d_bwd_data, conv2d_bwd_weight, moments_update_u8) -- TEST
INFRASTRUCTURE ONLY, in addition to tests/_torch_ops.py (whose stand-ins are used unchanged for everything else).  They restate each
kernel's contract on torch's F.conv2d and its autograd: arena rows through (rows_per_chunk, chunk_stride), uint8 frames / 255, NHWC or
NCHW rows, the normaliser over the env's own layout, split partials at the layer's flat offsets."""
import torch
import torch.nn.functional as F

import _torch_ops as T


def _input(X, geo, M, nhwc, rows_per_chunk, chunk_stride, x_ld, norm_mean, norm_std):
    """the conv input [M, C, H, W] as the kernel reads it"""
    C, H, W, _, _ = geo
    D = C * H * W
    x = T._rows(X, M, D, rows_per_chunk, chunk_stride, D if x_ld is None else x_ld)
    x = x.float() / 255.0 if x.dtype == torch.uint8 else x
    x = T._norm(x, norm_mean, norm_std)
    return x.view(M, H, W, C).permute(0, 3, 1, 2) if nhwc else x.view(M, C, H, W)


def conv2d_fwd(X, W, b, Y, geo, act, M, nhwc=False, rows_per_chunk=None, chunk_stride=0, x_ld=None, norm_mean=None, norm_std=None):
    x = _input(X, geo, M, nhwc, rows_per_chunk, chunk_stride, x_ld, norm_mean, norm_std)
    Y[:M] = T.ACT[act](F.conv2d(x, W, b, stride=geo[3], padding=geo[4]))


def conv2d_bwd_data(dY, W, A_prev, dX, geo, act_prev, M):
    C, H, Wd, st, pad = geo
    g = torch.nn.grad.conv2d_input((M, C, H, Wd), W, dY[:M], stride=st, padding=pad)
    dX[:M] = g if A_prev is None else g * T._act_grad_from_out(A_prev[:M], act_prev)


def conv2d_bwd_weight(dY, X, dW_part, db_part, W_shape, geo, n_splits, M, split_stride, nhwc=False, rows_per_chunk=None, chunk_stride=0,
                      x_ld=None, norm_mean=None, norm_std=None):
    x = _input(X, geo, M, nhwc, rows_per_chunk, chunk_stride, x_ld, norm_mean, norm_std)
    dW = torch.nn.grad.conv2d_weight(x, tuple(W_shape), dY[:M], stride=geo[3], padding=geo[4])
    db = dY[:M].sum((0, 2, 3))
    n, Cout = dW.numel(), W_shape[0]
    fw, fb = T._flat(dW_part), T._flat(db_part)
    for s in range(n_splits):          # the kernel spreads the rows over the splits; the sum is what matters: all of it in split 0
        fw[s * split_stride:s * split_stride + n] = dW.reshape(-1) if s == 0 else 0.0
        fb[s * split_stride:s * split_stride + Cout] = db if s == 0 else 0.0


def moments_update_u8(x, D, rows_per_chunk, n_chunks, chunk_stride, mean, var, count, mean_f32, std_f32, eps=1e-5):
    n = rows_per_chunk * n_chunks
    rows = T._rows(x, n, D, rows_per_chunk, chunk_stride, D).float() / 255.0
    T.moments_update(rows, D, n, 1, 0, mean, var, count, mean_f32, std_f32, None, None, eps)


def install_cnn(monkeypatch):
    """_torch_ops.install plus the conv trunk's stand-ins"""
    from rl_games_b200 import ops
    T.install(monkeypatch)
    for name in ('conv2d_fwd', 'conv2d_bwd_data', 'conv2d_bwd_weight', 'moments_update_u8'):
        monkeypatch.setattr(ops, name, globals()[name])
