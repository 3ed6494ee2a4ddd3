"""Torch stand-ins for the tensor-core entry points of the discrete agent's ``mixed_precision: True`` path (conv2d_*_tc, linear_*_tc,
cast_bf16) -- TEST INFRASTRUCTURE ONLY, on top of tests/_torch_ops.py and tests/_torch_ops_cnn.py.

They are a kernel-faithful model of conv_tc.cu / gemm_tc.cu: every operand is rounded to bf16 where the kernels stage it (the input
after the 1/255 scaling and the normaliser, dY, the weights READ FROM THE bf16 TWIN, never re-rounded from the fp32 arena), products
are summed in fp64 (the kernels' products are exact in fp32; only their fp32 summation order differs), bias, activation and outputs
are fp32.  Reading the twin means a stale twin shows up as a wrong result.  They run on CPU tensors (host tests) or CUDA tensors (the
reference model of the GPU tests)."""
import torch
import torch.nn.functional as F

import _torch_ops as T
import _torch_ops_cnn as TC


def bf(t):
    """round to bf16 (round to nearest even, like __float2bfloat16_rn), back to fp64"""
    return t.float().to(torch.bfloat16).double()


def twin(W, bf16_arena):
    """W's bf16 twin (a view of the twin arena at W's offset) as fp64"""
    flat, fb = bf16_arena
    off = (W.data_ptr() - flat.data_ptr()) // 4
    assert 0 <= off < flat.numel() and W.is_contiguous(), 'the tensor-core entry points read the weights from the bf16 twin'
    return fb[off:off + W.numel()].view(W.shape).double()


def _input(X, geo, M, nhwc, rows_per_chunk, chunk_stride, x_ld, norm_mean, norm_std):
    """tests/_torch_ops_cnn.py's reading of the conv input, with the kernels' correctly rounded fp32 divisions (x / 255 and the
    normaliser's division; a division in fp64 rounded once to fp32 is that): torch on a CUDA tensor divides by a scalar through its
    reciprocal, which is 1 ulp off for some bytes, and a bf16 rounding of that byte value then differs everywhere it occurs"""
    C, H, W, _, _ = geo
    D = C * H * W
    x = T._rows(X, M, D, rows_per_chunk, chunk_stride, D if x_ld is None else x_ld)
    x = (x.double() / 255.0).float() if x.dtype == torch.uint8 else x
    if norm_mean is not None:
        x = torch.clamp(((x - norm_mean).double() / norm_std.double()).float(), -5.0, 5.0)
    return x.view(M, H, W, C).permute(0, 3, 1, 2) if nhwc else x.view(M, C, H, W)


def _norm(x, mean, std):
    return x if mean is None else torch.clamp(((x - mean).double() / std.double()).float(), -5.0, 5.0)


def cast_bf16(src, dst):
    dst.copy_(src.to(torch.bfloat16))


def conv2d_fwd_tc(X, W, b, Y, geo, act, M, nhwc=False, rows_per_chunk=None, chunk_stride=0, x_ld=None, norm_mean=None, norm_std=None,
                  bf16_arena=None):
    x = bf(_input(X, geo, M, nhwc, rows_per_chunk, chunk_stride, x_ld, norm_mean, norm_std))
    pre = F.conv2d(x, twin(W, bf16_arena), None, stride=geo[3], padding=geo[4]).float()
    Y[:M] = T.ACT[act](pre + b.view(1, -1, 1, 1))


def conv2d_bwd_data_tc(dY, W, A_prev, dX, geo, act_prev, M, bf16_arena=None):
    C, H, Wd, st, pad = geo
    g = torch.nn.grad.conv2d_input((M, C, H, Wd), twin(W, bf16_arena), bf(dY[:M]), stride=st, padding=pad).float()
    dX[:M] = g if A_prev is None else g * T._act_grad_from_out(A_prev[:M], act_prev)


def conv2d_bwd_weight_tc(dY, X, dW_part, db_part, W_shape, geo, n_splits, M, split_stride, nhwc=False, rows_per_chunk=None, chunk_stride=0,
                         x_ld=None, norm_mean=None, norm_std=None):
    x = bf(_input(X, geo, M, nhwc, rows_per_chunk, chunk_stride, x_ld, norm_mean, norm_std))
    dy = bf(dY[:M])
    dW = torch.nn.grad.conv2d_weight(x, tuple(W_shape), dy, stride=geo[3], padding=geo[4]).float()
    db = dy.sum((0, 2, 3)).float()
    n, Cout = dW.numel(), W_shape[0]
    fw, fb = T._flat(dW_part), T._flat(db_part)
    for s in range(n_splits):          # the sum over the splits is what matters: all of it in split 0
        fw[s * split_stride:s * split_stride + n] = dW.reshape(-1) if s == 0 else 0.0
        fb[s * split_stride:s * split_stride + Cout] = db if s == 0 else 0.0


def linear_fwd_tc(X, W, b, Y, act, rows_per_chunk=None, chunk_stride=0, x_ld=None, norm_mean=None, norm_std=None, M=None, accumulate=False,
                  bf16_arena=None):
    Nout, K = W.shape
    M = Y.shape[0] if M is None else M
    x = bf(_norm(T._rows(X, M, K, rows_per_chunk, chunk_stride, K if x_ld is None else x_ld), norm_mean, norm_std))
    y = (x @ twin(W, bf16_arena).t()).float() + b
    if accumulate:
        y = y + Y[:M]
    Y[:M] = T.ACT[act](y)


def linear_bwd_data_tc(dY, W, A_prev, dX, act_prev, M=None, bf16_arena=None):
    M = dY.shape[0] if M is None else M
    g = (bf(dY[:M]) @ twin(W, bf16_arena)).float()
    dX[:M] = g if A_prev is None else g * T._act_grad_from_out(A_prev[:M], act_prev)


def linear_bwd_weight_tc(dY, X, dW_part, db_part, K, Nout, n_splits, rows_per_chunk=None, chunk_stride=0, x_ld=None, norm_mean=None,
                         norm_std=None, M=None, split_stride=None):
    M = dY.shape[0] if M is None else M
    x = bf(_norm(T._rows(X, M, K, rows_per_chunk, chunk_stride, K if x_ld is None else x_ld), norm_mean, norm_std))
    dy = bf(dY[:M])
    dW, db = (dy.t() @ x).float(), dy.sum(0).float()
    split_stride = dW_part.stride(0) if split_stride is None else split_stride
    fw, fb = T._flat(dW_part), T._flat(db_part)
    for s in range(n_splits):
        fw[s * split_stride:s * split_stride + Nout * K] = dW.reshape(-1) if s == 0 else 0.0
        fb[s * split_stride:s * split_stride + Nout] = db if s == 0 else 0.0


TC_OPS = ('conv2d_fwd_tc', 'conv2d_bwd_data_tc', 'conv2d_bwd_weight_tc', 'linear_fwd_tc', 'linear_bwd_data_tc', 'linear_bwd_weight_tc',
          'cast_bf16')


def install_tc_only(monkeypatch):
    """the tensor-core entry points and the twin refresh only (the rest of ``ops`` untouched: real kernels on a GPU)"""
    from rl_games_b200 import ops
    for name in TC_OPS:
        monkeypatch.setattr(ops, name, globals()[name])


def install_conv_tc(monkeypatch):
    """every op of the discrete agent, conv trunk and tensor-core path included, on torch"""
    TC.install_cnn(monkeypatch)
    install_tc_only(monkeypatch)
