"""Layer-wise MLPs: one GEMM launch per layer, on the fp32 CUDA-core kernels (mlp_simt.cu) or the bf16 tensor-core GEMMs (gemm_tc.cu).

Every layer-wise network of the package -- the continuous agent's trunk when it does not run on the fused kernels, the discrete
agent's trunks with their heads, the central value net, the SAC actor and critics -- runs its forward and backward through
``forward`` / ``backward`` over a list of ``Layer`` records built once with the model.

The first layer reads its input in the arena's chunked row order (``rows_per_chunk`` rows every ``chunk_stride`` rows, row stride
``x_ld``), optionally normalised by ``norm = (mean, std)``; later layers read the dense activations of the layer below.  The backward
writes each layer's weight gradient into the split-partial arena ``part`` at the layer's flat offsets and folds the activation
derivative of the layer below into its input gradient.
"""
import functools
from collections import namedtuple

from . import ops

# W [Nout, K] and b [Nout] views of a flat arena; w_off / b_off: their offsets in it (where the weight gradient goes); act: the
# activation id applied to the layer's output (0 = linear)
Layer = namedtuple('Layer', 'W b w_off b_off act')


def n_splits(M):
    """row splits of a weight-gradient GEMM over M rows: enough CTAs for small layers, few enough partial rows to reduce"""
    return max(1, min(64, M // 256))


class Kernels:
    """The three layer GEMMs of one precision, and the three convolutions of an image trunk: fp32, or the tensor cores with weight
    operands read from a bf16 twin of the fp32 arena, ``bf16_arena = (fp32 arena, bf16 arena)``, in the forward and the data gradient
    (the tensor-core convs need the twin).  The ``ops`` functions are looked up when the set is built, so that a substitute installed on
    ``ops`` before an agent is built is what runs."""

    def __init__(self, tc=False, bf16_arena=None):
        if not tc:
            self.fwd, self.bwd_data, self.bwd_weight = ops.linear_fwd, ops.linear_bwd_data, ops.linear_bwd_weight
            self.conv_fwd, self.conv_bwd_data, self.conv_bwd_weight = ops.conv2d_fwd, ops.conv2d_bwd_data, ops.conv2d_bwd_weight
            return
        self.fwd = functools.partial(ops.linear_fwd_tc, bf16_arena=bf16_arena)
        self.bwd_data = functools.partial(ops.linear_bwd_data_tc, bf16_arena=bf16_arena)
        self.bwd_weight = ops.linear_bwd_weight_tc
        self.conv_fwd = functools.partial(ops.conv2d_fwd_tc, bf16_arena=bf16_arena)
        self.conv_bwd_data = functools.partial(ops.conv2d_bwd_data_tc, bf16_arena=bf16_arena)
        self.conv_bwd_weight = ops.conv2d_bwd_weight_tc


def forward(k, layers, x, acts, M, x_ld, rows_per_chunk=None, chunk_stride=0, norm=(None, None)):
    """acts[l] = act_l(in_l W_l^T + b_l) for M rows: in_0 = x, read as the module docstring says, in_l = acts[l - 1]"""
    first = layers[0]
    k.fwd(x, first.W, first.b, acts[0], first.act, rows_per_chunk=rows_per_chunk, chunk_stride=chunk_stride, x_ld=x_ld,
          norm_mean=norm[0], norm_std=norm[1], M=M)
    for l in range(1, len(layers)):
        k.fwd(acts[l - 1], layers[l].W, layers[l].b, acts[l], layers[l].act, M=M)


def backward(k, layers, x, acts, grads, part, split_stride, n_splits, M, x_ld, rows_per_chunk=None, chunk_stride=0, norm=(None, None),
             dx_out=None, weights=True, dx_act=0):
    """grads[l] = dL/d(pre-activation of layer l); the caller fills grads[-1], the others are overwritten.  Weight gradients go to
    `n_splits` split rows of `part` (row stride `split_stride`) unless weights=False; with dx_out, dL/d(input) goes there, times the
    derivative of activation `dx_act` when the input x is the (dense) output of that activation."""
    for l in range(len(layers) - 1, -1, -1):
        lay = layers[l]
        if weights:
            if l > 0:
                k.bwd_weight(grads[l], acts[l - 1], part[0, lay.w_off:], part[0, lay.b_off:], lay.W.shape[1], lay.W.shape[0], n_splits,
                             M=M, split_stride=split_stride)
            else:
                k.bwd_weight(grads[0], x, part[0, lay.w_off:], part[0, lay.b_off:], lay.W.shape[1], lay.W.shape[0], n_splits,
                             rows_per_chunk=rows_per_chunk, chunk_stride=chunk_stride, x_ld=x_ld, norm_mean=norm[0], norm_std=norm[1], M=M,
                             split_stride=split_stride)
        if l > 0:
            k.bwd_data(grads[l], lay.W, acts[l - 1], grads[l - 1], layers[l - 1].act, M=M)
        elif dx_out is not None:
            k.bwd_data(grads[0], lay.W, x if dx_act else None, dx_out, dx_act, M=M)
