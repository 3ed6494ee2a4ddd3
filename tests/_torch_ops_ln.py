"""Torch (CPU) stand-ins for the layer-normed LSTM cell entry points (lstm_cell_ln_fwd, lstm_cell_ln_bwd) -- TEST INFRASTRUCTURE ONLY,
in addition to tests/_torch_ops.py (whose stand-ins are used unchanged for everything else).  The LayerNorm is torch's
(F.layer_norm, eps 1e-5); its backward comes from autograd, the cell halves from _torch_ops.lstm_cell_fwd / lstm_cell_bwd."""
import torch
import torch.nn.functional as F

import _torch_ops as T

EPS = 1e-5


def _scatter_rows(S, rpc, stride):
    s = torch.arange(S)
    return (s // rpc) * stride + s % rpc


def lstm_cell_ln_fwd(gates, cin, c_out, h_out, ln_w, ln_b, S, Hd, y_out=None, y_scatter=None, scatter_rpc=0, scatter_stride=0, hin_next=None,
                     cin_next=None, done_next=None, done_rpc=0, done_stride=0, mean=None, rstd=None):
    T.lstm_cell_fwd(gates, cin, c_out, h_out, S, Hd, hin_next=hin_next, cin_next=cin_next, done_next=done_next, done_rpc=done_rpc,
                    done_stride=done_stride)
    h = h_out[:S]
    mu = h.mean(1)
    r = 1.0 / torch.sqrt(((h - mu.unsqueeze(1)) ** 2).mean(1) + EPS)
    y = F.layer_norm(h, (Hd,), ln_w, ln_b, EPS)
    if y_out is not None:
        y_out[:S] = y
    if y_scatter is not None:
        rows = _scatter_rows(S, scatter_rpc, scatter_stride)
        T._flat(y_scatter)[rows.unsqueeze(1) * Hd + torch.arange(Hd).unsqueeze(0)] = y
    if mean is not None:
        mean[:S] = mu
        rstd[:S] = r


def lstm_cell_ln_bwd(gates_act, c_t, cin, dY, ln_w, mean, rstd, dgamma_part, dbeta_part, n_splits, dgates, dcin, S, Hd, scatter_rpc=0,
                     scatter_stride=0, dhin_next=None, dcin_next=None, done_next=None, done_rpc=0, done_stride=0, split_stride=0):
    rows = _scatter_rows(S, scatter_rpc, scatter_stride) if scatter_rpc > 0 else torch.arange(S)
    dy = T._flat(dY)[rows.unsqueeze(1) * Hd + torch.arange(Hd).unsqueeze(0)]
    h = (gates_act[:S, 3 * Hd:] * torch.tanh(c_t[:S])).requires_grad_(True)
    w = ln_w.detach().clone().requires_grad_(True)
    b = torch.zeros(Hd, requires_grad=True)
    F.layer_norm(h, (Hd,), w, b, EPS).backward(dy)
    T.lstm_cell_bwd(gates_act, c_t, cin, dgates, dcin, S, Hd, dH=h.grad, scatter_rpc=S, scatter_stride=0, dhin_next=dhin_next,
                    dcin_next=dcin_next, done_next=done_next, done_rpc=done_rpc, done_stride=done_stride)
    fw, fb = T._flat(dgamma_part), T._flat(dbeta_part)
    for s in range(n_splits):          # the kernel spreads the rows over the splits; the sum is what matters: all of it in split 0
        fw[s * split_stride:s * split_stride + Hd] = w.grad if s == 0 else 0.0
        fb[s * split_stride:s * split_stride + Hd] = b.grad if s == 0 else 0.0


def install_ln(monkeypatch):
    """_torch_ops.install_continuous plus the layer-normed LSTM cell stand-ins"""
    from rl_games_b200 import ops
    T.install_continuous(monkeypatch)
    monkeypatch.setattr(ops, 'lstm_cell_ln_fwd', lstm_cell_ln_fwd)
    monkeypatch.setattr(ops, 'lstm_cell_ln_bwd', lstm_cell_ln_bwd)
