"""Torch (CPU) stand-in for the players' one new C-ABI op, ``ops.categorical_argmax`` (csrc/player.cu) -- TEST INFRASTRUCTURE ONLY.

It restates the kernel's contract (per-head argmax of the allowed logits, ties to the lowest index, an all-masked head plays 0) so that
the players' host logic runs on the CPU together with the other stand-ins (tests/_torch_ops.py, _torch_ops_cnn.py, _torch_ops_sac.py).
It proves nothing about the kernel, which tests/test_players_gpu.py compares with torch.argmax on the GPU.
"""
import torch

import _torch_ops as T


def categorical_argmax(logits, ld, K, action_masks, actions_out, N, head_sizes=None):
    z = T._flat(logits)[(torch.arange(N) * ld).unsqueeze(1) + torch.arange(K).unsqueeze(0)]
    sizes = list(head_sizes) if head_sizes else [K]
    allowed = torch.ones(N, K, dtype=torch.bool) if action_masks is None else action_masks[:N].reshape(N, K).bool()
    out, off = [], 0
    for k in sizes:
        zj, mj = z[:, off:off + k], allowed[:, off:off + k]
        a = torch.where(mj, zj, torch.full_like(zj, -float('inf'))).argmax(dim=1)
        out.append(torch.where(mj.any(dim=1), a, torch.zeros_like(a)))
        off += k
    actions_out[:N] = torch.stack(out, dim=1).reshape(actions_out[:N].shape)


def install(monkeypatch):
    """the stand-ins of everything the three players call (fp32 kernels, no CUDA graph)"""
    import _torch_ops_cnn as C
    import _torch_ops_sac as S
    from rl_games_b200 import ops
    T.install_continuous(monkeypatch)
    C.install_cnn(monkeypatch)
    for name in ('sac_squash_fwd', 'sac_uniform_actions'):
        monkeypatch.setattr(ops, name, getattr(S, name))
    monkeypatch.setattr(ops, 'categorical_argmax', categorical_argmax)
