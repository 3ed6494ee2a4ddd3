"""uint8 frame tapes of the conv-trunk golden runs (tests/golden/gen_golden_cnn.py), computed rather than stored: an integer hash of
(seed, t, env, element) in int64 arithmetic, which is the same on every machine and torch version.  The fixtures keep only the small
tapes (dones, time-outs, masks, uniforms) and the recorded results."""
import torch

_M32 = 1 << 32


def _mix(h):
    h = (h ^ (h >> 15)) * 2246822519 % _M32
    h = (h ^ (h >> 13)) * 3266489917 % _M32
    return h ^ (h >> 16)


def frame_tape(T, N, shape, seed):
    """[T, N, *shape] uint8: per-env noise in 0..95 plus a bright 6 x 6 block (in the two spatial axes of the last three, whichever
    layout) that moves with t, so that frames, and the argmax of their first bytes, change from step to step"""
    D = 1
    for s in shape:
        D *= int(s)
    t = torch.arange(T, dtype=torch.int64).view(T, 1, 1)
    n = torch.arange(N, dtype=torch.int64).view(1, N, 1)
    e = torch.arange(D, dtype=torch.int64).view(1, 1, D)
    h = _mix((e * 2654435761 + t * 40503 + n * 9973 + seed * 7919) % _M32)
    frames = (h % 96).to(torch.uint8).view(T, N, *shape)
    side = min(shape[-2], shape[-1]) if shape[0] <= 4 else min(shape[0], shape[1])
    for ti in range(T):
        for ni in range(N):
            r0 = (3 * ti + 5 * ni) % max(1, side - 6)
            if shape[0] <= 4:                       # (C, H, W)
                frames[ti, ni, :, r0:r0 + 6, r0:r0 + 6] = 200
            else:                                   # (H, W, C)
                frames[ti, ni, r0:r0 + 6, r0:r0 + 6, :] = 200
    return frames
