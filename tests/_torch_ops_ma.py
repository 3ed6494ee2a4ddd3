"""Torch (CPU) stand-ins for ``ops.post_step_ma``, ``ops.cv_value_broadcast`` and ``ops.cv_gather_agent0`` -- TEST INFRASTRUCTURE
ONLY, in the style of ``tests/_torch_ops.py``.  They restate the multi-agent kernels' contracts (the reference's dones.nonzero()[::agents]
selection, a2c_common.py:1039-1051; the central value's env-row to agent-row mapping, central_value.py:224-244) so that the agents' host
logic runs against the multi-agent golden runs without a GPU.  They prove nothing about the kernels themselves (tests/test_multiagent_gpu.py
checks those against torch on the device)."""
import torch


def post_step_ma(rewards, dones, time_outs, values_t, valid_t, rewards_out_t, dones_cur, prev_dones, ep_state, meter, games_to_track,
                 bufs, N, agents, cfg):
    r = rewards.float()
    sh = torch.clamp((r + cfg.shift_value) * cfg.scale_value, cfg.min_val, cfg.max_val)
    if cfg.log_val:
        sh = torch.log(sh)
    if cfg.value_bootstrap and time_outs is not None:
        sh = sh + cfg.gamma * values_t * time_outs.float()
    rewards_out_t.copy_(sh)
    live = torch.ones(N) if valid_t is None else valid_t
    cr, cs, cl = ep_state[0] + r * live, ep_state[1] + sh * live, ep_state[2] + live
    d = dones.float()
    sel = (d != 0).nonzero().reshape(-1)[::agents]
    n = int(sel.numel())
    if n > 0:          # AverageMeter.update (torch_ext.py:333-342) over the selected rows
        size = min(n, games_to_track)
        old = min(games_to_track - size, float(meter[3]))
        tot = old + size
        for slot, x in ((0, cr), (1, cs), (2, cl)):
            meter[slot] = (float(meter[slot]) * old + float(x[sel].double().mean()) * size) / tot
        meter[3] = tot
        meter[4] += n
    nd = 1.0 - d
    ep_state[0], ep_state[1], ep_state[2] = cr * nd, cs * nd, cl * nd
    dones_cur.copy_((d != 0).to(torch.uint8))
    if prev_dones is not None:
        prev_dones.copy_(d)
    bufs[3][:n] = sel
    bufs[4][0] = n


def cv_value_broadcast(val, vms_mean, vms_var, normalize_value, out, N, agents):
    v = val.reshape(-1)[:N]
    if normalize_value:
        v = torch.sqrt(vms_var.float() + 1e-5) * torch.clamp(v, -5.0, 5.0) + vms_mean.float()
    out.copy_(v.repeat_interleave(agents))


def cv_gather_agent0(src_a, src_b, dst_a, dst_b, H, N, agents):
    dst_a.copy_(src_a.reshape(H, N, agents)[:, :, 0])
    dst_b.copy_(src_b.reshape(H, N, agents)[:, :, 0])


def install(monkeypatch):
    from rl_games_b200 import ops
    for name in ('post_step_ma', 'cv_value_broadcast', 'cv_gather_agent0'):
        monkeypatch.setattr(ops, name, globals()[name])
