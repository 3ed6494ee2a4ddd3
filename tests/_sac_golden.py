"""Shared by the SAC tests: build the B200 SACAgent for a golden fixture (tests/golden/sac_*.pt), replay the reference's tapes through it
and compare what it ends with against the reference's checkpoint.  TEST INFRASTRUCTURE ONLY."""
import copy
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, 'golden')
sys.path.insert(0, GOLDEN)
sys.path.insert(0, os.path.join(GOLDEN, '_stubs'))       # gymnasium spaces for the tape env
FIXTURES = ('sac_box_norm_same_step', 'sac_fixed_alpha_next_step')


def load(name):
    return torch.load(os.path.join(GOLDEN, name + '.pt'), weights_only=False)


def make_agent(g, device, tmp_path, over=None):
    from gen_golden_sac import SACTapeEnv
    from rl_games_b200.runner import Runner
    e = g['env']
    env = SACTapeEnv(e['obs'], e['rew'], e['done'], e['tout'], g['low'], g['high'], g['autoreset'], e['final'])
    config = copy.deepcopy(g['params'])
    config.update({'device': device, 'train_dir': str(tmp_path), 'env_info': env.get_env_info(), 'b200_cuda_graph': False})
    config.update(over or {})
    r = Runner()
    r.load({'params': {'seed': 11, 'algo': {'name': 'sac'}, 'model': {'name': 'soft_actor_critic'}, 'network': copy.deepcopy(g['network']),
                       'config': config}})
    r.params['config']['vec_env'] = env
    a = r.algo_factory.create('sac', base_name='golden', params=r.params)
    a.set_weights({k: g['init'][k] for k in ('actor', 'critic', 'critic_target')})
    a.model.log_alpha.copy_(g['init']['log_alpha'].reshape(1))
    return a


def run(a, g, use_tapes=True):
    if use_tapes:
        a.tapes = {k: iter(v) for k, v in g['tapes'].items()}
    a.init_tensors()
    a.obs = a.env_reset()
    rows = []
    for _ in range(g['epochs']):
        a.epoch_num += 1
        _, _, _, _, n_upd, actor_rows = a.train_epoch()
        st = a.stats[:n_upd].cpu()
        for i in range(n_upd):
            rows.append((st[i].clone(), i in actor_rows))
    a.frame = g['epochs'] * a.num_frames_per_epoch
    return rows


def compare(a, g, rows, rtol, atol):
    """per-update losses, the final weights / target weights / Adam states / log_alpha / replay buffer against the reference"""
    ref = g['losses']
    assert len(rows) == len(ref)
    learn = g['params']['learnable_temperature']
    for (st, actor), r in zip(rows, ref):
        torch.testing.assert_close(st[1], torch.tensor(r['c1']), rtol=rtol, atol=atol)
        torch.testing.assert_close(st[2], torch.tensor(r['c2']), rtol=rtol, atol=atol)
        assert actor == ('a_loss' in r)
        if actor:
            torch.testing.assert_close(st[3], torch.tensor(r['a_loss']), rtol=rtol, atol=atol)
            torch.testing.assert_close(st[4], torch.tensor(r['entropy']), rtol=rtol, atol=atol)
            if learn:
                torch.testing.assert_close(st[6], torch.tensor(r['alpha_loss']), rtol=rtol, atol=atol)
                torch.testing.assert_close(st[5], torch.tensor(r['alpha']), rtol=rtol, atol=atol)
    s, mine = g['state'], a.get_full_state_weights()
    assert set(s) == set(mine) - {'env_state'}, (sorted(s), sorted(mine))        # the fixture drops the tape env's None state
    for part in ('actor', 'critic', 'critic_target'):
        assert list(s[part]) == list(mine[part])
        for k in s[part]:
            torch.testing.assert_close(mine[part][k].cpu(), s[part][k], rtol=rtol, atol=atol, msg=f'{part}.{k}')
    for opt in ('actor_optimizer', 'critic_optimizer', 'log_alpha_optimizer'):
        so, mo = s[opt], mine[opt]
        assert sorted(so['state']) == sorted(mo['state']), opt
        assert so['param_groups'][0]['params'] == mo['param_groups'][0]['params']
        for i in so['state']:
            assert float(so['state'][i]['step']) == float(mo['state'][i]['step'])
            for k in ('exp_avg', 'exp_avg_sq'):
                torch.testing.assert_close(mo['state'][i][k].cpu().reshape(so['state'][i][k].shape), so['state'][i][k], rtol=rtol, atol=atol,
                                           msg=f'{opt}[{i}].{k}')
    torch.testing.assert_close(mine['log_alpha'].cpu(), s['log_alpha'], rtol=rtol, atol=atol)
    assert mine['epoch'] == s['epoch'] and mine['frame'] == s['frame']
    rb, mrb = s['replay_buffer'], mine['replay_buffer']
    assert rb['idx'] == mrb['idx'] and rb['full'] == mrb['full']
    for k in ('obses', 'next_obses', 'actions', 'rewards', 'dones', 'truncated'):
        if rb[k].dtype == torch.bool:
            assert torch.equal(mrb[k].cpu(), rb[k]), k
        else:
            torch.testing.assert_close(mrb[k].cpu(), rb[k], rtol=rtol, atol=atol, msg=k)
    if 'running_mean_std' in s:
        for k, v in s['running_mean_std'].items():
            torch.testing.assert_close(mine['running_mean_std'][k].cpu().to(v.dtype).reshape(v.shape), v, rtol=1e-6, atol=1e-6)
    size, mr, ml = a.game_stats()
    rs, rr, rl = g['meters'][-1]
    assert size == rs
    np.testing.assert_allclose([mr, ml], [rr, rl], rtol=1e-5, atol=1e-5)
