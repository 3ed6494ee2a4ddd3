"""Golden runs of the REAL reference DiscreteA2CAgent on action spaces wider than the narrow categorical kernels (Denys88/rl_games at
/root/reference, build container only):

    python tests/golden/gen_golden_cat_wide.py

Two train_epoch()s each, on gen_golden.py's tapes and uniform draws (gen_agent_discrete):
  agent_discrete_wide362.pt   Discrete(362) (Go 19x19), action masks, shared trunk, next_step autoreset
  agent_multidiscrete_wide.pt Tuple of 10 heads [3, 70, 5, 1, 65, 4, 9, 2, 6, 7] (two wider than 64, one of a single action), per-head
                              action masks, separate trunks
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from gen_golden import gen_agent_discrete  # noqa: E402

WIDE_HEADS = [3, 70, 5, 1, 65, 4, 9, 2, 6, 7]

if __name__ == '__main__':
    gen_agent_discrete('agent_discrete_wide362.pt', K=362, D=16, units=(32, 16), separate=False, use_action_masks=True,
                       autoreset='next_step', seed=31)
    gen_agent_discrete('agent_multidiscrete_wide.pt', K=WIDE_HEADS, D=sum(WIDE_HEADS), units=(16, 8), separate=True, use_action_masks=True,
                       seed=33)
