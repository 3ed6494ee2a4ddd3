"""Golden runs of the REAL reference with a state-dependent sigma head (fixed_sigma: False, network_builder.py:324-348, :441-444) and
the sigma parametrisations of models.py apply_sigma_parametrization.  Same recipe as gen_golden.py (whose gen_agent it calls):

    python tests/golden/gen_golden_sdsigma.py

writes tests/golden/agent_sdsigma.pt, agent_sdsigma_softplus.pt and agent_fixedsigma_{softplus,bounds}.pt (committed).  Kept as a
script of its own next to gen_golden.py, whose groups it leaves unchanged: regenerate these fixtures with this script."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from gen_golden import gen_agent  # noqa: E402


def gen_sdsigma():
    # 'exp' head initialised like any Linear (sigma_init: default), so every row has its own std from step 0; an entropy bonus (its
    # gradient flows through the sigma head into the trunk) and a bound loss on top
    gen_agent('agent_sdsigma.pt', N=8, H=8, D=8, A=3, units=(16, 12, 8), mb=32, seed=26,
              space_over={'fixed_sigma': False, 'sigma_init': {'name': 'default'}},
              overrides={'entropy_coef': 0.01, 'bounds_loss_coef': 0.001, 'bound_loss_type': 'bound', 'mini_epochs': 3})
    # configs/mjlab/ppo_wujihand_reorient.yaml's head: softplus, min_sigma 0.2, const bias -1.05; next_step autoreset (masked rows)
    gen_agent('agent_sdsigma_softplus.pt', N=8, H=8, D=8, A=4, units=(16, 12, 8), mb=32, seed=27, autoreset='next_step',
              space_over={'fixed_sigma': False, 'sigma_parametrization': 'softplus', 'min_sigma': 0.2,
                          'sigma_init': {'name': 'const_initializer', 'val': -1.05}},
              overrides={'entropy_coef': 0.005, 'use_smooth_clamp': False, 'learning_rate': 1e-3, 'kl_threshold': 0.01})

    # fixed sigma in the parametrisations that are mapped outside the kernels (model.py refresh_sigma_floor): softplus with a floor and
    # an entropy bonus; exp clamped to logstd_bounds whose upper bound the perturbed raw sigma straddles (zero gradient above it)
    gen_agent('agent_fixedsigma_softplus.pt', N=8, H=8, D=8, A=3, units=(16, 12, 8), mb=32, seed=28,
              space_over={'sigma_parametrization': 'softplus', 'min_sigma': 0.1}, overrides={'entropy_coef': 0.01, 'mini_epochs': 3})
    gen_agent('agent_fixedsigma_bounds.pt', N=8, H=8, D=8, A=4, units=(16, 12, 8), mb=32, seed=29, autoreset='next_step',
              space_over={'logstd_bounds': [-1.0, 0.0]}, overrides={'entropy_coef': 0.01, 'learning_rate': 1e-3})


if __name__ == '__main__':
    gen_sdsigma()
