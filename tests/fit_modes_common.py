"""Shared by the joint-fitting tests of the glob_only and expr_only deformation modes (test_fit_modes_cpu.py,
test_gpu_fit_modes.py) and tests/golden/make_golden_fit_joint_modes.py: the seeded deformation networks, the scans, lambdas
and schedule of the golden fit_joint_modes.npz."""
import contextlib
import io

import numpy as np
import torch

from npm_fit_common import LAMBDAS_JOINT, SCHEDULE, STEP_SCALE      # noqa: F401  (fitting_pointclouds.py:253-266)

MODES = ('expr_only', 'glob_only')
N_ITER = 4                        # iterations 0..3 at step_scale 0.01: the lr / lambda events at 2 and the first clamp change
N_OBS, N_POINTS = 3, 300          # the recipe of fit_joint.npz: 3 observations around the head, every point drawn each time
ID_SEED = 3                       # the fixed identity code: sample_latent(3), as in fit_expression.npz
CONDITION_WIDTH = {'compress': 232, 'expr_only': 200, 'glob_only': 264}


def make_deformation(mode, anchors, cls=None, device='cpu'):
    """conftest.make_deformation in ``mode`` (same sizes and seed 10), eval mode (fitting_pointclouds.py:229).  ``cls``: the
    reference's DeformationNetwork, or None for the mirror's."""
    if cls is None:
        from nphm_b200.models.deepSDF import DeformationNetwork as cls
    torch.manual_seed(10)
    with contextlib.redirect_stdout(io.StringIO()):          # the reference's constructor prints its widths
        dfn = cls(mode=mode, lat_dim_expr=200, lat_dim_id=32, lat_dim_glob_shape=64, lat_dim_loc_shape=32, n_loc=39,
                  anchors=anchors, hidden_dim=512, nlayers=6, out_dim=3, input_dim=3)
    dfn.eval()
    return dfn.to(device)


def make_scans(seed=500):
    rng = np.random.RandomState(seed)
    return [(rng.randn(N_POINTS, 3) * 0.1 + np.array([0.0, 0.05, -0.1])).astype(np.float32) for _ in range(N_OBS)]
