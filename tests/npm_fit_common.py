"""Shared by the NPM fitting tests (test_fit_npm_cpu.py, test_gpu_fit_npm.py) and tests/golden/make_golden_fit_npm.py: the
seeded NPM-sized decoders, scans, lambdas and schedule of the golden fit_npm.npz."""
import contextlib
import io

import numpy as np
import torch

from shape_common import state_dict_sha256        # noqa: F401  (re-exported for the golden script and the tests)

# scripts/fitting/fitting_pointclouds.py:253-266 (the identity fit takes the same dict without reg_expr, which its loss lacks)
LAMBDAS_JOINT = {'surface': 2.0, 'reg_expr': 0.01, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
LAMBDAS_IDENTITY = {k: v for k, v in LAMBDAS_JOINT.items() if k != 'reg_expr'}
SCHEDULE = {'lr': {200: 2, 400: 2, 600: 2, 800: 2}, 'symm_dist': {200: 10, 500: 9999}, 'reg_glob': {200: 3, 600: 10},
            'reg_loc': {500: 3, 600: 10}, 'reg_expr': {600: 10}}
STEP_SCALE = 0.01                 # iteration j stands for reference iteration 100 j: the lr / lambda / clamp events at j = 2 .. 8
N_ITER_IDENTITY = 10
N_ITER_JOINT = 7
# random weights make a useless deformation field: the expression decoder's output layer is scaled down (as tools/bench_joint.py
# does for the NPHM deformation network) so that most Broyden searches converge
EXPR_OUT_SCALE = 0.02
# the identity decoder at initialisation is nearly constant over the scans (s = -0.3995 +- 3e-4: eight random layers wash the
# point out), which would leave ~1 % of the points within the native value pass's ~5e-6 of zero, where the sign of their
# gradient is not resolved.  Its xyz input columns are scaled by XYZ_GAIN, which spreads s over the scans like a trained SDF's
# (std 0.05), and its output bias is raised by SURFACE_SHIFT, so that the zero level set passes through them; the clamps
# 0.1 / 0.05 / 0.0075 of the schedule then keep different sets.
XYZ_GAIN = 3000.0
SURFACE_SHIFT = 0.342


def make_decoders(shape_cls, device='cpu'):
    """The NPM baseline of fitting_npm.yaml: identity DeepSDF(512, 1024) (515 -> 1024 x 8 -> 1, geometric init, seed 12 as in
    train_shape.npz) and expression DeepSDF(512 + 200, 1024, out_dim=3) (seed 21, fitting_pointclouds.py:121-123) with its output
    layer scaled by EXPR_OUT_SCALE; the identity decoder's xyz columns are scaled by XYZ_GAIN and its output bias raised by SURFACE_SHIFT.
    ``shape_cls``: the reference's DeepSDF or the mirror."""
    with contextlib.redirect_stdout(io.StringIO()):          # the reference's constructor prints its widths
        torch.manual_seed(12)
        dec = shape_cls(lat_dim=512, hidden_dim=1024, nlayers=8, geometric_init=True)
        torch.manual_seed(21)
        expr = shape_cls(lat_dim=512 + 200, hidden_dim=1024, out_dim=3)
    with torch.no_grad():
        dec.lin0.weight[:, :3].mul_(XYZ_GAIN)
        dec.lin8.bias.add_(SURFACE_SHIFT)
        expr.lin8.weight.mul_(EXPR_OUT_SCALE)
        expr.lin8.bias.mul_(EXPR_OUT_SCALE)
    return dec.to(device).train(), expr.to(device).eval()


def make_scans(n_obs=3, n_points=200, seed=300):
    rng = np.random.RandomState(seed)
    return [(rng.randn(n_points, 3) * 0.1 + np.array([0.0, 0.05, -0.1])).astype(np.float32) for _ in range(n_obs)]
