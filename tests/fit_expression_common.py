"""Shared by the expression-space fitting tests (test_fit_expression_cpu.py, test_gpu_fit_expression.py) and
tests/golden/make_golden_fit_expression.py: the observations, lambdas and schedule of the golden fit_expression.npz."""
import numpy as np

from npm_fit_common import LAMBDAS_JOINT, SCHEDULE, STEP_SCALE      # noqa: F401  (fitting_pointclouds.py:253-266)

N_ITER = 7                        # iterations 0..6 at step_scale 0.01 cross the lr / lambda events at 2, 4, 5, 6 and both clamp changes
# the NPHM subject's scans have more than 1000 points (each draw subsamples 1000), the NPM subject's fewer (all points are drawn)
NPHM_SCAN_POINTS = (1100, 1300, 1050, 1200)
NPM_SCAN_POINTS = (300, 300, 300)


def make_scans(sizes, seed):
    rng = np.random.RandomState(seed)
    return [(rng.randn(n, 3) * 0.1 + np.array([0.0, 0.05, -0.1])).astype(np.float32) for n in sizes]
