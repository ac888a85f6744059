"""The pose contract of the fitters (DESIGN.md §4.24) in float64 on the CPU: the closed-form pose gradient against autograd,
the retraction, the rigid mode, argument checks, and frozen poses leaving the composite fitters' results bit for bit."""
import numpy as np
import pytest
import torch

from conftest import make_deformation, make_ensemble, make_npm
from pose_common import autograd_pose_grad, random_poses, random_rows
from nphm_b200.models import fitting as F
from nphm_b200.models.pose import ObservationPoses, apply_f64, compose_f64, grad_f64, rodrigues_f64


def test_closed_form_gradient_matches_autograd():
    poses = random_poses(4, seed=1)
    pts, rows, g = random_rows(9, 50, 4, seed=2)
    want, q = autograd_pose_grad(poses.table, pts.double(), g, rows, 2.5)
    got = grad_f64(poses.table, q, g, rows, 2.5)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-15), (got - want).abs().max()


def test_tangent_composition_gives_the_contract_gradient_and_the_applied_points():
    poses = random_poses(3, seed=3)
    pts, rows, g = random_rows(6, 40, 3, seed=4)
    xi = torch.zeros(3, 7, dtype=torch.float64, requires_grad=True)
    q = compose_f64(poses.table, pts.double(), rows, xi)
    (2.0 * (q * g.double()).sum()).backward()
    assert torch.allclose(xi.grad, grad_f64(poses.table, q.detach(), g, rows, 2.0), rtol=1e-12, atol=1e-15)
    assert torch.equal(compose_f64(poses.table, pts, rows, xi.detach()), apply_f64(poses.table, pts, rows))


def test_identity_maps_points_to_themselves_and_padding_passes_through():
    poses = ObservationPoses(2, 'cpu')
    pts, rows, _ = random_rows(5, 30, 2, seed=5)
    assert torch.equal(apply_f64(poses.table, pts, rows), pts)
    moved = random_poses(2, seed=6)
    rows = torch.tensor([0, -1, 1, 2, 1])
    q = apply_f64(moved.table, pts, rows)
    assert torch.equal(q[1], pts[1]) and torch.equal(q[3], pts[3]) and not torch.equal(q[0], pts[0])
    g = grad_f64(moved.table, q, torch.ones_like(q), rows, 1.0)
    keep = torch.tensor([True, False, True, False, True])
    assert torch.equal(g, grad_f64(moved.table, q[keep], torch.ones_like(q[keep]), rows[keep], 1.0))


def test_rodrigues_is_the_matrix_exponential():
    w = torch.tensor([[0.0, 0.0, 0.0], [1e-9, -2e-9, 0.0], [0.1, -0.2, 0.3], [2.0, 0.5, -1.0]], dtype=torch.float64)
    assert torch.equal(rodrigues_f64(w[:1])[0], torch.eye(3, dtype=torch.float64))
    for wi in w:
        z = torch.zeros((), dtype=torch.float64)
        K = torch.stack([torch.stack([z, -wi[2], wi[1]]), torch.stack([wi[2], z, -wi[0]]), torch.stack([-wi[1], wi[0], z])])
        assert torch.allclose(rodrigues_f64(wi[None])[0], torch.linalg.matrix_exp(K), atol=1e-14)


def test_retraction_stays_a_rotation_after_1000_steps():
    poses = random_poses(3, seed=7)
    g = torch.Generator().manual_seed(8)
    for step in range(1, 1001):
        poses.grad.copy_(torch.randn(3, 7, generator=g, dtype=torch.float64))
        poses.update(1.0, step)
    R = poses.table[:, :9].reshape(3, 3, 3)
    err = (R.transpose(1, 2) @ R - torch.eye(3, dtype=torch.float64)).abs().amax()
    assert err < 1e-12 and (torch.linalg.det(R) > 0).all()


def test_rigid_mode_holds_the_scale():
    poses = random_poses(2, seed=9, fit_scale=False)
    sigma = poses.table[:, 12].clone()
    poses.grad.fill_(0.3)
    for step in range(1, 6):
        poses.update(1.0, step)
    assert torch.equal(poses.table[:, 12], sigma)
    assert not torch.equal(poses.table[:, 9:12], random_poses(2, seed=9).table[:, 9:12])


def test_frozen_poses_skip_the_update():
    for kw in ({'fit': False}, {'lr': (0.0, 0.0, 0.0)}):
        poses = random_poses(2, seed=10, **kw)
        before = poses.table.clone()
        poses.grad.fill_(1.0)
        poses.update(1.0, 1)
        assert torch.equal(poses.table, before)


def test_matrices_and_frame_round_trip():
    poses = random_poses(3, seed=11)
    M = poses.matrices()
    p = torch.randn(100, 3, dtype=torch.float64)
    for o in range(3):
        q = poses.to_model(p, o)
        assert torch.allclose(q, p @ M[o, :3, :3].T + M[o, :3, 3], atol=1e-14)
        assert torch.allclose(poses.to_scan(q, o), p, atol=1e-13)
        assert torch.equal(poses.to_model(p[None].float(), o),
                           apply_f64(poses.table, p[None].float(), torch.tensor([o])))


def test_bad_arguments_raise():
    bad_R = torch.eye(3, dtype=torch.float64).repeat(2, 1, 1)
    bad_R[1, 0, 0] = 1.001
    reflect = torch.diag(torch.tensor([1.0, 1.0, -1.0], dtype=torch.float64)).repeat(2, 1, 1)
    for kw in ({'R': bad_R}, {'R': reflect}, {'R': torch.eye(3).repeat(3, 1, 1)}, {'t': torch.zeros(2, 2)},
               {'log_scale': torch.zeros(3)}, {'lr': (1e-3, -1.0, 0.0)}, {'lr': (1e-3, 1e-3)},
               {'t': torch.tensor([[0.0, 0.0, float('nan')]] * 2)}):
        with pytest.raises(ValueError):
            ObservationPoses(2, 'cpu', **kw)
    for n in (0, -1, 2.0):
        with pytest.raises(ValueError):
            ObservationPoses(n, 'cpu')
    dec = make_npm()
    obs = [torch.randn(100, 3) * 0.1 for _ in range(2)]
    with pytest.raises(ValueError):
        F.inference_identity_space(dec, obs, {'surface': 1.0}, 1, {}, poses=ObservationPoses(3, 'cpu'))
    with pytest.raises(ValueError):
        F.inference_identity_space_batched(dec, [obs, obs], {'surface': 1.0}, 1, {}, poses=[ObservationPoses(2, 'cpu')])
    with pytest.raises(ValueError):
        F.inference_identity_space(dec, obs, {'surface': 1.0}, 1, {}, poses='identity')


# ------------------------------------------------------------------------------------------- frozen poses: composite fitters
LAMBDAS = {'surface': 2.0, 'reg_expr': 0.01, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
SCHEDULE = {'lr': {200: 2, 400: 2}, 'symm_dist': {200: 10}, 'reg_glob': {200: 3}, 'reg_loc': {200: 3}, 'reg_expr': {200: 10}}


def _scans(sizes, seed):
    rng = np.random.RandomState(seed)
    return [torch.from_numpy((rng.randn(n, 3) * 0.1 + np.array([0.0, 0.05, -0.1])).astype(np.float32)) for n in sizes]


def _twice(fit, n_obs, lambdas=LAMBDAS):
    """``fit(lambdas, poses)`` without poses and with a frozen identity pose (rates 0): results, generator state, lambdas."""
    out = []
    for poses in (None, ObservationPoses(n_obs, 'cpu', lr=(0.0, 0.0, 0.0))):
        torch.manual_seed(5)
        lam = dict(lambdas)
        res = fit(lam, poses)
        out.append((res, torch.get_rng_state(), lam, poses))
    return out


def _flat(res):
    return [r for r in (res if isinstance(res, (tuple, list)) else [res]) if isinstance(r, torch.Tensor)]


def _assert_same(a, b):
    (ra, ga, la, _), (rb, gb, lb, poses) = a, b
    for x, y in zip(_flat(ra), _flat(rb)):
        assert torch.equal(x.detach(), y.detach())
    assert torch.equal(ga, gb) and la == lb
    assert torch.isfinite(poses.grad).all()


@pytest.mark.parametrize('decoder', ['npm', 'ensemble'])
def test_frozen_pose_identity_fit_is_unchanged(decoder):
    dec = make_npm() if decoder == 'npm' else make_ensemble(0).train()
    obs = _scans((1100, 1000, 1200), seed=1)
    lam = {k: v for k, v in LAMBDAS.items() if k != 'reg_expr'}
    _assert_same(*_twice(lambda l, p: F.inference_identity_space(dec, obs, l, 300, SCHEDULE, 0.01, poses=p), 3, lam))


def test_frozen_pose_joint_and_expression_fits_are_unchanged():
    dec = make_ensemble(0).train()
    dfn = make_deformation()
    obs = _scans((300, 300, 300), seed=2)
    _assert_same(*_twice(lambda l, p: F.inference_iterative_root_finding_joint(dec, dfn, obs, l, 200, SCHEDULE, 0.01, poses=p), 3))
    z_id = torch.randn(1, 1, dec.lat_dim) * 0.01
    _assert_same(*_twice(lambda l, p: F.inference_expression_space(dec, dfn, z_id, obs, l, 200, SCHEDULE, 0.01, poses=p), 3))
