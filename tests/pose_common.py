"""Shared by the pose tests (test_pose_cpu.py, test_gpu_pose.py): random poses and sampled rows, and the float64 autograd
statement of the pose gradient (q = exp(sigma) Exp(omega) R p + t, differentiated at omega = 0) that the closed form and the
kernels are compared against."""
import math

import numpy as np
import torch

from nphm_b200.models.pose import ObservationPoses


def random_rotation(rng, max_angle=0.3):
    w = rng.randn(3)
    w *= rng.uniform(0.0, max_angle) / np.linalg.norm(w)
    W = torch.tensor([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]], dtype=torch.float64)
    return torch.linalg.matrix_exp(W)


def random_poses(n, seed, device='cpu', **kw):
    rng = np.random.RandomState(seed)
    R = torch.stack([random_rotation(rng) for _ in range(n)])
    t = torch.from_numpy(rng.randn(n, 3) * 0.05)
    s = torch.from_numpy(rng.randn(n) * 0.03)
    return ObservationPoses(n, device, R=R.to(device), t=t.to(device), log_scale=s.to(device), **kw)


def random_rows(n_rows, n_point, n_obs, seed):
    """Points (n_rows x n_point x 3 fp32), rows' observations with repeats (int64), and an fp32 gradient per point."""
    g = torch.Generator().manual_seed(seed)
    pts = (torch.randn(n_rows, n_point, 3, generator=g) * 0.3).float()
    rows = torch.randint(0, n_obs, (n_rows,), generator=g)
    rows[-1] = rows[0]                                       # at least one repeated observation
    grad = (torch.randn(n_rows, n_point, 3, generator=g) * 1e-3).float()
    return pts, rows, grad


def autograd_pose_grad(table, p64, g, rows, lam_s):
    """d/d(omega, t, sigma) of lam_s sum <g, q> with q = exp(sigma + ds) Exp(dw) R p + t + dt at 0, by autograd in float64."""
    n = table.shape[0]
    xi = torch.zeros(n, 7, dtype=torch.float64, requires_grad=True)
    w = xi[:, :3]
    z = torch.zeros_like(w[:, 0])
    K = torch.stack([torch.stack([z, -w[:, 2], w[:, 1]], -1), torch.stack([w[:, 2], z, -w[:, 0]], -1),
                     torch.stack([-w[:, 1], w[:, 0], z], -1)], -2)
    R = torch.linalg.matrix_exp(K) @ table[:, :9].reshape(n, 3, 3)
    t = table[:, 9:12] + xi[:, 3:6]
    s = torch.exp(table[:, 12] + xi[:, 6])
    r = rows.long()
    q = s[r][:, None, None] * torch.einsum('rij,rnj->rni', R[r], p64) + t[r][:, None, :]
    (lam_s * (q * g.to(torch.float64)).sum()).backward()
    return xi.grad, q.detach()


def similarity(angle_deg, axis, t, scale):
    """R (3 x 3), t (3), log scale of a similarity, float64."""
    a = np.asarray(axis, dtype=np.float64)
    a = a / np.linalg.norm(a) * math.radians(angle_deg)
    W = torch.tensor([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]], dtype=torch.float64)
    return torch.linalg.matrix_exp(W), torch.tensor(t, dtype=torch.float64), math.log(scale)


# ------------------------------------------------------------------------ the pose gradient of the composite path in float64
def identity_pose_gradient(Q, obs, rows, table, z_id, lam_s, clamp, period=0):
    """d (lam_s mean |s(q)| over |s| < clamp) / d (omega, t, sigma), q = the pose of ``table`` applied to the sampled rows
    ``obs`` (nb x n x 3), in Q's dtype (joint_f64_common's decoder parameters); returns (n_obs x 7 float64, kept count)."""
    import joint_f64_common as J
    from nphm_b200.models.pose import compose_f64
    xi = torch.zeros(table.shape[0], 7, dtype=torch.float64, device=obs.device, requires_grad=True)
    q = compose_f64(table.double(), obs.double(), rows, xi).to(Q.dtype)
    a = J.identity_sdf(Q, q, z_id.to(Q.dtype), period).abs()
    kept = a.detach() < clamp
    (g,) = torch.autograd.grad(lam_s * a[kept].mean(), [xi])
    return g, int(kept.sum())


def joint_pose_gradient(Q, obs, rows, table, p, valid, z_id, z_ex, obs_idx, lam_s, clamp, period=0):
    """The same for one joint iteration at the Broyden roots ``p`` of x + F_ex(x) = q (held fixed, as the reference holds the
    correspondences): value(xc) = p and d xc / d q = J^-1 (joint_f64_common's formulation with q as the target)."""
    import chain_shapes_common as C
    import joint_f64_common as J
    from nphm_b200.models.pose import compose_f64
    dt = Q.dtype
    xi = torch.zeros(table.shape[0], 7, dtype=torch.float64, device=obs.device, requires_grad=True)
    q = compose_f64(table.double(), obs.double(), rows, xi).to(dt)
    p = p.to(dt)
    cond = J.condition(Q, z_id.to(dt), z_ex.to(dt), obs_idx)
    _, j_inv = C.ref_inverse_jacobian(Q.expr, p, cond)
    xc = p + torch.einsum('bnij,bnj->bni', j_inv.detach(), q - q.detach())
    a = J.identity_sdf(Q, xc, z_id.to(dt), period).abs()
    kept = valid.reshape(-1) & (a.detach() < clamp)
    (g,) = torch.autograd.grad(lam_s * a[kept].mean(), [xi])
    return g, int(kept.sum())


def clamp_in_a_gap(a):
    """A clamp in the widest gap between consecutive |s| within the middle half of their range: fp32 rounding cannot move a
    point across it."""
    a = a.reshape(-1).sort().values
    lo, hi = a.numel() // 4, a.numel() * 3 // 4
    gaps = a[lo + 1:hi + 1] - a[lo:hi]
    i = int(gaps.argmax())
    return float((a[lo + i] + a[lo + i + 1]) / 2)
