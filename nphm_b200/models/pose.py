"""Per-observation similarity transforms fitted together with the latent codes (DESIGN.md §4.24).

Observation ``o`` of a scan maps scan-frame points ``p`` to the model's canonical frame by

    q = exp(sigma_o) R_o p + t_o

The fitters sample rows of ``p`` exactly as without poses, move them to ``q`` with the pre-update pose and use ``q`` wherever
they used the observed points.  The surface term's derivative ``g_q = d surface / d q`` then gives, summed over the sampled rows
of observation ``o`` (``lam_s = lambdas['surface']``)::

    g_t = lam_s sum g_q        g_omega = lam_s sum (q - t) x g_q        g_sigma = lam_s sum g_q . (q - t)

for the left perturbation ``R <- Exp(omega) R``, and Adam on ``(omega, t, sigma)`` updates the pose in the same step as the
codes.  On CUDA the three steps are the kernels of csrc/pose.cu; the functions ``*_f64`` below restate them in torch float64
and are what CPU fits and the tests use.  The fit is local: it corrects errors of degrees and centimetres, not arbitrary
orientations - initialise far-off poses with :func:`nphm_b200.models.registration.register_scans` (DESIGN.md §4.25) before
fitting.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence

import torch

from .. import _native

# (lr_rot [rad], lr_trans [model units], lr_scale [log scale]) per Adam step at the fitters' initial code lr 0.01; each is
# multiplied by lr / lr_initial, so the fitters' schedule halves them with the codes' rate.  Adam moves a parameter by about
# its rate per step, so these reach a 10 degree, 0.1 unit, 5 % misalignment within the first ~100 of the fitters' several
# hundred steps and settle as the schedule halves them (the recovery tests in tests/test_gpu_pose.py).
DEFAULT_POSE_LR = (2e-3, 1e-3, 1e-3)

_ORTHO_TOL = 1e-6


# ------------------------------------------------------------------------------------------------------------ float64 mirror
def _cross_matrix(w: torch.Tensor) -> torch.Tensor:
    """... x 3 -> ... x 3 x 3, K w' = w x w'."""
    z = torch.zeros_like(w[..., 0])
    return torch.stack([torch.stack([z, -w[..., 2], w[..., 1]], -1),
                        torch.stack([w[..., 2], z, -w[..., 0]], -1),
                        torch.stack([-w[..., 1], w[..., 0], z], -1)], -2)


def rodrigues_f64(w: torch.Tensor) -> torch.Tensor:
    """Exp(w) = I + A K + B K^2 for n x 3 float64 rotation vectors, the series near 0 so that Exp(0) is exactly I."""
    th2 = (w * w).sum(-1)
    small = th2 < 1e-16
    th = th2.clamp_min(1e-300).sqrt()
    A = torch.where(small, 1.0 - th2 / 6.0, torch.sin(th) / th)
    B = torch.where(small, 0.5 - th2 / 24.0, (1.0 - torch.cos(th)) / th2.clamp_min(1e-300))
    K = _cross_matrix(w)
    eye = torch.eye(3, dtype=w.dtype, device=w.device).expand_as(K)
    return eye + A[:, None, None] * K + B[:, None, None] * (K @ K)


def orthonormalise_f64(R: torch.Tensor) -> torch.Tensor:
    """Gram-Schmidt on the rows of n x 3 x 3 matrices, the third row the cross product of the first two (det +1)."""
    r0 = R[:, 0] / R[:, 0].norm(dim=-1, keepdim=True)
    r1 = R[:, 1] - (r0 * R[:, 1]).sum(-1, keepdim=True) * r0
    r1 = r1 / r1.norm(dim=-1, keepdim=True)
    return torch.stack([r0, r1, torch.linalg.cross(r0, r1)], 1)


def _split(table: torch.Tensor):
    return table[:, :9].reshape(-1, 3, 3), table[:, 9:12], table[:, 12]


def apply_f64(table: torch.Tensor, points: torch.Tensor, rows: torch.Tensor) -> torch.Tensor:
    """``nphm_pose_apply``: q of rows x n x 3 points, row r moved by observation ``rows[r]``, in float64 in the kernel's order
    and rounded once to the points' dtype; rows outside [0, n_obs) are passed through."""
    n_obs = table.shape[0]
    rows = rows.long().to(table.device)
    pad = (rows < 0) | (rows >= n_obs)
    R, t, sigma = _split(table[rows.clamp(0, n_obs - 1)])
    s = torch.exp(sigma)
    p = points.to(torch.float64)
    q = (R[:, None, :, 0] * p[..., 0:1] + R[:, None, :, 1] * p[..., 1:2] + R[:, None, :, 2] * p[..., 2:3]) * s[:, None, None] \
        + t[:, None, :]
    q = q.to(points.dtype)
    return torch.where(pad[:, None, None], points, q)


def grad_f64(table: torch.Tensor, q: torch.Tensor, g: torch.Tensor, rows: torch.Tensor, lam_s: float) -> torch.Tensor:
    """``nphm_pose_grad`` in float64: n_obs x 7 ``(g_omega, g_t, g_sigma)`` of rows x n x 3 points ``q`` and ``g = d/d q``."""
    n_obs = table.shape[0]
    rows = rows.long().to(table.device)
    keep = (rows >= 0) & (rows < n_obs)
    t = table[rows.clamp(0, n_obs - 1), 9:12]
    a = q.to(torch.float64) - t[:, None, :]
    gg = g.to(torch.float64)
    per_row = torch.cat([torch.linalg.cross(a, gg).sum(1), gg.sum(1), (gg * a).sum(-1).sum(1, keepdim=True)], 1)
    out = torch.zeros(n_obs, 7, dtype=torch.float64, device=table.device)
    out.index_add_(0, rows[keep], per_row[keep])
    return lam_s * out


def adam_f64(table: torch.Tensor, m: torch.Tensor, v: torch.Tensor, grad: torch.Tensor, lrs: Sequence[float], fit_scale: bool,
             step: int) -> None:
    """``nphm_pose_adam`` in float64, in place on ``table``, ``m`` and ``v``."""
    m.mul_(0.9).add_(0.1 * grad)
    v.mul_(0.999).add_(0.001 * (grad * grad))
    bc1, bc2 = 1.0 - 0.9 ** step, 1.0 - 0.999 ** step
    lr = torch.tensor([lrs[0]] * 3 + [lrs[1]] * 3 + [lrs[2]], dtype=torch.float64, device=table.device)
    d = -((lr / bc1) * (m / (v.sqrt() / math.sqrt(bc2) + 1e-8)))
    R, t, sigma = _split(table)
    R_new = orthonormalise_f64(rodrigues_f64(d[:, :3]) @ R)
    table[:, :9] = R_new.reshape(-1, 9)
    table[:, 9:12] += d[:, 3:6]
    if fit_scale:
        table[:, 12] += d[:, 6]


def compose_f64(table: torch.Tensor, points: torch.Tensor, rows: torch.Tensor, xi: torch.Tensor) -> torch.Tensor:
    """The autograd fallback's q: the pose of ``table`` perturbed by the tangent ``xi`` (n_obs x 7, zero, a leaf), to first
    order - exact at ``xi = 0``, where its value is :func:`apply_f64`'s and ``d q / d xi`` is the contract's."""
    rows = rows.long().to(table.device)
    R, t, sigma = _split(table)
    R = R + _cross_matrix(xi[:, :3]) @ R
    t = t + xi[:, 3:6]
    sigma = sigma + xi[:, 6]
    R, t, s = R[rows], t[rows], torch.exp(sigma[rows])
    p = points.to(torch.float64)
    q = (R[:, None, :, 0] * p[..., 0:1] + R[:, None, :, 1] * p[..., 1:2] + R[:, None, :, 2] * p[..., 2:3]) * s[:, None, None] \
        + t[:, None, :]
    return q.to(points.dtype)


# ------------------------------------------------------------------------------------------------------------ the state
def _device(device) -> torch.device:
    """``device`` with an index-less ``'cuda'`` resolved to the current CUDA device, as tensors created there carry it."""
    d = torch.device(device)
    if d.type == 'cuda' and d.index is None:
        d = torch.device('cuda', torch.cuda.current_device())
    return d


class ObservationPoses:
    """Similarity transforms scan -> model of ``n_observations`` observations, fitted by the fitters that take ``poses=``.

    ``R`` (n x 3 x 3, orthonormal with det +1 to 1e-6), ``t`` (n x 3) and ``log_scale`` (n) initialise the pose (default: the
    identity).  ``lr = (lr_rot, lr_trans, lr_scale)``: Adam rates at the fitters' initial code rate, scaled with it by the
    schedule (default :data:`DEFAULT_POSE_LR`).  ``fit_scale=False`` holds the scale fixed (a rigid fit); ``fit=False`` or all
    rates 0 holds the whole pose fixed, and the fit then gives the result it gives without poses.  The fitters update the
    object in place: ``table`` (n x 13 float64 on ``device``: R row-major, t, sigma), the Adam moments ``m`` / ``v`` and the last
    step's gradient ``grad`` (n x 7: omega, t, sigma)."""

    def __init__(self, n_observations: int, device, R=None, t=None, log_scale=None, fit_scale: bool = True,
                 lr=DEFAULT_POSE_LR, fit: bool = True):
        if isinstance(n_observations, bool) or not isinstance(n_observations, int) or n_observations < 1:
            raise ValueError('n_observations must be a positive int, got %r' % (n_observations,))
        self.device = _device(device)
        n = n_observations
        lr = tuple(float(x) for x in lr)
        if len(lr) != 3 or not all(math.isfinite(x) and x >= 0 for x in lr):
            raise ValueError('lr must be three finite non-negative rates (rot, trans, scale), got %r' % (lr,))
        table = torch.zeros(n, 13, dtype=torch.float64)
        table[:, [0, 4, 8]] = 1.0
        if R is not None:
            R = self._input(R, (n, 3, 3), 'R')
            err = (R.transpose(1, 2) @ R - torch.eye(3, dtype=torch.float64)).abs().amax()
            if not bool(err <= _ORTHO_TOL) or not bool((torch.linalg.det(R) > 0).all()):
                raise ValueError('R must be rotations: orthonormal to %g with det +1' % _ORTHO_TOL)
            table[:, :9] = R.reshape(n, 9)
        if t is not None:
            table[:, 9:12] = self._input(t, (n, 3), 't')
        if log_scale is not None:
            table[:, 12] = self._input(log_scale, (n,), 'log_scale')
        self.n = n
        self.lr, self.fit_scale, self.fit = lr, bool(fit_scale), bool(fit)
        self.table = table.to(self.device)
        self.m = torch.zeros(n, 7, dtype=torch.float64, device=self.device)
        self.v = torch.zeros_like(self.m)
        self.grad = torch.zeros_like(self.m)

    def _input(self, x, shape, name) -> torch.Tensor:
        if isinstance(x, torch.Tensor) and x.device != self.device:
            raise ValueError('%s is on %s, the poses on %s' % (name, x.device, self.device))
        x = torch.as_tensor(x, dtype=torch.float64).cpu()
        if tuple(x.shape) != shape or not bool(torch.isfinite(x).all()):
            raise ValueError('%s must be finite with shape %s, got %s' % (name, shape, tuple(x.shape)))
        return x

    @property
    def frozen(self) -> bool:
        """Whether a fit leaves the pose unchanged (``fit=False`` or all rates 0)."""
        return not self.fit or not any(self.lr)

    def matrices(self) -> torch.Tensor:
        """n x 4 x 4 float64: the scan -> model transforms ``[[s R, t], [0, 1]]``."""
        R, t, sigma = _split(self.table)
        out = torch.zeros(self.n, 4, 4, dtype=torch.float64, device=self.device)
        out[:, :3, :3] = torch.exp(sigma)[:, None, None] * R
        out[:, :3, 3] = t
        out[:, 3, 3] = 1.0
        return out

    def to_model(self, points: torch.Tensor, o: int) -> torch.Tensor:
        """Points (... x 3) of observation ``o``'s scan frame in the model frame (float64 arithmetic, the points' dtype)."""
        R, t, sigma = _split(self.table[o:o + 1].to(points.device))
        p = points.to(torch.float64)
        return (torch.exp(sigma[0]) * (p @ R[0].T) + t[0]).to(points.dtype)

    def to_scan(self, points: torch.Tensor, o: int) -> torch.Tensor:
        """The inverse of :meth:`to_model`: model-frame points (a fitted or posed mesh's vertices) in observation ``o``'s frame."""
        R, t, sigma = _split(self.table[o:o + 1].to(points.device))
        q = points.to(torch.float64)
        return (((q - t[0]) @ R[0]) * torch.exp(-sigma[0])).to(points.dtype)

    # -------------------------------------------------------------------------------------- the fitters' three steps
    def check_for(self, n_observations: int, device) -> None:
        if self.n != n_observations:
            raise ValueError('the poses hold %d observations, the fit has %d' % (self.n, n_observations))
        if self.device != _device(device):
            raise ValueError('the poses are on %s, the observations on %s' % (self.device, device))

    def _rows_args(self, points: torch.Tensor, rows: torch.Tensor, what: str):
        if points.dim() != 3 or points.shape[-1] != 3 or rows.dim() != 1 or rows.shape[0] != points.shape[0]:
            raise ValueError('%s: points must be rows x n x 3 and rows one index per row, got %s and %s'
                             % (what, tuple(points.shape), tuple(rows.shape)))
        return (points.to(device=self.device, dtype=torch.float32).contiguous(),
                rows.to(device=self.device, dtype=torch.int32).contiguous())

    def apply(self, points: torch.Tensor, rows: torch.Tensor) -> torch.Tensor:
        """q of rows x n x 3 fp32 points, row r drawn from observation ``rows[r]`` (``nphm_pose_apply`` on CUDA).  Inputs on
        another device are copied to the poses' device."""
        if self.device.type != 'cuda':
            return apply_f64(self.table, points, rows)
        pts, rows = self._rows_args(points, rows, 'apply')
        out = torch.empty_like(pts)
        with torch.cuda.device(self.device):
            _native.check(_native.lib().nphm_pose_apply(pts.data_ptr(), rows.data_ptr(), pts.shape[0], pts.shape[1],
                                                        self.table.data_ptr(), self.n, out.data_ptr(),
                                                        _native._stream_ptr(self.device)), 'nphm_pose_apply')
        return out

    def gradient(self, q: torch.Tensor, g_q: torch.Tensor, rows: torch.Tensor, lam_s: float) -> None:
        """``grad`` from the points ``q`` and ``g_q = d surface / d q`` (rows x n x 3) (``nphm_pose_grad`` on CUDA)."""
        if self.device.type != 'cuda':
            self.grad.copy_(grad_f64(self.table, q, g_q, rows, lam_s))
            return
        if g_q.shape != q.shape:
            raise ValueError('gradient: g_q has shape %s, q %s' % (tuple(g_q.shape), tuple(q.shape)))
        q, rows = self._rows_args(q, rows, 'gradient')
        g_q = g_q.to(device=self.device, dtype=torch.float32).contiguous()
        with torch.cuda.device(self.device):
            _native.check(_native.lib().nphm_pose_grad(q.data_ptr(), g_q.data_ptr(), rows.data_ptr(), q.shape[0], q.shape[1],
                                                       self.table.data_ptr(), self.n, float(lam_s), self.grad.data_ptr(),
                                                       _native._stream_ptr(self.device)), 'nphm_pose_grad')

    def rates(self, lr_factor: float):
        return tuple(x * lr_factor for x in self.lr)

    def update(self, lr_factor: float, step: int, native: bool = True) -> None:
        """Adam on ``grad`` with the rates times ``lr_factor`` (the fitter's lr / lr_initial) at the fitter's 1-based ``step``;
        nothing when the pose is frozen.  ``native=False``: the float64 mirror (the autograd fallback's update)."""
        if self.frozen:
            return
        lrs = self.rates(lr_factor)
        if self.device.type != 'cuda' or not native:
            adam_f64(self.table, self.m, self.v, self.grad, lrs, self.fit_scale, step)
            return
        with torch.cuda.device(self.device):
            _native.check(_native.lib().nphm_pose_adam(self.table.data_ptr(), self.m.data_ptr(), self.v.data_ptr(),
                                                       self.grad.data_ptr(), self.n, lrs[0], lrs[1], lrs[2], int(self.fit_scale),
                                                       int(step), _native._stream_ptr(self.device)), 'nphm_pose_adam')

    # ------------------------------------------------------------------------------- one table for a batch of scans
    @staticmethod
    def concat(poses: List['ObservationPoses']) -> 'ObservationPoses':
        """One object over the observations of several scans in order (the batched fitters' shared table).  The batched
        fitters run one Adam update over the whole table, so all scans' poses must share device, rates, ``fit_scale`` and
        ``fit`` (``ValueError`` otherwise).  :meth:`scatter` writes the fitted state back."""
        first = poses[0]
        for p in poses[1:]:
            if (p.device, p.lr, p.fit_scale, p.fit) != (first.device, first.lr, first.fit_scale, first.fit):
                raise ValueError('the batched fitters need one device, rate set and flags for every scan\'s poses')
        out = ObservationPoses.__new__(ObservationPoses)
        out.n, out.device = sum(p.n for p in poses), first.device
        out.lr, out.fit_scale, out.fit = first.lr, first.fit_scale, first.fit
        out.table = torch.cat([p.table for p in poses]).contiguous()
        out.m = torch.cat([p.m for p in poses]).contiguous()
        out.v = torch.cat([p.v for p in poses]).contiguous()
        out.grad = torch.cat([p.grad for p in poses]).contiguous()
        return out

    def scatter(self, poses: List['ObservationPoses']) -> None:
        o = 0
        for p in poses:
            for mine, theirs in ((self.table, p.table), (self.m, p.m), (self.v, p.v), (self.grad, p.grad)):
                theirs.copy_(mine[o:o + p.n])
            o += p.n


def check_poses(poses: Optional[ObservationPoses], n_observations: int, device) -> None:
    if poses is None:
        return
    if not isinstance(poses, ObservationPoses):
        raise ValueError('poses must be an ObservationPoses, got %s' % type(poses).__name__)
    poses.check_for(n_observations, device)
