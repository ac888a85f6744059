"""Global registration of observations against a head's SDF (DESIGN.md §4.25): the start of the pose fit.

:func:`register_observations` searches, for every observation of every scan, the similarity ``q = exp(sigma) R p + t`` that
lays its points on the zero level set of an SDF grid, and returns the :class:`~nphm_b200.models.pose.ObservationPoses` that the
fitters' ``poses=`` argument takes.  :func:`register_scans` builds the grid of one head from a decoder first.  The pipeline is::

    poses = register_scans(decoder, scans)
    inference_identity_space_batched(decoder, scans, ..., poses=poses)     # or poses[0] with the single-scan fitters

The search (csrc/register.cu on CUDA; the float64 mirror below on the CPU and in the tests):

1. The volume becomes a float4 grid of the SDF and its central-difference gradient (:func:`prepare_torch`).
2. Every observation gets ``n_rotations`` near-uniform rotations (:func:`rotation_set`) times five scale seeds
   ``s0 2^{-1/2 .. 1/2}`` (one, rigid, with a known ``log_scale``), ``s0`` the ratio of the template's near-surface RMS radius
   to the observation's, and the translation that maps the observation's centroid onto the template's.
3. Each hypothesis runs a truncated Gauss-Newton on ``r = sdf(q) u / s`` (``u`` the observation's reference scale ``s0``), the
   Levenberg-Marquardt-damped 7 x 7 (6 x 6 rigid) system solved in float64, ``R <- Exp(d omega) R``, ``sigma`` held within
   ``log 2 / 8`` of its seed.  Score ``mean(min(r^2, tau^2))``, a point outside the grid scoring ``tau^2``.
4. A coarse stage runs every hypothesis on a few hundred points; the best ``top_k`` per observation (a stable sort on the
   device, ties by hypothesis index) run a fine stage on up to 8192 points, and the best fine score wins.  No host
   synchronisation between the stages.

The search assumes a distance-like SDF (gradient norm near 1 at the surface): its truncation, its score and the template's
near-surface shell are in distance units, so a field far from a distance is not a usable target.

Neither function draws from torch's global generators (the fitters reproduce the reference's random stream); the point subsets
come from a local generator seeded with ``seed``.
"""
from __future__ import annotations

import math
from ctypes import byref, c_float
from typing import Optional, Sequence

import numpy as np
import torch

from .. import _native
from .pose import DEFAULT_POSE_LR, ObservationPoses, orthonormalise_f64, rodrigues_f64

MINI = (-.55, -.5, -.95)                 # the fitting grid's bounds (fitting_pointclouds.py)
MAXI = (0.55, 0.75, 0.4)

N_ROTATIONS = 1024                       # largest gap to a uniform random rotation: 22.0 degrees (2e5 samples)
SCALE_SEEDS = (-0.5, -0.25, 0.0, 0.25, 0.5)     # log2 offsets from s0; each seed covers +- log 2 / 8 of sigma
SIGMA_BAND = math.log(2.0) / 8
COARSE = dict(points=512, iters=10, tau=(0.2, 0.05))
FINE = dict(points=8192, iters=30, tau=(0.05, 0.01), top_k=16)
DAMPING = 1e-3
RUNNER_UP_DEG = 20.0


# ------------------------------------------------------------------------------------------------------------ hypotheses
def rotation_set(n: int) -> torch.Tensor:
    """n x 4 float64 unit quaternions (w, x, y, z): the super-Fibonacci spiral (Alexa, CVPR 2022), deterministic and
    near-uniform on SO(3)."""
    phi, psi = math.sqrt(2.0), 1.533751168755204288118041
    s = np.arange(n, dtype=np.float64) + 0.5
    r, R = np.sqrt(s / n), np.sqrt(1.0 - s / n)
    alpha, beta = 2.0 * np.pi * s / phi, 2.0 * np.pi * s / psi
    q = np.stack([r * np.sin(alpha), r * np.cos(alpha), R * np.sin(beta), R * np.cos(beta)], 1)
    return torch.from_numpy(q / np.linalg.norm(q, axis=1, keepdims=True))


def quaternion_matrices(q: torch.Tensor) -> torch.Tensor:
    """n x 4 unit quaternions (w, x, y, z) -> n x 3 x 3 rotation matrices."""
    w, x, y, z = q.unbind(-1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                        2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                        2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)


# ------------------------------------------------------------------------------------------------------------ the grid
class Grid:
    """A res^3 grid from ``mini`` with fp32 spacing ``h = (maxi - mini) / (res - 1)``, the numbers the kernels see."""

    def __init__(self, res: int, mini, maxi):
        self.res = int(res)
        self.mini = np.asarray(mini, dtype=np.float32)
        self.h = ((np.asarray(maxi, dtype=np.float64) - np.asarray(mini, dtype=np.float64)) / (res - 1)).astype(np.float32)

    def coordinates(self, device) -> torch.Tensor:
        """res^3 x 3 float64 grid points, x slowest, z fastest (create_grid_points_from_bounds' order)."""
        ax = [torch.arange(self.res, dtype=torch.float64, device=device) * float(self.h[a]) + float(self.mini[a])
              for a in range(3)]
        return torch.stack(torch.meshgrid(*ax, indexing='ij'), -1).reshape(-1, 3)


def prepare_torch(volume: torch.Tensor, grid: Grid) -> torch.Tensor:
    """``nphm_register_prepare``: res^3 x 4 fp32 (sdf, d/dx, d/dy, d/dz), central differences ``(v+ - v-) / (2 h)``, one-sided
    ``(v1 - v0) / h`` at the faces, every operation an fp32 operation rounded once (the kernel's bits)."""
    n = grid.res
    v = volume.reshape(n, n, n).to(torch.float32)
    out = [v]
    for a in range(3):
        h = torch.tensor(float(grid.h[a]), dtype=torch.float32, device=v.device)
        vm = v.movedim(a, 0)
        g = torch.empty_like(vm)
        g[1:-1] = (vm[2:] - vm[:-2]) / (h * 2)
        g[0] = (vm[1] - vm[0]) / h
        g[-1] = (vm[-1] - vm[-2]) / h
        out.append(g.movedim(0, a))
    return torch.stack(out, -1).reshape(-1, 4).contiguous()


def sample_f64(field: torch.Tensor, grid: Grid, q: torch.Tensor):
    """Trilinear (value, gradient) of the float4 grid at ... x 3 points, in float64: (inside, f, n)."""
    res = grid.res
    u = (q - torch.as_tensor(grid.mini, dtype=torch.float64, device=q.device)) \
        / torch.as_tensor(grid.h, dtype=torch.float64, device=q.device)
    inside = ((u >= 0) & (u <= res - 1)).all(-1)
    u = torch.where(inside[..., None], u, torch.zeros_like(u))
    i = u.floor().long().clamp(max=res - 2)
    f = u - i
    F = field.to(torch.float64)
    out = 0
    for dx in (0, 1):
        for dy in (0, 1):
            for dz in (0, 1):
                w = ((f[..., 0] if dx else 1 - f[..., 0]) * (f[..., 1] if dy else 1 - f[..., 1])
                     * (f[..., 2] if dz else 1 - f[..., 2]))
                idx = ((i[..., 0] + dx) * res + i[..., 1] + dy) * res + i[..., 2] + dz
                out = out + w[..., None] * F[idx]
    return inside, out[..., 0], out[..., 1:]


# ------------------------------------------------------------------------------------------------------------ float64 mirror
def tau_at(tau, it: int, n_iter: int) -> float:
    """The truncation of iteration ``it``: geometric from tau[0] (first) to tau[1] (last and scoring)."""
    tau0, tau1 = tau
    if it >= n_iter or tau0 == tau1:
        return tau1
    return tau0 * (tau1 / tau0) ** (it / (n_iter - 1)) if n_iter > 1 else tau0


def _hypothesis_points(points, offsets, counts, hyp_obs, n_use):
    """H x M x 3 float64 points of every hypothesis' observation (the first min(count, n_use)) and their mask."""
    m = torch.clamp(counts.long(), max=n_use)[hyp_obs.long()]
    M = int(min(int(counts.max()), n_use))
    j = torch.arange(M, device=points.device)
    mask = j[None, :] < m[:, None]
    idx = (offsets[hyp_obs.long()][:, None] + torch.minimum(j[None, :], (m - 1).clamp_min(0)[:, None]))
    return points[idx].to(torch.float64), mask


def residuals_f64(field, grid, table, p, unit):
    """At the poses of ``table`` (H x 13) and points ``p`` (H x M x 3 float64): the inside flags, the residuals
    ``r = sdf(q) u / s``, the Jacobian rows (H x M x 7: omega, t, sigma) and the raw samples (a = q - t, f, n)."""
    R, t, sigma = table[:, :9].reshape(-1, 3, 3), table[:, 9:12], table[:, 12]
    s = torch.exp(sigma)
    a = s[:, None, None] * torch.einsum('hij,hmj->hmi', R, p)
    q = a + t[:, None, :]
    inside, f, n = sample_f64(field, grid, q)
    ws = (unit / s)[:, None]
    J = torch.cat([torch.linalg.cross(a, n), n, ((n * a).sum(-1) - f)[..., None]], -1) * ws[..., None]
    return inside, f * ws, J, (a, f, n)


def normal_equations_f64(field, grid, table, p, mask, unit, tau, fit_scale):
    """A = J^T W J (H x D x D), b = J^T W r (H x D) and the weight count, W the truncation ``|r| < tau`` inside the grid."""
    inside, r, J, _ = residuals_f64(field, grid, table, p, unit)
    w = (mask & inside & (r.abs() < tau)).to(torch.float64)
    D = 7 if fit_scale else 6
    J = J[..., :D]
    A = torch.einsum('hm,hmi,hmj->hij', w, J, J)
    b = torch.einsum('hm,hmi,hm->hi', w, J, r)
    return A, b, w.sum(1)


def score_f64(field, grid, table, p, mask, unit, tau1):
    """(score, inlier count): mean over the points of min(r^2, tau1^2), tau1^2 for a point outside the grid."""
    inside, r, _, _ = residuals_f64(field, grid, table, p, unit)
    per = torch.where(inside, torch.minimum(r * r, torch.full_like(r, tau1 * tau1)), torch.full_like(r, tau1 * tau1))
    m = mask.to(torch.float64)
    count = m.sum(1)
    score = torch.where(count > 0, (per * m).sum(1) / count.clamp_min(1), torch.full_like(count, tau1 * tau1))
    inl = ((r.abs() < tau1) & inside & mask).sum(1).to(torch.int32)
    return score, inl


def step_f64(table, A, b, count, sigma_seed, damping, fit_scale):
    """One damped Gauss-Newton step in place on ``table``: delta = -(A + damping diag(A))^-1 b, R <- Exp(d omega) R
    re-orthonormalised, t += d t, sigma += d sigma clamped to sigma_seed +- log 2 / 8; no step with fewer weights than
    parameters, a non-positive pivot or a non-finite step."""
    D = A.shape[-1]
    Ad = A + torch.diag_embed(A.diagonal(dim1=-2, dim2=-1) * damping)
    L, info = torch.linalg.cholesky_ex(Ad)
    delta = -torch.cholesky_solve(b[..., None], L)[..., 0]
    ok = (count >= D) & (info == 0) & torch.isfinite(delta).all(-1)
    delta = torch.where(ok[:, None], delta, torch.zeros_like(delta))
    R = table[:, :9].reshape(-1, 3, 3)
    R_new = orthonormalise_f64(rodrigues_f64(delta[:, :3]) @ R)
    table[:, :9] = torch.where(ok[:, None], R_new.reshape(-1, 9), table[:, :9])
    table[:, 9:12] += delta[:, 3:6]
    if fit_scale:
        table[:, 12] = torch.minimum(torch.maximum(table[:, 12] + delta[:, 6], sigma_seed - SIGMA_BAND), sigma_seed + SIGMA_BAND)
    return delta


def search_f64(field, grid, points, offsets, counts, unit, table, sigma_seed, hyp_obs, n_use, n_iter, tau, damping,
               fit_scale, chunk_points: int = 1 << 21):
    """``nphm_register_search`` in float64: ``table`` updated in place; returns (score, inliers).  Hypotheses are
    independent, so they run in chunks of about ``chunk_points`` hypothesis-points, which bounds the memory."""
    H = table.shape[0]
    per = max(1, chunk_points // max(1, min(int(counts.max()), n_use)))
    scores, inliers = [], []
    for h0 in range(0, H, per):
        sl = slice(h0, min(H, h0 + per))
        tab = table[sl]
        p, mask = _hypothesis_points(points, offsets, counts, hyp_obs[sl], n_use)
        u = unit[hyp_obs[sl].long()]
        for it in range(n_iter):
            A, b, count = normal_equations_f64(field, grid, tab, p, mask, u, tau_at(tau, it, n_iter), fit_scale)
            step_f64(tab, A, b, count, sigma_seed[sl], damping, fit_scale)
        sc, inl = score_f64(field, grid, tab, p, mask, u, tau[1])
        scores.append(sc)
        inliers.append(inl)
    return torch.cat(scores), torch.cat(inliers)


# ------------------------------------------------------------------------------------------------------------ native
def prepare(volume: torch.Tensor, grid: Grid) -> torch.Tensor:
    """The float4 field of a volume: ``nphm_register_prepare`` on CUDA, :func:`prepare_torch` elsewhere."""
    if volume.device.type != 'cuda':
        return prepare_torch(volume, grid)
    vol = volume.reshape(-1).to(torch.float32).contiguous()
    out = torch.empty(vol.numel(), 4, dtype=torch.float32, device=vol.device)
    with torch.cuda.device(vol.device):
        _native.check(_native.lib().nphm_register_prepare(vol.data_ptr(), grid.res, float(grid.h[0]), float(grid.h[1]),
                                                          float(grid.h[2]), out.data_ptr(), _native._stream_ptr(vol.device)),
                      'nphm_register_prepare')
    return out


def search(field, grid, points, offsets, counts, unit, table, sigma_seed, hyp_obs, n_use, n_iter, tau, damping, fit_scale,
           max_points):
    """One stage over every hypothesis, ``table`` updated in place; returns (score H fp64, inliers H int32).  CUDA runs
    ``nphm_register_search``; anything else :func:`search_f64`.  ``max_points``: the largest min(count, n_use)."""
    if field.device.type != 'cuda':
        return search_f64(field, grid, points, offsets, counts, unit, table, sigma_seed, hyp_obs, n_use, n_iter, tau,
                          damping, fit_scale)
    H = table.shape[0]
    prm = _native.RegisterParams(grid.res, (c_float * 3)(*map(float, grid.mini)), (c_float * 3)(*map(float, grid.h)),
                                 int(unit.shape[0]), int(n_use), int(H), int(n_iter), int(bool(fit_scale)), float(tau[0]),
                                 float(tau[1]), float(damping))
    score = torch.empty(H, dtype=torch.float64, device=field.device)
    inliers = torch.empty(H, dtype=torch.int32, device=field.device)
    with torch.cuda.device(field.device):
        _native.check(_native.lib().nphm_register_search(
            byref(prm), field.data_ptr(), points.data_ptr(), offsets.data_ptr(), counts.data_ptr(), unit.data_ptr(),
            table.data_ptr(), sigma_seed.data_ptr(), hyp_obs.data_ptr(), int(max_points), score.data_ptr(),
            inliers.data_ptr(), _native._stream_ptr(field.device)), 'nphm_register_search')
    return score, inliers


# ------------------------------------------------------------------------------------------------------------ public API
def _check_volume(volume, mini, maxi):
    if not isinstance(volume, torch.Tensor) or not volume.is_floating_point():
        raise ValueError('volume must be a floating-point tensor')
    n = volume.numel()
    res = int(round(n ** (1.0 / 3.0)))
    if res ** 3 != n or (volume.dim() != 1 and tuple(volume.shape) != (res,) * 3):
        raise ValueError('volume must hold res^3 values (flat or res x res x res), got shape %s' % (tuple(volume.shape),))
    if res < 2:
        raise ValueError('the volume needs at least 2 points per axis, got res = %d' % res)
    mini, maxi = np.asarray(mini, dtype=np.float64), np.asarray(maxi, dtype=np.float64)
    if mini.shape != (3,) or maxi.shape != (3,) or not (np.isfinite(mini).all() and np.isfinite(maxi).all()) \
            or not (maxi > mini).all():
        raise ValueError('mini and maxi must be 3 finite bounds with maxi > mini')
    return res


def _check_scans(scans, device=None):
    """Validates the scans; ``device``: the one they must be on (default: the first observation's)."""
    if not isinstance(scans, (list, tuple)) or not scans:
        raise ValueError('scans must be a non-empty list of scans, each a list of (n, 3) observations')
    for k, scan in enumerate(scans):
        if not isinstance(scan, (list, tuple)) or not scan:
            raise ValueError('scan %d must be a non-empty list of (n, 3) observations' % k)
        for o, x in enumerate(scan):
            if not isinstance(x, torch.Tensor) or x.dim() != 2 or x.shape[1] != 3 or x.shape[0] < 1:
                raise ValueError('scan %d, observation %d must be a non-empty (n, 3) tensor' % (k, o))
            device = x.device if device is None else device
            if x.device != device:
                raise ValueError('scan %d, observation %d is on %s, the volume on %s' % (k, o, x.device, device))
            if not bool(torch.isfinite(x).all()):
                raise ValueError('scan %d, observation %d has non-finite points' % (k, o))


def _log_scales(log_scale, n_scans):
    """None, or one finite log scale per scan (a single number applies to every scan)."""
    if log_scale is None:
        return None

    def number(v):
        return isinstance(v, (int, float)) and not isinstance(v, bool)
    if number(log_scale):
        vals = [float(log_scale)] * n_scans
    elif isinstance(log_scale, (list, tuple)) and all(number(v) for v in log_scale):
        vals = [float(v) for v in log_scale]
    else:
        vals = None
    if vals is None or len(vals) != n_scans or not all(math.isfinite(v) for v in vals):
        raise ValueError('log_scale must be a finite number or one per scan, got %r' % (log_scale,))
    return vals


def register_observations(volume: torch.Tensor, mini, maxi, scans: Sequence[Sequence[torch.Tensor]], log_scale=None,
                          return_stats: bool = False, n_rotations: int = N_ROTATIONS, coarse: Optional[dict] = None,
                          fine: Optional[dict] = None, damping: float = DAMPING, seed: int = 0, lr=DEFAULT_POSE_LR):
    """Register every observation of ``scans`` (a list of scans, each a list of (n_o, 3) observations in the scan's frame, on
    the volume's device) against the SDF ``volume`` (res^3 values in get_logits' layout over the box [mini, maxi]).

    Returns one :class:`ObservationPoses` per scan, one pose per observation, ready for the fitters' ``poses=``.  With
    ``log_scale`` (the known log of the scan -> model scale: one number, or one per scan) the search is rigid and the poses
    have ``fit_scale=False``.  ``coarse`` / ``fine`` override :data:`COARSE` / :data:`FINE` (points, iters, tau, top_k).  With
    ``return_stats`` also a list per scan of dicts of per-observation tensors: ``score`` (the winner's, model units^2),
    ``inlier_fraction`` and ``runner_up`` (the best fine score whose rotation ends more than 20 degrees from the winner's;
    ``tau^2`` when there is none).  A runner-up close to the score flags an ambiguous registration."""
    res = _check_volume(volume, mini, maxi)
    device = volume.device
    _check_scans(scans, device)
    log_scales = _log_scales(log_scale, len(scans))
    if isinstance(n_rotations, bool) or not isinstance(n_rotations, int) or n_rotations < 1:
        raise ValueError('n_rotations must be a positive int')
    if not (math.isfinite(damping) and damping >= 0):
        raise ValueError('damping must be finite and non-negative')
    cs, fs = dict(COARSE, **(coarse or {})), dict(FINE, **(fine or {}))
    for st in (cs, fs):
        tau = tuple(float(x) for x in st['tau'])
        if len(tau) != 2 or not all(x > 0 for x in tau) or int(st['points']) < 1 or int(st['iters']) < 0 \
                or int(st.get('top_k', 1)) < 1:
            raise ValueError('stage settings need points >= 1, iters >= 0, top_k >= 1 and two positive taus, got %r' % (st,))
        st['tau'] = tau
    rigid = log_scales is not None
    grid = Grid(res, mini, maxi)
    field = prepare(volume, grid)

    # template: centroid and RMS radius of the near-surface grid points
    near = (volume.reshape(-1).abs() < float(grid.h.max())).to(torch.float64)
    if not bool(near.any()):
        raise ValueError('the volume has no grid point within one spacing of its zero level set: no surface to register to')
    xyz = grid.coordinates(device)
    n_near = near.sum().clamp_min(1)
    c_t = (xyz * near[:, None]).sum(0) / n_near
    rms_t = (((xyz - c_t).square().sum(1) * near).sum() / n_near).sqrt()

    # observations, each subsampled by a local generator; points of observation o at offsets[o] .. + counts[o]
    obs = [x for scan in scans for x in scan]
    n_obs_per_scan = [len(s) for s in scans]
    O = len(obs)
    n_keep = max(int(cs['points']), int(fs['points']))
    subsets, counts_h = [], []
    for x in obs:          # a fresh generator per observation: its subset does not depend on the other observations
        idx = torch.randperm(x.shape[0], generator=torch.Generator().manual_seed(int(seed)))[:n_keep]
        subsets.append(x[idx.to(device)].to(torch.float32))
        counts_h.append(int(idx.numel()))
    points = torch.cat(subsets).contiguous()
    offsets = torch.tensor(np.concatenate([[0], np.cumsum(counts_h)[:-1]]), dtype=torch.int64, device=device)
    counts = torch.tensor(counts_h, dtype=torch.int32, device=device)
    c_o = torch.stack([x.to(torch.float64).mean(0) for x in obs])
    rms_o = torch.stack([(x.to(torch.float64) - c).square().sum(1).mean().sqrt() for x, c in zip(obs, c_o)])
    if rigid:
        log_s0 = torch.tensor([v for v, n in zip(log_scales, n_obs_per_scan) for _ in range(n)], dtype=torch.float64,
                              device=device)
    else:
        log_s0 = (rms_t / rms_o.clamp_min(1e-30)).log()
    unit = log_s0.exp().contiguous()

    # coarse hypotheses: observation-major, then rotation, then scale seed
    Rs = quaternion_matrices(rotation_set(n_rotations)).to(device)
    offs = torch.tensor([0.0] if rigid else [o * math.log(2.0) for o in SCALE_SEEDS], dtype=torch.float64, device=device)
    n_s = offs.numel()
    H0 = n_rotations * n_s
    sigma = (log_s0[:, None, None] + offs[None, None, :]).expand(O, n_rotations, n_s).reshape(-1)
    R = Rs[None, :, None].expand(O, n_rotations, n_s, 3, 3).reshape(-1, 3, 3)
    c_rep = c_o[:, None, None, :].expand(O, n_rotations, n_s, 3).reshape(-1, 3)
    t = c_t[None] - sigma.exp()[:, None] * torch.einsum('hij,hj->hi', R, c_rep)
    table = torch.cat([R.reshape(-1, 9), t, sigma[:, None]], 1).contiguous()
    sigma_seed = sigma.clone().contiguous()
    hyp_obs = torch.arange(O, dtype=torch.int32, device=device).repeat_interleave(H0).contiguous()

    def max_points(n_use):
        return min(max(counts_h), n_use)

    fit_scale = not rigid
    n_c = int(cs['points'])
    score, _ = search(field, grid, points, offsets, counts, unit, table, sigma_seed, hyp_obs, n_c, int(cs['iters']),
                      cs['tau'], damping, fit_scale, max_points(n_c))

    # the best top_k per observation (stable: ties by hypothesis index) go on to the fine stage
    k = min(int(fs['top_k']), H0)
    order = torch.sort(score.reshape(O, H0), dim=1, stable=True).indices[:, :k]
    pick = (order + torch.arange(O, device=device)[:, None] * H0).reshape(-1)
    table_f = table[pick].contiguous()
    seed_f = sigma_seed[pick].contiguous()
    obs_f = hyp_obs[pick].contiguous()
    n_f = int(fs['points'])
    score_f, inl_f = search(field, grid, points, offsets, counts, unit, table_f, seed_f, obs_f, n_f, int(fs['iters']),
                            fs['tau'], damping, fit_scale, max_points(n_f))
    order_f = torch.sort(score_f.reshape(O, k), dim=1, stable=True).indices
    win = order_f[:, 0] + torch.arange(O, device=device) * k
    best = table_f[win]

    poses, o = [], 0
    for n in n_obs_per_scan:
        rows = best[o:o + n]
        poses.append(ObservationPoses(n, device, R=rows[:, :9].reshape(n, 3, 3), t=rows[:, 9:12], log_scale=rows[:, 12],
                                      fit_scale=fit_scale, lr=lr))
        o += n
    if not return_stats:
        return poses

    tau1 = fs['tau'][1]
    Rf = table_f[:, :9].reshape(O, k, 3, 3)
    Rw = best[:, :9].reshape(O, 1, 3, 3)
    cos = (((Rw.transpose(-1, -2) @ Rf).diagonal(dim1=-2, dim2=-1).sum(-1) - 1) / 2).clamp(-1, 1)
    far = torch.rad2deg(torch.arccos(cos)) > RUNNER_UP_DEG
    sf = score_f.reshape(O, k)
    runner = torch.where(far, sf, torch.full_like(sf, tau1 * tau1)).min(1).values
    used = torch.clamp(counts.to(torch.float64), max=n_f)
    stats, o = [], 0
    for n in n_obs_per_scan:
        sl = slice(o, o + n)
        stats.append({'score': score_f[win[sl]], 'inlier_fraction': inl_f[win[sl]].to(torch.float64) / used[sl],
                      'runner_up': runner[sl]})
        o += n
    return poses, stats


def head_volume(decoder, lat_rep_shape=None, resolution: int = 128, mini=MINI, maxi=MAXI, device=None) -> torch.Tensor:
    """The res^3 SDF of one head (``lat_rep_shape``, default the zero code) on get_logits' grid, from the decoder's native grid
    query without the eval-mode last-point quirk (``FastEnsembleDeepSDFMirrored``, or a native ``DeepSDF``, on CUDA); on the
    CPU from the module's forward."""
    from ..models.deepSDF import DeepSDF
    from ..models.EnsembledDeepSDF import FastEnsembleDeepSDFMirrored
    from ..models.fitting import _native_npm_decoder
    from ..utils.reconstruction import create_grid_points_from_bounds
    if device is None:
        device = next(decoder.parameters()).device
    lat = (torch.zeros(1, decoder.lat_dim, device=device) if lat_rep_shape is None
           else lat_rep_shape.reshape(1, -1).to(device=device, dtype=torch.float32))
    pts = torch.from_numpy(create_grid_points_from_bounds(np.asarray(mini), np.asarray(maxi), resolution)).to(
        device=device, dtype=torch.float32).reshape(1, -1, 3)
    with torch.no_grad():
        if device.type == 'cuda':
            if isinstance(decoder, FastEnsembleDeepSDFMirrored):
                return decoder.engine().query(pts, lat, eval_quirk=False)[0].reshape(-1)
            if isinstance(decoder, DeepSDF) and _native_npm_decoder(decoder, 1):
                return decoder.engine().query(pts, lat).reshape(-1)
            raise ValueError('register_scans: %s has no native grid query (FastEnsembleDeepSDFMirrored, or a native one-output '
                             'DeepSDF on CUDA)' % type(decoder).__name__)
        from .reconstruction import _per_point, _sweep
        training = decoder.training
        decoder.train()                  # the module's eval mode applies the ensemble's last-point quirk per chunk
        try:
            values, _ = _sweep(pts, 100000, lambda p: decoder(p, _per_point(lat[None], p.shape[1]), None))
        finally:
            decoder.train(training)
        return torch.from_numpy(values).to(device)


def register_scans(decoder, scans: Sequence[Sequence[torch.Tensor]], lat_rep_shape=None, resolution: int = 128, mini=MINI,
                   maxi=MAXI, **kwargs):
    """:func:`register_observations` against one head of ``decoder``: the zero code by default (the fitters' start), or a
    known identity ``lat_rep_shape``, sampled on a ``resolution``^3 grid over [mini, maxi] (:func:`head_volume`)."""
    _check_scans(scans)
    device = scans[0][0].device
    volume = head_volume(decoder, lat_rep_shape, resolution, mini, maxi, device)
    return register_observations(volume, mini, maxi, scans, **kwargs)
