"""Shared by the registration tests (test_register_cpu.py, test_gpu_register.py): analytic SDF volumes (an asymmetric smooth
union of three ellipsoids, and an ellipsoid of revolution as the ambiguous case), surface points and one-sided patches of them,
uniform random similarities, and the composed-transform error of test_gpu_pose.py::test_recovers_a_known_similarity."""
import math

import numpy as np
import torch

from conftest import MAXI, MINI

# (centre, radii): distinct axes and off-axis centres, so no rotation or reflection maps the union onto itself
ASYMMETRIC = [((0.0, 0.1, -0.3), (0.30, 0.38, 0.33)),
              ((0.12, 0.28, -0.05), (0.10, 0.13, 0.20)),
              ((-0.08, -0.18, -0.22), (0.22, 0.10, 0.16))]
REVOLUTION = [((0.0, 0.1, -0.3), (0.25, 0.40, 0.25))]       # symmetric about the y axis

# a small NPM DeepSDF whose zero-code head is ASYMMETRIC (tests/golden/make_golden_register_head.py -> register_head.npz)
HEAD_CONFIG = dict(lat_dim=8, hidden_dim=64, nlayers=6, geometric_init=True, radius_init=0.35)


def fitted_head(device):
    """The DeepSDF fitted to the asymmetric analytic head at the zero code: a distance-like decoder head."""
    from conftest import load_golden
    from nphm_b200.models.deepSDF import DeepSDF
    g = load_golden('register_head.npz')
    dec = DeepSDF(**HEAD_CONFIG)
    dec.load_state_dict({k: torch.from_numpy(g[k]) for k in g.files})
    return dec.to(device)


def _ellipsoid(x, centre, radii):
    r = torch.tensor(radii, dtype=x.dtype, device=x.device)
    y = (x - torch.tensor(centre, dtype=x.dtype, device=x.device)) / r
    return (y.norm(dim=-1) - 1.0) * float(min(radii))


def analytic_sdf(parts, x, k=0.05):
    """Smooth union (polynomial smin, width k) of the ellipsoids ``parts`` at ... x 3 points."""
    d = _ellipsoid(x, *parts[0])
    for part in parts[1:]:
        e = _ellipsoid(x, *part)
        h = (0.5 + 0.5 * (e - d) / k).clamp(0.0, 1.0)
        d = e + (d - e) * h - k * h * (1.0 - h)
    return d


def volume(parts, res, device='cpu'):
    """res^3 fp32 SDF on get_logits' grid over [MINI, MAXI] (x slowest, z fastest, end points included)."""
    ax = [torch.linspace(MINI[a], MAXI[a], res, dtype=torch.float64) for a in range(3)]
    X = torch.stack(torch.meshgrid(*ax, indexing='ij'), -1).reshape(-1, 3)
    return analytic_sdf(parts, X).float().to(device)


def surface_points(parts, n, seed):
    """n x 3 float64 points on the zero level set (Newton projection from jittered points of the near-surface shell) and
    their unit normals."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(40 * n, 3, generator=g, dtype=torch.float64)
    x = torch.tensor(MINI, dtype=torch.float64) + x * (torch.tensor(MAXI, dtype=torch.float64) - torch.tensor(MINI, dtype=torch.float64))
    keep = analytic_sdf(parts, x).abs() < 0.1
    x = x[keep][:n]
    assert x.shape[0] == n
    for _ in range(20):
        x = x.detach().requires_grad_(True)
        f = analytic_sdf(parts, x)
        (gr,) = torch.autograd.grad(f.sum(), [x])
        x = x - (f / gr.square().sum(-1).clamp_min(1e-12))[:, None] * gr
    x = x.detach().requires_grad_(True)
    (gr,) = torch.autograd.grad(analytic_sdf(parts, x).sum(), [x])
    assert float(analytic_sdf(parts, x.detach()).abs().max()) < 1e-8
    return x.detach(), gr / gr.norm(dim=-1, keepdim=True)


def patch(points, normals, seed, n, max_angle=70.0):
    """Up to n points whose normals lie within ``max_angle`` degrees of a random view direction (one-sided)."""
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(3, generator=g, dtype=torch.float64)
    v = v / v.norm()
    sel = points[(normals @ v) > math.cos(math.radians(max_angle))]
    return sel[:n]


def random_similarity(rng, max_trans=0.5, scale_range=(0.5, 2.0)):
    """A uniform random rotation, a translation uniform in the ball of radius max_trans and a log-uniform scale:
    (R 3 x 3, t 3, log scale), float64, the transform model -> scan."""
    q = rng.randn(4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    R = torch.tensor([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                      [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                      [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]], dtype=torch.float64)
    d = rng.randn(3)
    t = torch.tensor(d / np.linalg.norm(d) * max_trans * rng.uniform() ** (1 / 3), dtype=torch.float64)
    ls = rng.uniform(math.log(scale_range[0]), math.log(scale_range[1]))
    return R, t, ls


def to_scan(x, R, t, ls):
    """Model points -> the scan frame of the similarity (R, t, log scale)."""
    return math.exp(ls) * x @ R.T + t


def pose_error(poses, o, R, t, ls):
    """(degrees, translation, |scale - 1|) of the pose of observation o composed with the applied similarity (model -> scan):
    the identity when the pose inverts it."""
    A = torch.eye(4, dtype=torch.float64)
    A[:3, :3], A[:3, 3] = math.exp(ls) * R, t
    E = poses.matrices()[o].cpu() @ A
    s = E[:3, :3].det().abs() ** (1 / 3)
    ang = math.degrees(math.acos(max(-1.0, min(1.0, (float((E[:3, :3] / s).trace()) - 1) / 2))))
    return ang, float(E[:3, 3].norm()), abs(float(s) - 1)
