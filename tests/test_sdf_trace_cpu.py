"""The sphere tracer's contract on analytic fields, through the float64 mirror of its state machine (sdf_trace_common.py): first
hits against closed forms, grazing and empty rays, the step limit, and render.cu's pixel rays through samples_from_images."""
import numpy as np
import torch

import sdf_trace_common as T
from conftest import MAXI, MINI

BIG = ([-10.0] * 3, [10.0] * 3)


def _rays_towards(target, n=200, spread=0.05, seed=0):
    """Rays from (0, 0, 2) to points around ``target`` - unit directions."""
    rng = np.random.RandomState(seed)
    o = np.tile([0.0, 0.0, 2.0], (n, 1))
    d = np.asarray(target) + rng.uniform(-spread, spread, (n, 3)) - o
    return o, d / np.linalg.norm(d, axis=-1, keepdims=True)


def _march(field, o, u, box=BIG, scale=1.0, **kw):
    s_in, s_out = T.box_interval(o, u, np.ones(len(o)), box[0], box[1], scale, 0.1, 100.0)
    return T.march(field, o, u, s_in, s_out, scale=scale, **kw)


def test_sphere_first_hit_matches_the_closed_form():
    c, r = (0.0, 0.0, 0.0), 0.3
    for scale, step_factor in ((1.0, 0.6), (4.0, 0.6), (1.0, 1.2)):       # 1.2: overshoots, so the bracket and its refinement
        o, u = _rays_towards(np.asarray(c) / scale, spread=0.1 / scale)
        status, s, _ = _march(T.sphere(c, r), o, u, scale=scale, step_factor=step_factor, hit_eps=5e-4, max_steps=500)
        t = T.sphere_first_hit(o, u, c, r, scale)
        assert np.isfinite(t).all() and (status == T.HIT).all()
        cos = np.abs((((o + t[:, None] * u) * scale - c) * u).sum(-1)) / r        # |cos| of the incidence
        bound = 5e-4 / scale / np.maximum(cos, 0.2) + 1e-9
        assert (np.abs(s - t) <= bound).all(), float(np.abs(s - t).max())
        if step_factor > 1:
            assert np.median(np.abs(s - t)) < 1e-4                           # bracketed from 1.9 long, refined in 6 steps


def test_two_spheres_in_a_row_hit_the_nearer():
    a, b = T.sphere((0, 0, 0.5), 0.2), T.sphere((0, 0, -0.5), 0.2)
    o, u = _rays_towards((0, 0, 0), spread=0.05)
    for step_factor in (0.6, 1.2):
        status, s, _ = _march(lambda x: np.minimum(a(x), b(x)), o, u, step_factor=step_factor, max_steps=500)
        t = T.sphere_first_hit(o, u, (0, 0, 0.5), 0.2)
        assert (status == T.HIT).all() and np.abs(s - t).max() < 5e-4


def test_ray_entering_inside_finds_the_first_crossing():
    o, u = _rays_towards((0, 0, 0), n=50, spread=0.05)
    # the box starts inside the sphere of radius 1.2 around (0, 0, 1.5): the first crossing is where the ray leaves it
    status, s, _ = _march(T.sphere((0, 0, 1.5), 1.2), o, u, box=([-0.5] * 3, [0.5, 0.5, 1.0]), max_steps=500)
    oc = o - np.array([0, 0, 1.5])
    b = (oc * u).sum(-1)
    t = -b + np.sqrt(b * b - ((oc * oc).sum(-1) - 1.44))
    assert (status == T.HIT).all() and np.abs(s - t).max() < 1e-3


def test_thin_slab_is_not_skipped():
    hit_eps, step_factor = 5e-4, 0.9
    width = 2.5 * hit_eps / step_factor                                       # thicker than hit_eps / step_factor
    slab = lambda x: np.abs(x[:, 2] - 0.1) - width / 2                        # noqa: E731
    o, u = _rays_towards((0, 0, 0), spread=0.3)
    status, s, _ = _march(slab, o, u, step_factor=step_factor, hit_eps=hit_eps, max_steps=2000)
    t = (0.1 + width / 2 - o[:, 2]) / u[:, 2]
    assert (status == T.HIT).all() and np.abs(s - t).max() <= hit_eps / np.abs(u[:, 2]).min() + 1e-12


def test_grazing_and_empty_rays_are_misses():
    r, scale, hit_eps = 0.3, 1.0, 5e-4
    # rays along x that pass the sphere at 2 hit_eps above its top: they approach it, never within hit_eps, and leave the box
    o = np.array([[-1.0, 0.0, r + 2 * hit_eps + z] for z in (0.0, 1e-4, 1e-3)])
    u = np.tile([1.0, 0.0, 0.0], (3, 1))
    status, _, steps = _march(T.sphere((0, 0, 0), r), o, u, box=([-1.5] * 3, [1.5] * 3), hit_eps=hit_eps, max_steps=100000)
    assert (status == T.MISS).all() and (steps > 0).all()
    # rays that miss the box: background without a single query
    calls = []
    o = np.tile([0.0, 0.0, 2.0], (4, 1))
    u = np.array([[0, 0, 1.0], [1.0, 0, 0], [0, 1.0, 0], [0.6, 0, 0.8]])
    status, _, steps = _march(lambda x: calls.append(len(x)) or np.ones(len(x)), o, u, box=(MINI, MAXI))
    assert (status == T.MISS).all() and (steps == 0).all() and calls == []


def test_step_limit_is_reported():
    o, u = _rays_towards((0, 0, 0), n=20)
    status, _, steps = _march(T.sphere((0, 0, 0), 0.3), o, u, step_factor=0.05, max_steps=3)
    assert (status == T.OUT_OF_STEPS).all() and (steps == 3).all()


def test_invalid_samples_make_invalid_rays():
    o, u = _rays_towards((0, 0, 0), n=50)
    status, s, _ = _march(T.sphere((0, 0, 0), 0.3), o, u, max_steps=500, valid_fn=lambda x: x[:, 0] < 0.0)
    x = o + s[:, None] * u
    assert set(np.unique(status)) <= {T.HIT, T.INVALID}
    assert (x[status == T.INVALID, 0] >= 0).all() and (x[status == T.HIT, 0] < 0).all()


def test_pixel_rays_follow_the_rasterizer_and_back_project_onto_the_sphere():
    from nphm_b200.evaluation.render_utils import KK, render_cameras, samples_from_images
    H, W, scale, c, r = 160, 120, 4.0, (0.01, -0.02, 0.03), 0.35
    K = KK.astype(np.float64).copy()
    K[:2] /= 8.0                                                               # the evaluation cameras at 1/8 resolution
    cams, poses = render_cameras(3)
    o, u, cos = T.pixel_rays(poses, K, (H, W))
    # render.cu's convention: the point at eye depth 1 of pixel (r, c) projects to its centre (c + 0.5, r + 0.5)
    for v, Rt in enumerate(poses):
        e = (np.linalg.inv(Rt)[:3, :3] @ (o[v] + u[v] / cos[v][..., None] - Rt[:3, 3]).reshape(-1, 3).T).T
        assert np.allclose(-e[:, 2], 1.0)
        col = K[0, 0] * e[:, 0] / -e[:, 2] + K[0, 2] - 0.5
        row = K[1, 2] - K[1, 1] * e[:, 1] / -e[:, 2] - 0.5
        rr, cc = np.meshgrid(np.arange(H), np.arange(W), indexing='ij')
        assert np.abs(col - cc.reshape(-1)).max() < 1e-9 and np.abs(row - rr.reshape(-1)).max() < 1e-9
    o, u, cos = o.reshape(-1, 3), u.reshape(-1, 3), cos.reshape(-1)
    s_in, s_out = T.box_interval(o, u, cos, MINI, MAXI, scale, 0.1, 2.0)
    status, s, _ = T.march(T.sphere(c, r), o, u, s_in, s_out, scale=scale, max_steps=500)
    hit = status == T.HIT
    assert hit.mean() > 0.1
    depth = np.where(hit, s * cos, 0.0).astype(np.float32).reshape(3, H, W)
    x = scale * (o + s[:, None] * u)
    nrm = np.zeros((len(s), 3), np.uint8)
    nrm[hit] = T.encode_normals(x[hit] - np.asarray(c))
    pts, _ = samples_from_images(torch.from_numpy(depth), torch.from_numpy(nrm.reshape(3, H, W, 3)), cams, poses, scale, K=K,
                                 rend_size=(H, W))
    d = np.abs(np.linalg.norm(pts.numpy() - np.asarray(c), axis=-1) - r)
    # depth rounded to fp32 and its NDC value in fp32 (glcam_images): ~1e-7 relative in depth, times the NDC slope near zfar
    assert len(pts) > 0.5 * hit.sum() and d.max() < 2e-3 * scale, d.max()
