"""Meshes and cameras shared by the rendering tests, tools/bench_render.py and tests/golden/make_golden_render.py."""
import numpy as np


def icosphere(level, radius=1.0, bumps=0.0, center=(0.0, 0.0, 0.0)):
    """Closed, consistently wound icosphere (20 * 4^level faces); ``bumps`` > 0 modulates the radius so that views occlude."""
    t = (1.0 + 5 ** 0.5) / 2
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t), (t, 0, -1), (t, 0, 1),
         (-t, 0, -1), (-t, 0, 1)]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6), (7, 1, 8),
         (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7), (9, 8, 1)]
    v = [np.array(p, np.float64) / np.linalg.norm(p) for p in v]
    for _ in range(level):
        mid, nf = {}, []

        def m(a, b):
            key = (min(a, b), max(a, b))
            if key not in mid:
                p = v[a] + v[b]
                v.append(p / np.linalg.norm(p))
                mid[key] = len(v) - 1
            return mid[key]
        for a, b, c in f:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        f = nf
    v = np.array(v)
    if bumps:
        v = v * (1 + bumps * np.sin(5 * v[:, 0]) * np.cos(4 * v[:, 1] + 1) * np.sin(3 * v[:, 2] + 0.5))[:, None]
    return v * radius + np.asarray(center), np.array(f, np.int64)


def look_at_views(cams, distance=0.6):
    """world-to-eye (V, 3, 4) of the camera poses ``m3dLookAt(cam * distance, 0, +y)`` (render_utils.render_cameras)."""
    from nphm_b200.evaluation.render_utils import m3dLookAt
    return np.stack([np.linalg.inv(m3dLookAt(np.array(c) * distance, np.zeros(3), np.array([0, 1, 0])))[:3] for c in cams])


def intrinsics_for(H, W, V, f_scale=1.0):
    """KK of render_utils rescaled to an H x W image (cx, cy at the centre), repeated for V views: (V, 4) fx fy cx cy."""
    s = W / 960.0 * f_scale
    return np.tile(np.array([2440.0 * s, 2440.0 * s, W / 2.0, H / 2.0]), (V, 1))


def adversarial_scene(obj_v, obj_f, dist=0.6):
    """The object in front of a full-viewport quad, plus the awkward cases of a rasterizer, all for a camera at (0, 0, dist)
    looking down -z: a triangle crossing the near plane, one beyond zfar, one behind the eye, zero-area triangles (repeated
    vertex, collinear), both windings, and coplanar duplicates (same vertices, and separately stored copies)."""
    V = [np.asarray(obj_v, np.float64)]
    F = [np.asarray(obj_f, np.int64)]
    n = len(V[0])

    def add(verts, faces):
        nonlocal n
        V.append(np.asarray(verts, np.float64)); F.append(np.asarray(faces, np.int64) + n); n += len(verts)
    z_back = dist - 1.5                                               # depth 1.5 < zfar = 2
    add([(-5, -5, z_back), (5, -5, z_back), (5, 5, z_back), (-5, 5, z_back)], [(0, 1, 2), (0, 2, 3)])     # full viewport
    add([(-0.02, -0.03, dist - 0.05), (0.03, -0.02, dist + 0.2), (0.0, 0.04, dist - 0.3)], [(0, 1, 2)])   # crosses znear
    add([(-0.3, -0.3, dist - 2.5), (0.3, -0.3, dist - 2.5), (0.0, 0.3, dist - 2.5)], [(0, 1, 2)])         # beyond zfar
    add([(-0.1, -0.1, dist + 0.5), (0.1, -0.1, dist + 0.5), (0.0, 0.1, dist + 0.5)], [(0, 1, 2)])         # behind the eye
    add([(0.0, 0.0, 0.0625), (0.0625, 0.03125, 0.0625), (0.03125, 0.015625, 0.0625)], [(0, 0, 1), (0, 1, 2)])  # zero area
    quad = [(-0.09, 0.05, 0.06), (-0.05, 0.05, 0.06), (-0.05, 0.09, 0.07), (-0.09, 0.09, 0.07)]
    add(quad, [(0, 1, 2), (0, 2, 3), (2, 1, 0), (0, 2, 3)])                                               # both windings, duplicate
    add(quad, [(0, 2, 3), (3, 2, 0)])                                                                     # stored copies
    return np.concatenate(V), np.concatenate(F)
