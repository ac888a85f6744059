#!/usr/bin/env python
"""Generate render.npz: the reference's own rendering post-processing and surface sampling (src/NPHM/evaluation/render_utils.py,
scripts/evaluation/eval.py:30-96), unmodified, on known images.

pyrender (OpenGL) is not available, so stub modules stand in for the reference's imports:
  * ``pyrender``: ``OffscreenRenderer.render`` returns the images of oracle/render_oracle.py (float64 ray caster) in pyrender's
    format - (H, W, 3) uint8 normals (the kernel's quantisation of the unit face normal) and (H, W) float32 eye depth, 0 for
    background - and ``IntrinsicsCamera.get_projection_matrix`` is pyrender's matrix restated;
  * ``pyvista``, ``tyro``, a minimal ``trimesh`` (a mesh with vertices / faces / vertex_normals / copy) and ``NPHM.*`` modules
    that eval.py imports but this part of it does not use.
numpy 2 no longer has ``np.NaN`` (render_utils.py:128); it is aliased to ``np.nan`` for the run.

Fixture: a closed, bumpy icosphere of 5120 triangles, small enough that ``gen_render_samples``' default scale (4) gives it about
50 x 50 pixels per 1280 x 960 view, and a 5023-vertex FLAME stand-in with vertex normals.  Stored: the fixture, the oracle
images of the 10 views (foreground pixels only), ``fibonacci_sphere`` / ``m3dLookAt`` / ``get_3d_points`` results,
``gen_render_samples`` and a seeded ``sample_surface_points``.  To keep the file small, exactly and verified here:
  * the fixture mesh is not stored (the images are; ``render_common.icosphere`` rebuilds it), nor are FLAME vertices that
    ``sample_surface_points`` never reads (the stand-in is zero there);
  * normals - the reference's ``uint8 / 255 * 2 - 1`` - are stored as their uint8 codes, after checking that numpy's
    ``np.arange(256) / 255 * 2 - 1`` of the codes gives the reference's arrays bit for bit;
  * of the 22 k ``gen_render_samples`` points, every count and a random 2000 rows in float64; of the seeded draws, the row
    indices into the sliced samples (checked to reproduce the reference's returned points exactly) and 200 rows in float64.
Needs a reference checkout with src/NPHM/evaluation/render_utils.py and scripts/evaluation/eval.py (one of the roots
oracle/ref_loader.py looks in):

    python tests/golden/make_golden_render.py
"""
import importlib.util
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from oracle import ref_loader as R                      # noqa: E402
from oracle import render_oracle as O                   # noqa: E402
from render_common import icosphere                     # noqa: E402

SEED = 5
NUM_SAMPS = 3000


class Mesh:
    def __init__(self, vertices, faces, vertex_normals=None):
        self.vertices = np.array(vertices, np.float64)
        self.faces = np.array(faces, np.int64)
        self.vertex_normals = vertex_normals

    def copy(self):
        return Mesh(self.vertices.copy(), self.faces.copy(), self.vertex_normals)


def _stub_pyrender():
    pr = types.ModuleType('pyrender')

    class Scene:
        def __init__(self, **kw):
            self.nodes = []

        def add(self, obj, pose=None):
            self.nodes.append((obj, pose))

    class PrMesh:
        @staticmethod
        def from_trimesh(mesh, smooth=True):
            m = PrMesh()
            m.positions = np.asarray(mesh.vertices, np.float32)        # pyrender keeps float32 positions
            m.faces = np.asarray(mesh.faces)
            return m

    class IntrinsicsCamera:
        def __init__(self, fx, fy, cx, cy, znear=0.05, zfar=None, name=None):
            self.fx, self.fy, self.cx, self.cy = float(fx), float(fy), float(cx), float(cy)
            self.znear, self.zfar = float(znear), float(zfar)

        def get_projection_matrix(self, width=None, height=None):
            width, height = float(width), float(height)
            P = np.zeros((4, 4))
            P[0][0] = 2.0 * self.fx / width
            P[1][1] = 2.0 * self.fy / height
            P[0][2] = 1.0 - 2.0 * self.cx / width
            P[1][2] = 2.0 * self.cy / height - 1.0
            P[3][2] = -1.0
            n, f = self.znear, self.zfar
            P[2][2] = (f + n) / (n - f)
            P[2][3] = (2 * f * n) / (n - f)
            return P

    class OffscreenRenderer:
        def __init__(self, viewport_width, viewport_height, point_size=1.0):
            self.W, self.H = viewport_width, viewport_height
            self._renderer = types.SimpleNamespace()

        def render(self, scene, flags=None):
            mesh = [o for o, _ in scene.nodes if isinstance(o, PrMesh)][0]
            cam, pose = [(o, p) for o, p in scene.nodes if isinstance(o, IntrinsicsCamera)][0]
            w2e = np.linalg.inv(np.asarray(pose, np.float64))[:3]
            out = O.render_view(mesh.positions, mesh.faces, w2e, (cam.fx, cam.fy, cam.cx, cam.cy), self.H, self.W, cam.znear,
                                cam.zfar)
            RENDERS.append(out)
            normals = O.quantize_normals(out['normal'])
            normals[out['tri'] < 0] = 0
            return normals, out['depth'].astype(np.float32)

        def delete(self):
            pass

    pr.Scene, pr.Mesh, pr.IntrinsicsCamera, pr.OffscreenRenderer = Scene, PrMesh, IntrinsicsCamera, OffscreenRenderer
    pr.PointLight = lambda **kw: types.SimpleNamespace(**kw)
    pr.constants = types.SimpleNamespace(RenderFlags=types.SimpleNamespace(SKIP_CULL_FACES=1))
    pr.shader_program = types.SimpleNamespace(ShaderProgram=None)
    return pr


RENDERS = []


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


RU = os.path.join('src', 'NPHM', 'evaluation', 'render_utils.py')
EVAL = os.path.join('scripts', 'evaluation', 'eval.py')
UNIT = np.arange(256) / 255 * 2 - 1


def reference_root():
    for root in R._CANDIDATES:
        if os.path.exists(os.path.join(root, RU)) and os.path.exists(os.path.join(root, EVAL)):
            return root
    raise R.ReferenceUnavailable('no reference checkout with %s and %s' % (RU, EVAL))


def codes(normals):
    """uint8 codes of reference normals (u8 / 255 * 2 - 1), checked to reproduce them exactly."""
    c = np.rint((np.asarray(normals) + 1) / 2 * 255).astype(np.uint8)
    assert np.array_equal(UNIT[c], normals)
    return c


def load_reference():
    root = reference_root()
    np.NaN = np.nan
    tm = types.ModuleType('trimesh')
    tm.Trimesh = Mesh
    tm.load = None
    for name, mod in (('pyrender', _stub_pyrender()), ('pyvista', types.ModuleType('pyvista')), ('tyro', types.ModuleType('tyro')),
                      ('trimesh', tm)):
        sys.modules[name] = mod
    for pkg in ('NPHM', 'NPHM.evaluation', 'NPHM.data'):
        sys.modules[pkg] = types.ModuleType(pkg)
    sys.modules['NPHM.evaluation.metrics'] = types.SimpleNamespace(eval_pointcloud=None)
    sys.modules['NPHM.env_paths'] = types.SimpleNamespace()
    sys.modules['NPHM'].env_paths = sys.modules['NPHM.env_paths']
    sys.modules['NPHM.data.manager'] = types.SimpleNamespace(DataManager=None)
    ru = _load('NPHM.evaluation.render_utils', os.path.join(root, RU))
    ev = _load('ref_eval', os.path.join(root, EVAL))
    return ru, ev


def flame_standin(rng):
    """5023 vertices, of which the 150 face-region ones lie around the fixture with unit vertex normals and the cut plane
    (3276, 3207, 3310) is tilted through the fixture's lower part; every other vertex is zero (never read)."""
    face_idx = np.sort(rng.choice([i for i in range(5023) if i not in (3276, 3207, 3310)], 150, replace=False))
    v, n = np.zeros((5023, 3)), np.zeros((5023, 3))
    v[face_idx] = rng.uniform(-0.1, 0.1, (150, 3))
    n[face_idx] = rng.randn(150, 3)
    n[face_idx] /= np.linalg.norm(n[face_idx], axis=1, keepdims=True)
    v[3276] = (0.0, -0.012, 0.0)
    v[3207] = (1.0, -0.012, 0.1)
    v[3310] = (0.0, -0.012 - 0.2, -1.0)
    return v, n, face_idx


def main():
    ru, ev = load_reference()
    rng = np.random.RandomState(SEED)
    verts, faces = icosphere(4, radius=0.025, bumps=0.25)
    mesh = Mesh(verts, faces)
    fib = np.array(ru.fibonacci_sphere(12))
    look = np.stack([ru.m3dLookAt(np.array(c) * 0.6, np.zeros([3]), np.array([0, 1, 0])) for c in fib[1:-1]])        # the poles look along +y

    # get_3d_points on a small synthetic NDC depth image (some texels >= 1: background)
    g_size = (24, 18)
    g_depth = rng.uniform(0.2, 1.1, g_size).astype(np.float32)
    g_K = np.array([[50, 0, 9], [0, 50, 12], [0, 0, 1]], np.float32)
    g_points = ru.get_3d_points(g_depth, g_K, look[3], rend_size=g_size)

    RENDERS.clear()
    points, normals = ru.gen_render_samples(mesh, 10)
    imgs = RENDERS[:]
    H, W = 1280, 960
    tri = np.stack([r['tri'] for r in imgs])
    fg = np.flatnonzero(tri.reshape(-1) >= 0)
    depth = np.stack([r['depth'] for r in imgs]).reshape(-1)[fg].astype(np.float32)
    qn = np.stack([O.quantize_normals(r['normal']) for r in imgs]).reshape(-1, 3)[fg]
    mesh4 = mesh.copy()
    mesh4.vertices /= 4                                  # the first view of gen_render_samples, on its scaled copy
    ndc0, nrm0 = ru.render_glcam(mesh4, ru.KK, ev.np.asarray(ru.m3dLookAt(fib[10] * 0.6, np.zeros(3), np.array([0, 1, 0]))),
                                 rend_size=(H, W))
    fg0 = fg[fg < H * W]

    fv, fn, face_idx = flame_standin(rng)
    flame = Mesh(fv, np.zeros((0, 3), np.int64), fn)
    np.random.seed(SEED)
    s_points, s_normals, s_points_face, s_normals_face = ev.sample_surface_points(mesh, flame, face_idx, NUM_SAMPS)
    # the draws as row indices: replay them on the reference's own sliced samples and check they give its returned points
    samps, samps_n = ev.slice_properly(flame, points, extra=normals)
    # restated face-region mask of eval.py:76-83 (cKDTree, float64), for a finer comparison than the draws
    from scipy.spatial import cKDTree
    d, i = cKDTree(fv[face_idx]).query(samps)
    p2p = np.abs(np.sum((samps - fv[face_idx][i]) * fn[face_idx][i], axis=-1))
    valids = (p2p <= 0.02) & (d <= 0.04)
    np.random.seed(SEED)
    s_idx = np.random.randint(0, samps.shape[0], NUM_SAMPS)
    s_idx_face = np.random.randint(0, int(valids.sum()), NUM_SAMPS)
    assert np.array_equal(samps[s_idx], s_points) and np.array_equal(samps_n[s_idx], s_normals)
    assert np.array_equal(samps[valids][s_idx_face], s_points_face) and np.array_equal(samps_n[valids][s_idx_face], s_normals_face)
    print('fixture: %d faces; %d foreground pixels over 10 views; %d samples, %d above the cut, %d in the face region'
          % (len(faces), len(fg), len(points), len(samps), int(valids.sum())))
    rows = np.sort(rng.choice(len(points), 2000, replace=False))
    glcam_rows = np.sort(rng.choice(len(fg0), 300, replace=False))
    flame_rows = np.r_[face_idx, [3276, 3207, 3310]]
    np.savez_compressed(os.path.join(HERE, 'render.npz'), fib=fib, look=look,
                        g_depth=g_depth, g_K=g_K, g_size=np.array(g_size), g_points=g_points,
                        img_shape=np.array([10, H, W]), img_index_step=np.diff(fg, prepend=0).astype(np.uint32),
                        img_depth=depth, img_normals=qn,
                        glcam_ndc=ndc0.reshape(-1)[fg0], glcam_ndc_bg=ndc0.reshape(-1)[0 if 0 not in fg0 else -1],
                        glcam_rows=glcam_rows, glcam_normals=nrm0.reshape(-1, 3)[fg0][glcam_rows],
                        n_points=np.array(len(points)), point_rows=rows, points=points[rows], normal_codes=codes(normals),
                        flame_rows=flame_rows, flame_verts=fv[flame_rows], flame_normals=fn[flame_rows], face_idx=face_idx,
                        seed=np.array(SEED), num_samps=np.array(NUM_SAMPS), valids=np.packbits(valids), n_samps=np.array(len(samps)),
                        s_idx=s_idx.astype(np.int32), s_idx_face=s_idx_face.astype(np.int32),
                        s_points=s_points[:200], s_points_face=s_points_face[:200])

if __name__ == '__main__':
    main()
