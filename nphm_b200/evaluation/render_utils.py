"""Drop-in mirror of the reference's ``NPHM.evaluation.render_utils`` (src/NPHM/evaluation/render_utils.py) without OpenGL.

  * ``render_glcam``        :26-89    pyrender's offscreen render -> ``nphm_render_depth_normals`` (csrc/render.cu)
  * ``get_3d_points``       :92-107
  * ``unproject_points``    :110-130
  * ``m3dLookAt``           :134-148
  * ``fibonacci_sphere``    :151-166
  * ``gen_render_samples``  :169-201  all N views in ONE native call

Same names, signatures and numpy return types.  Rasterization is native (CUDA only, no fallback); everything after it is
float64 torch code that runs on CPU or CUDA tensors alike and repeats the reference's arithmetic step for step:
  * depth 0 (background) -> inf, then NDC z = (zfar + znear - 2 znear zfar / depth) / (zfar - znear) in float32, as numpy 2
    evaluates the reference's expression on pyrender's float32 depth; normals = uint8 / 255 * 2 - 1 in float64;
  * ``unproject_points`` maps pixel indices to NDC with ``/ (W - 1)`` and ``/ (H - 1)`` (not pixel centres), as the reference
    does, and points with NDC z >= 1 become NaN;
  * ``gen_render_samples`` orders the points of a view column-major (k = c H + r), drops back faces (angle < -0.01 against the
    stored, quantized normals) and keeps the reference's view order, so that index draws into its output pick the same points.
Meshes are anything with ``.vertices`` and ``.faces`` (``SimpleMesh``, ``trimesh.Trimesh``); a path goes to ``trimesh.load``
when trimesh is installed.  What this cannot reproduce - pyrender's multisampling - is described in DESIGN.md §4.12.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from .. import _native

KK = np.array([
    [2440, 0, 480],
    [0, 2440, 640],
    [0, 0, 1]], dtype=np.float32)

_UNIT_NORMAL = np.arange(256) / 255 * 2 - 1            # the reference's normals / 255 * 2 - 1 of every uint8 (float64)


def _device():
    if not torch.cuda.is_available():
        raise _native.NativeError('nphm_b200.evaluation.render_utils renders on a CUDA device (no CPU fallback)')
    return torch.device('cuda', torch.cuda.current_device())


def _load(model_in):
    if isinstance(model_in, str):
        try:
            import trimesh
        except ImportError:
            raise ValueError('loading %r needs trimesh, which is not installed; pass a mesh with .vertices and .faces' % model_in)
        return trimesh.load(model_in, process=False)
    return model_in


def projection_matrix(fx, fy, cx, cy, width, height, znear, zfar):
    """pyrender ``IntrinsicsCamera(fx, fy, cx, cy, znear, zfar).get_projection_matrix(width, height)`` (float64)."""
    fx, fy, cx, cy, width, height = float(fx), float(fy), float(cx), float(cy), float(width), float(height)
    P = np.zeros((4, 4))
    P[0][0] = 2.0 * fx / width
    P[1][1] = 2.0 * fy / height
    P[0][2] = 1.0 - 2.0 * cx / width
    P[1][2] = 2.0 * cy / height - 1.0
    P[3][2] = -1.0
    P[2][2] = (zfar + znear) / (znear - zfar)
    P[2][3] = (2 * zfar * znear) / (znear - zfar)
    return P


def render_views(vertices, faces, poses, K, rend_size, znear=0.1, zfar=2.0, device=None):
    """Native render of one mesh into len(poses) views in one call: vertices (n, 3) float32, faces (m, 3), poses camera-to-world
    4 x 4 (the reference's ``Rt``), K 3 x 3.  Returns ``(depth (V, H, W) float32 eye depth, 0 = background; normals (V, H, W, 3)
    uint8)``, CUDA tensors - pyrender's two outputs for each view."""
    dev = device or _device()
    v = torch.as_tensor(np.asarray(vertices, np.float32)).to(dev)
    f = torch.as_tensor(np.asarray(faces, np.int64)).to(dev)
    w2e = np.stack([np.linalg.inv(np.asarray(Rt, np.float64))[:3, :4] for Rt in poses])
    k = np.asarray(K, np.float64)
    intr = np.tile(np.array([k[0][0], k[1][1], k[0][2], k[1][2]]), (len(poses), 1))
    depth, normals, _ = _native.render_depth_normals(v, f, torch.from_numpy(w2e), torch.from_numpy(intr), rend_size[0], rend_size[1],
                                                     znear, zfar)
    return depth, normals


def glcam_images(depth, normals_u8, znear=0.1, zfar=2.0):
    """The post-processing of ``render_glcam`` on pyrender-format images (torch, any device): ``(NDC depth float32, normals
    float64)``."""
    f32 = lambda x: torch.tensor(x, dtype=torch.float32, device=depth.device)     # noqa: E731  numpy 2: python scalars -> float32
    d = torch.where(depth == 0, torch.full_like(depth, float('inf')), depth)
    ndc = (f32(zfar + znear) - f32(2.0 * znear * zfar) / d) / f32(zfar - znear)
    # a table of the 256 values (numpy's arithmetic): torch on CUDA divides by a scalar through its reciprocal, one ulp off
    return ndc, torch.from_numpy(_UNIT_NORMAL).to(depth.device)[normals_u8.long()]


def _unproject(rows, cols, z, rend_size, P, Rt):
    """unproject_points on torch tensors: pixel rows / columns (float64), NDC depth z -> world points, NaN where z >= 1."""
    z = z.to(torch.float64)
    x = cols / (rend_size[1] - 1) * 2 - 1
    y = -(rows / (rend_size[0] - 1) * 2 - 1)
    points = torch.stack([x, y, z, torch.ones_like(z)], dim=1)
    clipping_to_world = torch.from_numpy(np.matmul(np.asarray(Rt, np.float64), np.linalg.inv(P))).to(z.device)
    points = points @ clipping_to_world.T
    points = (points / points[:, 3:4])[:, :3]
    return torch.where((z >= 1)[:, None], torch.full_like(points, float('nan')), points)


def _points_image(ndc, K, Rt, rend_size, znear, zfar):
    """get_3d_points on a torch NDC depth image: (W H, 3) float64 in the reference's column-major order."""
    H, W = rend_size
    dev = ndc.device
    P = projection_matrix(K[0][0], K[1][1], K[0][2], K[1][2], W, H, znear, zfar)
    rows = torch.arange(H, dtype=torch.float64, device=dev).repeat(W)
    cols = torch.arange(W, dtype=torch.float64, device=dev).repeat_interleave(H)
    return _unproject(rows, cols, ndc.T.reshape(-1), rend_size, P, Rt)


def samples_from_images(depth, normals_u8, cam_origins, poses, scale, K=KK, rend_size=(1280, 960), znear=0.1, zfar=2.0):
    """Everything ``gen_render_samples`` does after rendering, on pyrender-format images depth (V, H, W) float32 and normals
    (V, H, W, 3) uint8 (torch, any device): ``(points, normals)`` float64 tensors."""
    all_points, all_normals = [], []
    for i, cam in enumerate(cam_origins):
        ndc, nrm = glcam_images(depth[i], normals_u8[i], znear, zfar)
        points3d = _points_image(ndc, K, poses[i], rend_size, znear, zfar)
        valid = ~torch.isnan(points3d).any(dim=-1)
        points3d = points3d[valid]
        nrm = nrm.permute(1, 0, 2).reshape(-1, 3)[valid]
        ray_dir = points3d - torch.from_numpy(np.array(cam) * 0.6).to(points3d.device)
        ray_dir = ray_dir / torch.linalg.norm(ray_dir, dim=-1, keepdim=True)
        front = (ray_dir * nrm).sum(dim=-1) < -0.01
        all_points.append(points3d[front])
        all_normals.append(nrm[front])
    return torch.cat(all_points) * scale, torch.cat(all_normals)


def render_glcam(model_in, K, Rt, rend_size=(512, 512), znear=0.1, zfar=2.0):
    """(NDC depth (H, W) float32, world-space normals (H, W, 3) float64) of one view, as the reference returns them."""
    mesh = _load(model_in)
    depth, normals = render_views(mesh.vertices, mesh.faces, [Rt], K, rend_size, znear, zfar)
    ndc, nrm = glcam_images(depth[0], normals[0], znear, zfar)
    return ndc.cpu().numpy(), nrm.cpu().numpy()


def get_3d_points(depth, K, Rt, rend_size=(512, 512), normals=None, znear=0.1, zfar=2.0):
    """Back-projection of every pixel of an NDC depth image: (W H, 3) float64, column-major, NaN where depth >= 1."""
    ndc = depth if isinstance(depth, torch.Tensor) else torch.from_numpy(np.asarray(depth))
    return _points_image(ndc, K, Rt, rend_size, znear, zfar).cpu().numpy()


def unproject_points(ppos, depth, rend_size, K, Rt):
    """Pixel indices ppos (n, 2) = (row, column) of an NDC depth image -> world points; K is the 4 x 4 projection matrix.
    Clips ``ppos`` in place, as the reference does."""
    ppos[:, 0] = np.clip(ppos[:, 0], 0, rend_size[0])
    ppos[:, 1] = np.clip(ppos[:, 1], 0, rend_size[1])
    rows = torch.from_numpy(np.asarray(ppos[:, 0], np.float64))
    cols = torch.from_numpy(np.asarray(ppos[:, 1], np.float64))
    z = torch.from_numpy(np.asarray(depth)[ppos[:, 0], ppos[:, 1]])
    return _unproject(rows, cols, z, rend_size, K, Rt).numpy()


def m3dLookAt(eye, target, up):
    mz = (eye - target)
    mz /= np.linalg.norm(mz, keepdims=True)  # inverse line of sight
    mx = np.cross(up, mz)
    mx /= np.linalg.norm(mx, keepdims=True)
    my = np.cross(mz, mx)
    my /= np.linalg.norm(my)
    return np.array([[mx[0], my[0], mz[0], eye[0]],
                     [mx[1], my[1], mz[1], eye[1]],
                     [mx[2], my[2], mz[2], eye[2]],
                     [0, 0, 0, 1]])


def fibonacci_sphere(samples=1000):
    points = []
    phi = math.pi * (math.sqrt(5.) - 1.)  # golden angle in radians
    for i in range(samples):
        y = 1 - (i / float(samples - 1)) * 2  # y goes from 1 to -1
        radius = math.sqrt(1 - y * y)
        theta = phi * i
        points.append((math.cos(theta) * radius, y, math.sin(theta) * radius))
    return points


def render_cameras(N):
    """The N camera origins (unit sphere) and camera-to-world poses of ``gen_render_samples``, in its order."""
    cams = fibonacci_sphere(N + 2)[1:-1]
    cams.reverse()
    poses = [m3dLookAt(np.array(c) * 0.6, np.zeros([3]), np.array([0, 1, 0])) for c in cams]
    return cams, poses


def gen_render_samples(m, N, scale=4):
    """Surface samples of a mesh from N views at 1280 x 960: ``(points (n, 3), normals (n, 3))`` float64 numpy arrays."""
    mesh = _load(m)
    vertices = (np.array(mesh.vertices, dtype=np.float64) / scale).astype(np.float32)
    cams, poses = render_cameras(N)
    depth, normals = render_views(vertices, mesh.faces, poses, KK, (1280, 960))
    points, nrm = samples_from_images(depth, normals, cams, poses, scale)
    return points.cpu().numpy(), nrm.cpu().numpy()


from .sdf_render import render_sdf_views  # noqa: E402,F401  (sphere-traced images of SDF heads in this module's format)
