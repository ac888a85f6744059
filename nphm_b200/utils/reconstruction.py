"""Drop-in mirror of the reference module ``NPHM.utils.reconstruction``.

  * ``create_grid_points_from_bounds``  src/NPHM/utils/reconstruction.py:5-20
  * ``mesh_from_logits``                src/NPHM/utils/reconstruction.py:22-37  (mcubes.marching_cubes -> the
    sm_90a marching-cubes kernels of ``nphm_b200/csrc/marching_cubes.cu``)
"""
from __future__ import annotations

import numpy as np
import torch

from .. import _native
from .mesh import make_mesh


def create_grid_points_from_bounds(minimun, maximum, res, scale=None):
    """(res^3, 3) float64 grid, x slowest / z fastest, end points included."""
    if scale is not None:
        res = int(scale * res)
        minimun = scale * minimun
        maximum = scale * maximum
    axes = [np.linspace(minimun[a], maximum[a], res) for a in range(3)]
    pts = np.empty((res, res, res, 3), dtype=np.float64)
    pts[..., 0] = axes[0][:, None, None]
    pts[..., 1] = axes[1][None, :, None]
    pts[..., 2] = axes[2][None, None, :]
    return pts.reshape(-1, 3)


def marching_cubes(volume, isovalue=0.0):
    """== ``mcubes.marching_cubes(volume, isovalue)`` on the GPU: (verts (V,3) float64 in index units,
    tris (T,3) uint64).  Accepts a numpy array (host round trip through torch's pinned staging and caching
    allocator) or a CUDA tensor."""
    if isinstance(volume, torch.Tensor) and volume.is_cuda:
        v, t = _native.marching_cubes_device(volume.float(), isovalue)
        return v.cpu().numpy(), t.cpu().numpy().view(np.uint64)
    vol = np.ascontiguousarray(volume, dtype=np.float32)
    if vol.ndim != 3:
        raise ValueError('marching_cubes expects a 3-D volume')
    if torch.cuda.is_available():
        dev = torch.device('cuda', torch.cuda.current_device())
        v, t = _native.marching_cubes_device(torch.from_numpy(vol).to(dev), isovalue)
        return _to_host(v), _to_host(t).view(np.uint64)
    return _native.marching_cubes_host(vol, isovalue)          # raises: there is no CPU fallback


def _to_host(t: torch.Tensor) -> np.ndarray:
    """Device tensor -> numpy through a pinned buffer of torch's caching host allocator."""
    if t.numel() == 0:
        return t.cpu().numpy()
    out = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
    out.copy_(t, non_blocking=True)
    torch.cuda.current_stream(t.device).synchronize()
    return out.numpy()


def mesh_from_logits(logits, mini, maxi, resolution):
    """SDF volume -> mesh.  Like the reference, NEGATES ``logits`` in place (caller's array), extracts the 0
    level set of ``-sdf``, and maps index units to world units with ``step = (maxi-mini)/(resolution-1)``."""
    logits = np.reshape(logits, (resolution,) * 3)
    logits *= -1
    step = (np.array(maxi) - np.array(mini)) / (resolution - 1)
    dev_verts = None
    if torch.cuda.is_available() and not (isinstance(logits, torch.Tensor) and logits.is_cuda):
        # keep the device copy of the vertices: deform_mesh() takes it from the mesh instead of uploading them again
        dev = torch.device('cuda', torch.cuda.current_device())
        vol = np.ascontiguousarray(logits, dtype=np.float32)
        v_dev, t_dev = _native.marching_cubes_device(torch.from_numpy(vol).to(dev), 0.0)
        vertices, triangles = _to_host(v_dev), _to_host(t_dev).view(np.uint64)
        dev_verts = v_dev * torch.as_tensor(step, device=dev) + torch.as_tensor(np.asarray(mini, dtype=np.float64), device=dev)
    else:
        vertices, triangles = marching_cubes(logits, 0.0)
    vertices = vertices * np.expand_dims(step, axis=0)
    vertices += [mini[0], mini[1], mini[2]]
    mesh = make_mesh(vertices, triangles)
    if dev_verts is not None and len(mesh.vertices) == dev_verts.shape[0]:     # trimesh's process=True may have merged vertices
        try:
            mesh._nphm_device_vertices = dev_verts.to(torch.float32)
        except AttributeError:
            pass
    return mesh
