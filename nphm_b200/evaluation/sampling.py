"""Mirror of the surface sampling of the evaluation protocol (scripts/evaluation/eval.py:30-96).

  * ``slice_properly``         eval.py:30-57  cut at the plane through FLAME vertices 3276, 3207, 3310 (0.003 margin)
  * ``sample_surface_points``  eval.py:61-96  render samples -> slice -> face region -> two ``np.random.randint`` draws

The cKDTree query of the face-region filter runs as ``nphm_nearest_neighbors`` on the GPU; the distance of each sample to the
vertex it picks is then taken in float64, as cKDTree reports it, so the filter only differs from the reference where two
vertices tie to within fp32 round-off.  The draws run in the reference's order, so a seeded run picks the same points.
"""
from __future__ import annotations

import numpy as np
import torch

from .. import _native
from . import render_utils

FLAME_PLANE_IDS = (3276, 3207, 3310)


def slice_properly(regi, surf_points, extra=None):
    v = np.asarray(regi.vertices)
    v1, v2, v3 = (v[i, :].copy() for i in FLAME_PLANE_IDS)
    normal = np.cross(v2 - v1, v3 - v1)
    angle = np.sum(normal * (surf_points - v1), axis=-1)
    above = angle > 0.003  # a bit of margin to exclude the bottom of the reconstructed mesh
    if extra is not None:
        extra = extra[above]
    return surf_points[above], extra


def face_region_mask(samps, mesh_flame, face_idx, threshold=0.02, threshold_point2point=0.04):
    """Samples within ``threshold`` of the tangent plane of, and ``threshold_point2point`` of, their nearest face-region vertex."""
    face_vertices = np.array(np.asarray(mesh_flame.vertices)[face_idx, :])
    dev = render_utils._device()
    _, nn_idx = _native.nearest_neighbors(torch.from_numpy(np.ascontiguousarray(samps, np.float32)).to(dev),
                                          torch.from_numpy(np.ascontiguousarray(face_vertices, np.float32)).to(dev))
    nn_idx = nn_idx.cpu().numpy()
    nn_vertices = face_vertices[nn_idx, :]
    nn_normals = np.asarray(mesh_flame.vertex_normals)[face_idx, :][nn_idx, :]
    dist = np.linalg.norm(samps - nn_vertices, axis=-1)
    point2plane_distance = np.abs(np.sum((samps - nn_vertices) * nn_normals, axis=-1))
    return (point2plane_distance <= threshold) & (dist <= threshold_point2point)


def sample_surface_points(mesh, mesh_flame, face_idx, num_samps):
    """-> (points, normals, points_face, normals_face): ``num_samps`` draws from all samples above the cut, and from those in
    the face region."""
    samps, samps_normals = render_utils.gen_render_samples(mesh, 10)
    samps, samps_normals = slice_properly(mesh_flame, samps, extra=samps_normals)
    valids = face_region_mask(samps, mesh_flame, face_idx)
    samps_face = samps[valids, :]
    samps_normals_face = samps_normals[valids, :]
    random_idx = np.random.randint(0, samps.shape[0], num_samps)
    random_idx_face = np.random.randint(0, samps_face.shape[0], num_samps)
    return samps[random_idx, :], samps_normals[random_idx, :], samps_face[random_idx_face, :], samps_normals_face[random_idx_face, :]
