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
    if torch.cuda.is_available() and not (isinstance(logits, torch.Tensor) and logits.is_cuda):
        dev = torch.device('cuda', torch.cuda.current_device())
        vol = np.ascontiguousarray(logits, dtype=np.float32)
        v_dev, t_dev = _native.marching_cubes_device(torch.from_numpy(vol).to(dev), 0.0)
        return _device_mesh(v_dev, t_dev, mini, maxi, resolution)
    step = (np.array(maxi) - np.array(mini)) / (resolution - 1)
    vertices, triangles = marching_cubes(logits, 0.0)
    vertices = vertices * np.expand_dims(step, axis=0)
    vertices += [mini[0], mini[1], mini[2]]
    return make_mesh(vertices, triangles)


def _device_mesh(v_dev, t_dev, mini, maxi, resolution):
    """Marching-cubes output on the device (index units) -> mesh in world units, as ``mesh_from_logits`` builds it.  The
    device copy of the vertices stays with the mesh: deform_mesh() takes it instead of uploading them again."""
    dev = v_dev.device
    step = (np.array(maxi) - np.array(mini)) / (resolution - 1)
    vertices, triangles = _to_host(v_dev), _to_host(t_dev).view(np.uint64)
    dev_verts = v_dev * torch.as_tensor(step, device=dev) + torch.as_tensor(np.asarray(mini, dtype=np.float64), device=dev)
    vertices = vertices * np.expand_dims(step, axis=0)
    vertices += [mini[0], mini[1], mini[2]]
    mesh = make_mesh(vertices, triangles)
    if len(mesh.vertices) == dev_verts.shape[0]:     # trimesh's process=True may have merged vertices
        try:
            mesh._nphm_device_vertices = dev_verts.to(torch.float32)
        except AttributeError:
            pass
    return mesh


# ------------------------------------------------------------------------------------------ narrow-band extraction
def default_margin(mini, maxi, resolution, block=4):
    """Default band margin tau of :func:`extract_mesh_narrowband`: ``block * |h|`` with h the grid step of each axis, i.e. twice the
    half diagonal of a block.  The band mesh is then exact for every SDF with ``|grad sdf| <= 2`` (DESIGN §4.13)."""
    h = (np.asarray(maxi, dtype=np.float64) - np.asarray(mini, dtype=np.float64)) / (resolution - 1)
    return float(block * np.linalg.norm(h))


def narrowband_volume(evaluate, mini, maxi, resolution, device, block=4, margin=None, quirk_period=0, evaluate_quirk=None):
    """The band of :func:`extract_mesh_narrowband` for any ``evaluate(points (n, 3) float32 CUDA) -> values (n,)``.

    Evaluates the block corners, then every voxel of the blocks with a corner ``|sdf| <= margin`` or a sign change, grows the band
    until no evaluated face voxel of an inactive block disagrees with that block's fill, and fills the rest.  ``quirk_period > 0``:
    the voxels ``g % p == p - 1`` and ``g == res^3 - 1`` go to ``evaluate_quirk`` instead, and the blocks around them are active.
    Returns ``(volume (res, res, res) float32 CUDA, stats, band)`` with ``band`` the :class:`_native.NarrowBand` (block states)."""
    if quirk_period and evaluate_quirk is None:
        raise ValueError('narrowband_volume: quirk_period > 0 needs evaluate_quirk')
    res = int(resolution)
    tau = default_margin(mini, maxi, res, block) if margin is None else float(margin)
    band = _native.NarrowBand(res, block, device)
    vol = torch.empty(res ** 3, device=device, dtype=torch.float32)

    def run(n, fn):
        if n:
            band.scatter(fn(band.gather(n, mini, maxi)).reshape(-1), vol)
        return n

    evaluated = run(band.begin(int(quirk_period)), evaluate_quirk)
    evaluated += run(band.corners(), evaluate)
    evaluated += run(band.classify(tau, vol), evaluate)
    rounds = 0
    while True:
        n = band.grow(vol)
        if not n:
            break
        rounds += 1
        evaluated += run(n, evaluate)
    band.fill(vol)
    stats = {'blocks_active': int(band.active_blocks), 'blocks_total': band.blocks_per_axis ** 3,
             'voxels_evaluated': int(evaluated), 'voxels_total': res ** 3, 'growth_rounds': rounds, 'margin': tau}
    return vol.view(res, res, res), stats, band


def _band_evaluators(decoder, encoding, device):
    """(evaluate, evaluate_quirk | None) for the decoders whose native query gives every point a value independent of the other
    points of its call, or None (then the caller extracts densely)."""
    from ..models.EnsembledDeepSDF import FastEnsembleDeepSDFMirrored
    from ..models.deepSDF import DeepSDF
    if device.type != 'cuda':
        return None
    if isinstance(decoder, FastEnsembleDeepSDFMirrored):
        engine = decoder.engine()
        lat = encoding.reshape(1, -1).to(device)

        def query(pts, quirk):
            sdf, _ = engine.query(pts[None], lat, eval_quirk=quirk, quirk_period=1 if quirk else None)
            return sdf.reshape(-1)
        return (lambda pts: query(pts, False)), (lambda pts: query(pts, True))
    if isinstance(decoder, DeepSDF) and decoder.out_dim_net == 1:
        code = encoding.reshape(1, 1, -1).to(device)
        with torch.no_grad():
            if not decoder._fused_ok(torch.zeros(1, 1, 3, device=device), code):
                return None

        def evaluate(pts):
            return decoder(pts[None], code.expand(1, pts.shape[0], code.shape[-1]), None)[0].reshape(-1)
        return evaluate, None
    return None


def extract_mesh_narrowband(decoder, encoding, mini, maxi, resolution, nbatch_points=100000, block=4, margin=None,
                            return_stats=False):
    """The mesh of ``mesh_from_logits(get_logits(decoder, encoding, grid, nbatch_points), mini, maxi, resolution)`` for the grid
    of ``create_grid_points_from_bounds(mini, maxi, resolution)``, with the decoder evaluated only in a band of ``block^3``-cell
    blocks around the surface (DESIGN §4.13): the same vertex ids, float64 positions and triangles whenever every piece of the
    surface inside a block outside the band reaches one of its faces, which ``margin`` (SDF units, default
    :func:`default_margin`; ``inf`` evaluates every voxel) guarantees for ``|grad sdf| <= 2 margin / (block |h|)``.

    Takes ``FastEnsembleDeepSDFMirrored`` (honouring ``decoder.training`` like ``get_logits``: in eval mode the voxels of
    ``get_logits``' last-point-of-chunk quirk are evaluated with it) and one-output ``DeepSDF`` stacks on the native query;
    other decoders and CPU devices take ``get_logits`` + ``mesh_from_logits``.  ``return_stats``: also return a dict with
    ``blocks_active``, ``voxels_evaluated`` and ``growth_rounds`` (and the totals and the margin used)."""
    from ..models.reconstruction import get_logits
    device = next(decoder.parameters()).device
    fns = _band_evaluators(decoder, encoding, device)
    if fns is None:
        grid = torch.from_numpy(create_grid_points_from_bounds(mini, maxi, resolution)).to(device, dtype=torch.float32)
        mesh = mesh_from_logits(get_logits(decoder, encoding, grid[None], nbatch_points=nbatch_points), mini, maxi, resolution)
        n = int(resolution) ** 3
        stats = {'blocks_active': None, 'blocks_total': None, 'voxels_evaluated': n, 'voxels_total': n, 'growth_rounds': 0,
                 'margin': None}
        return (mesh, stats) if return_stats else mesh
    evaluate, evaluate_quirk = fns
    quirk_period = 0 if (decoder.training or evaluate_quirk is None) else int(nbatch_points)
    with torch.no_grad(), torch.cuda.device(device):
        vol, stats, _ = narrowband_volume(evaluate, mini, maxi, resolution, device, block=block, margin=margin,
                                          quirk_period=quirk_period, evaluate_quirk=evaluate_quirk)
        v_dev, t_dev = _native.marching_cubes_device(vol, 0.0, negate=True)     # == mesh_from_logits' negation, bit for bit
        mesh = _device_mesh(v_dev, t_dev, mini, maxi, resolution)
    return (mesh, stats) if return_stats else mesh
