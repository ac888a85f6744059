"""Drop-in mirror of the reference module ``NPHM.utils.reconstruction``.

  * ``create_grid_points_from_bounds``  src/NPHM/utils/reconstruction.py:5-20
  * ``mesh_from_logits``                src/NPHM/utils/reconstruction.py:22-37  (mcubes.marching_cubes -> the
    sm_90a marching-cubes kernels of ``nphm_b200/csrc/marching_cubes.cu``)
"""
from __future__ import annotations

from typing import Callable, List, Optional, Tuple

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


def plan_block_slabs(res: int, block: int, world: int) -> List[Tuple[int, int]]:
    """Block layers [l0, l1) of each rank: the ceil((res-1)/block) layers split as evenly as possible (first ranks get the extra),
    so that every slab boundary is a block face; ranks past the number of layers get an empty range."""
    n_layers = -(-(int(res) - 1) // int(block))
    base, extra = divmod(n_layers, world)
    out, c = [], 0
    for r in range(world):
        n = base + (1 if r < extra else 0)
        out.append((c, c + n))
        c += n
    return out


class LocalExchange:
    """Every slab of one grid, driven by this process in rank order: planes move between the entries of the slab list and the
    collectives reduce over it.  Lets one process (one device, or the CPU oracle) run the protocol of every rank in lockstep;
    with one slab it is the one-GPU band, and nothing moves."""

    def __init__(self, n_slabs: int):
        self.ranks = list(range(n_slabs))

    def swap(self, sends, expects, nbytes):
        """sends[i] = (buffer to the lower, to the upper neighbour) of slab i; expects[i] = (from the lower, from the upper)."""
        return [(sends[i - 1][1] if lo else None, sends[i + 1][0] if hi else None) for i, (lo, hi) in enumerate(expects)]

    def any(self, counts) -> bool:
        return any(c > 0 for c in counts)

    def rows(self, rows):
        return [list(r) for r in rows]

    def counts(self, counts):
        return list(counts)

    def gather(self, parts, counts):
        if len(parts) == 1:                            # one slab: its mesh as it is, without a device copy
            return parts[0]
        return torch.cat([v for v, _ in parts]), torch.cat([t for _, t in parts])


def narrowband_slab_volumes(slabs, evaluate, mini, maxi, tau: float, exchange, quirk_period: int = 0, evaluate_quirk=None):
    """The band of :func:`extract_mesh_narrowband` on x-slabs for any ``evaluate(points (n, 3) float32 CUDA) -> values (n,)``.
    ``slabs``: the slabs this process drives (:class:`_native.NarrowBand`, or None for a rank without block layers), in the order
    of ``exchange.ranks``.

    Evaluates the block corners, then every voxel of the blocks with a corner ``|sdf| <= tau`` or a sign change, grows the band
    until no evaluated face voxel of an inactive block disagrees with that block's fill, and fills the rest.  ``quirk_period > 0``:
    the voxels ``g % p == p - 1`` and ``g == res^3 - 1`` go to ``evaluate_quirk`` instead, and the blocks around them are active.
    Every round: list, gather / evaluate / scatter, swap the planes shared with the neighbours, growth check, and ask the exchange
    whether any slab listed anything.  After the last round: fill, then hand each slab its neighbour's filled ghost plane.
    Returns ``(volumes, stats)``: one ``(n_planes, res, res)`` volume per slab (None for None), ``stats`` with ``growth_rounds``
    and, per slab, ``blocks_active``, ``voxels_evaluated`` and ``bytes_sent`` (one entry per plane exchange)."""
    if quirk_period and evaluate_quirk is None:
        raise ValueError('narrowband_slab_volumes: quirk_period > 0 needs evaluate_quirk')
    vols = [None if s is None else s.volume() for s in slabs]
    evaluated = [0] * len(slabs)
    sent = [[] for _ in slabs]
    nbytes = next((s.plane_bytes for s in slabs if s is not None), 0)

    def run(ns, fn):
        for i, (s, n) in enumerate(zip(slabs, ns)):
            if n:
                s.scatter(fn(s.gather(n, mini, maxi)).reshape(-1), vols[i])
                evaluated[i] += n

    def swap(plane_lo, plane_hi, ghost):
        sends, expects = [], []
        for s, v in zip(slabs, vols):
            if s is None:
                sends.append((None, None))
                expects.append((False, False))
                continue
            lo, hi = s.l0 > 0, s.x1 < s.res - 1
            sends.append((s.export(plane_lo(s), v) if lo and not ghost else None, s.export(plane_hi(s), v) if hi else None))
            expects.append((lo, hi and not ghost))
        got = exchange.swap(sends, expects, nbytes)
        for i, (s, v) in enumerate(zip(slabs, vols)):
            sent[i].append(sum(nbytes for b in sends[i] if b is not None))
            if s is None:
                continue
            if got[i][0] is not None:
                s.import_(s.x0 - 1 if ghost else s.x0, got[i][0], v)
            if got[i][1] is not None:
                s.import_(s.x1, got[i][1], v)

    ns = [0 if s is None else s.begin(quirk_period) for s in slabs]
    if quirk_period:
        run(ns, evaluate_quirk)
    run([0 if s is None else s.corners() for s in slabs], evaluate)
    run([0 if s is None else s.classify(tau, v) for s, v in zip(slabs, vols)], evaluate)
    swap(lambda s: s.x0, lambda s: s.x1, ghost=False)
    rounds = 0
    while True:
        ns = [0 if s is None else s.grow(v) for s, v in zip(slabs, vols)]
        if not exchange.any(ns):
            break
        rounds += 1
        run(ns, evaluate)
        swap(lambda s: s.x0, lambda s: s.x1, ghost=False)
    for s, v in zip(slabs, vols):
        if s is not None:
            s.fill(v)
    swap(None, lambda s: s.x1 - 1, ghost=True)
    stats = {'growth_rounds': rounds, 'blocks_active': [0 if s is None else int(s.active_blocks) for s in slabs],
             'voxels_evaluated': evaluated, 'bytes_sent': sent}
    return vols, stats


def _slab_mesh(slabs, vols, exchange, mc_count, mc_emit, device):
    """mc_count -> exchange.counts -> mc_emit -> exchange.gather over the filled slab volumes: (verts, tris) in global index units,
    ids as on one GPU, on rank 0 (None, None elsewhere)."""
    local, params = [], []
    for s, v in zip(slabs, vols):
        if s is None:
            local.append((0, 0))
            params.append(None)
            continue
        nv, nt, p, ws = mc_count(v, 0.0, True, x_global0=s.first_plane, ghost_lo=s.ghost)
        local.append((nv, nt))
        params.append((p, ws))
    counts = exchange.counts(local)
    parts = []
    for i, (s, v) in enumerate(zip(slabs, vols)):
        if s is None:
            parts.append((torch.empty(0, 3, dtype=torch.float64, device=device), torch.empty(0, 3, dtype=torch.int64, device=device)))
            continue
        base = sum(c[0] for c in counts[:exchange.ranks[i]])
        parts.append(mc_emit(v, params[i][0], params[i][1], local[i][0], local[i][1], base))
    return exchange.gather(parts, counts)


def narrowband_slabs_mesh(slabs, evaluate, mini, maxi, res: int, block: int, tau: float, exchange, quirk_period: int = 0,
                          evaluate_quirk=None, mc_count: Optional[Callable] = None, mc_emit: Optional[Callable] = None,
                          device='cpu'):
    """:func:`narrowband_slab_volumes` + the sharded marching cubes.  Returns ``(verts, tris, stats)`` with the mesh in global
    index units on the process that holds rank 0 (None elsewhere) and ``stats`` for every rank of the grid.  ``mc_count`` /
    ``mc_emit`` default to the CUDA kernels; tests inject CPU stand-ins, as for
    :func:`nphm_b200.distributed.extract_mesh_sharded`."""
    if mc_count is None or mc_emit is None:
        mc_count, mc_emit = _native.marching_cubes_count, _native.marching_cubes_emit
    vols, st = narrowband_slab_volumes(slabs, evaluate, mini, maxi, tau, exchange, quirk_period, evaluate_quirk)
    verts, tris = _slab_mesh(slabs, vols, exchange, mc_count, mc_emit, device)
    rows = exchange.rows([[a, e] + b for a, e, b in zip(st['blocks_active'], st['voxels_evaluated'], st['bytes_sent'])])
    nb = -(-(res - 1) // block)
    stats = {'blocks_active': [r[0] for r in rows], 'blocks_total': nb ** 3, 'voxels_evaluated': [r[1] for r in rows],
             'voxels_total': res ** 3, 'growth_rounds': st['growth_rounds'], 'bytes_exchanged': [r[2:] for r in rows],
             'margin': tau}
    return verts, tris, stats


def _band_class(sparse: bool):
    return _native.SparseNarrowBand if sparse else _native.NarrowBand


def _mc_pair(sparse: bool):
    """(mc_count, mc_emit) of :func:`_slab_mesh` for the band's storage."""
    if sparse:
        return _native.sparse_marching_cubes_count, _native.sparse_marching_cubes_emit
    return _native.marching_cubes_count, _native.marching_cubes_emit


def narrowband_volume(evaluate, mini, maxi, resolution, device, block=4, margin=None, quirk_period=0, evaluate_quirk=None,
                      sparse=False):
    """:func:`narrowband_slab_volumes` on the whole grid, one slab, for any ``evaluate(points (n, 3) float32 CUDA) -> values (n,)``
    with ``tau = margin`` (default :func:`default_margin`).  Returns ``(volume (res, res, res) float32 CUDA, stats, band)`` with
    ``band`` the :class:`_native.NarrowBand` (block states).  ``sparse``: the band is a :class:`_native.SparseNarrowBand` and
    ``volume`` is the band's brick store (``band.dense_volume()`` materialises it)."""
    res = int(resolution)
    tau = default_margin(mini, maxi, res, block) if margin is None else float(margin)
    band = _band_class(sparse)(res, block, device)
    (vol,), st = narrowband_slab_volumes([band], evaluate, mini, maxi, tau, LocalExchange(1), quirk_period, evaluate_quirk)
    stats = {'blocks_active': st['blocks_active'][0], 'blocks_total': band.blocks_per_axis ** 3,
             'voxels_evaluated': st['voxels_evaluated'][0], 'voxels_total': res ** 3, 'growth_rounds': st['growth_rounds'],
             'margin': tau}
    return vol, stats, band


def _heads_evaluators(decoder, codes, device):
    """(evaluate, evaluate_quirk | None) on ``S x n x 3`` points -> ``S x n`` values, head h under ``codes[h]`` (``codes`` S x D),
    for the decoders whose native query gives every point a value independent of the other points and heads of its call: one
    ``nphm_ensemble_query`` with S latents, or one ``nphm_mlp_query`` with S condition rows.  None for the other decoders (then the
    caller extracts densely)."""
    from ..models.EnsembledDeepSDF import FastEnsembleDeepSDFMirrored
    from ..models.deepSDF import DeepSDF
    if device.type != 'cuda':
        return None
    S = codes.shape[0]
    if isinstance(decoder, FastEnsembleDeepSDFMirrored):
        engine = decoder.engine()
        lat = codes.reshape(S, -1).to(device)

        def query(pts, quirk):
            sdf, _ = engine.query(pts, lat, eval_quirk=quirk, quirk_period=1 if quirk else None)
            return sdf.reshape(S, -1)
        return (lambda pts: query(pts, False)), (lambda pts: query(pts, True))
    if isinstance(decoder, DeepSDF) and decoder.out_dim_net == 1:
        code = codes.reshape(S, 1, -1).to(device)
        with torch.no_grad():
            if not decoder._fused_ok(torch.zeros(S, 1, 3, device=device), code):
                return None

        def evaluate(pts):
            return decoder(pts, code.expand(S, pts.shape[1], code.shape[-1]), None)[0].reshape(S, -1)
        return evaluate, None
    return None


def _band_evaluators(decoder, encoding, device):
    """:func:`_heads_evaluators` of one code, on ``(n, 3)`` points -> ``(n,)`` values."""
    fns = _heads_evaluators(decoder, encoding.reshape(1, -1), device)
    if fns is None:
        return None
    return tuple(None if f is None else (lambda pts, f=f: f(pts[None]).reshape(-1)) for f in fns)


def extract_mesh_narrowband(decoder, encoding, mini, maxi, resolution, nbatch_points=100000, block=4, margin=None,
                            return_stats=False, sparse=False):
    """The mesh of ``mesh_from_logits(get_logits(decoder, encoding, grid, nbatch_points), mini, maxi, resolution)`` for the grid
    of ``create_grid_points_from_bounds(mini, maxi, resolution)``, with the decoder evaluated only in a band of ``block^3``-cell
    blocks around the surface (DESIGN §4.13): the same vertex ids, float64 positions and triangles whenever every piece of the
    surface inside a block outside the band reaches one of its faces, which ``margin`` (SDF units, default
    :func:`default_margin`; ``inf`` evaluates every voxel) guarantees for ``|grad sdf| <= 2 margin / (block |h|)``.

    Takes ``FastEnsembleDeepSDFMirrored`` (honouring ``decoder.training`` like ``get_logits``: in eval mode the voxels of
    ``get_logits``' last-point-of-chunk quirk are evaluated with it) and one-output ``DeepSDF`` stacks on the native query;
    other decoders and CPU devices take ``get_logits`` + ``mesh_from_logits``.  ``return_stats``: also return a dict with
    ``blocks_active``, ``voxels_evaluated`` and ``growth_rounds`` (and the totals and the margin used).

    ``sparse=True`` keeps the band in block-sparse storage (DESIGN §4.17): device memory follows the active blocks instead of the
    grid, for grids up to 6497 points per axis with 4^3-cell blocks (8192 with larger blocks), and the mesh and stats are the same; the stats then also give
    ``device_bytes``, the band's workspace and brick pool and the largest marching-cubes chunk."""
    from ..models.reconstruction import get_logits
    device, fns, quirk_period, tau = _band_setup(decoder, encoding, mini, maxi, resolution, nbatch_points, block, margin)
    if fns is None:
        grid = torch.from_numpy(create_grid_points_from_bounds(mini, maxi, resolution)).to(device, dtype=torch.float32)
        mesh = mesh_from_logits(get_logits(decoder, encoding, grid[None], nbatch_points=nbatch_points), mini, maxi, resolution)
        n = int(resolution) ** 3
        stats = {'blocks_active': None, 'blocks_total': None, 'voxels_evaluated': n, 'voxels_total': n, 'growth_rounds': 0,
                 'margin': None}
        return (mesh, stats) if return_stats else mesh
    with torch.no_grad(), torch.cuda.device(device):
        vol, stats, band = narrowband_volume(fns[0], mini, maxi, resolution, device, block=block, margin=tau,
                                             quirk_period=quirk_period, evaluate_quirk=fns[1], sparse=sparse)
        verts, tris = _slab_mesh([band], [vol], LocalExchange(1), *_mc_pair(sparse), device)
        mesh = _device_mesh(verts, tris, mini, maxi, resolution)
    if sparse:
        stats['device_bytes'] = _sparse_bytes(band)
    return (mesh, stats) if return_stats else mesh


def _band_setup(decoder, encoding, mini, maxi, resolution, nbatch_points, block, margin):
    """(device, evaluators | None, quirk period, tau) of extract_mesh_narrowband for this decoder."""
    device = next(decoder.parameters()).device
    fns = _band_evaluators(decoder, encoding, device)
    quirk_period = 0 if (fns is None or decoder.training or fns[1] is None) else int(nbatch_points)
    tau = default_margin(mini, maxi, resolution, block) if margin is None else float(margin)
    return device, fns, quirk_period, tau


def _sparse_bytes(band):
    """Device bytes of a sparse band: {'band': workspace and brick pool, 'mc': the largest marching-cubes chunk}."""
    return {'band': band.device_bytes(), 'mc': band.mc_bytes}


def _run_band(decoder, encoding, mini, maxi, resolution, nbatch_points, block, margin, slab_plan, pick, exchange, return_stats,
              sparse=False):
    res = int(resolution)
    device, fns, quirk_period, tau = _band_setup(decoder, encoding, mini, maxi, res, nbatch_points, block, margin)
    if fns is None:
        raise ValueError('extract_mesh_narrowband_slabs: the decoder has no native band query on %s' % device)
    with torch.no_grad(), torch.cuda.device(device):
        slabs = [None if l1 <= l0 else _band_class(sparse)(res, block, device, l0, l1) for l0, l1 in pick(slab_plan)]
        mc_count, mc_emit = _mc_pair(sparse)
        verts, tris, stats = narrowband_slabs_mesh(slabs, fns[0], mini, maxi, res, block, tau, exchange, quirk_period, fns[1],
                                                   mc_count=mc_count, mc_emit=mc_emit, device=device)
        mesh = None if verts is None else _device_mesh(verts, tris, mini, maxi, res)
    stats['slabs'] = slab_plan
    if sparse:
        stats['device_bytes'] = [None if s is None else _sparse_bytes(s) for s in slabs]
    return (mesh, stats) if return_stats else mesh


def extract_mesh_narrowband_slabs(decoder, encoding, mini, maxi, resolution, world: int, nbatch_points=100000, block=4, margin=None,
                                  return_stats=False, sparse=False):
    """What :func:`nphm_b200.distributed.extract_mesh_narrowband_sharded` computes on ``world`` ranks, with every slab on the
    decoder's device in this process (:class:`LocalExchange`): the protocol of every rank in lockstep, on one GPU.  ``sparse``: each
    slab in block-sparse storage, as in :func:`extract_mesh_narrowband` (``device_bytes`` per slab in the stats)."""
    res = int(resolution)
    return _run_band(decoder, encoding, mini, maxi, res, nbatch_points, block, margin, plan_block_slabs(res, block, world),
                     lambda plan: plan, LocalExchange(world), return_stats, sparse)


# ------------------------------------------------------------------------------------------ many heads in one band run
PAD_ROWS = 128                    # the head-major rows of a round are padded to a multiple of one decoder tile


def pad_rows(counts, multiple: int = PAD_ROWS) -> int:
    """Rows per head of a round in which the heads listed ``counts`` voxels: the largest count rounded up to ``multiple``."""
    m = max(int(c) for c in counts)
    return -(-m // multiple) * multiple


def split_heads(flat: torch.Tensor, counts) -> List[torch.Tensor]:
    """The parts of ``flat`` (rows one head after the other) with ``counts[h]`` rows each."""
    out, c = [], 0
    for n in counts:
        out.append(flat[c:c + int(n)])
        c += int(n)
    return out


def plan_head_chunks(n_heads: int, bytes_per_head: int, budget_bytes: int, max_heads: Optional[int] = None) -> List[Tuple[int, int]]:
    """Heads ``[h0, h1)`` of each chunk, in order: as many heads per chunk as ``budget_bytes`` holds at ``bytes_per_head`` (at least
    one, at most ``max_heads``), every chunk that size but the last."""
    per = max(1, int(budget_bytes) // max(int(bytes_per_head), 1))
    if max_heads is not None:
        if int(max_heads) < 1:
            raise ValueError('max_heads must be >= 1 (got %r)' % (max_heads,))
        per = min(per, int(max_heads))
    return [(h, min(h + per, n_heads)) for h in range(0, n_heads, per)]


def _as_codes(encodings) -> torch.Tensor:
    """``S x D`` tensor or a list of codes (any shape of D elements each) -> ``S x D``."""
    if isinstance(encodings, torch.Tensor):
        if encodings.dim() < 1 or encodings.shape[0] == 0:
            raise ValueError('extract_meshes_narrowband: no latent codes')
        return encodings.reshape(encodings.shape[0], -1)
    codes = [torch.as_tensor(e).reshape(-1) for e in encodings]
    if not codes:
        raise ValueError('extract_meshes_narrowband: no latent codes')
    widths = sorted({c.numel() for c in codes})
    if len(widths) > 1:
        raise ValueError('extract_meshes_narrowband: the codes have different widths %s' % widths)
    return torch.stack([c.to(codes[0].device) for c in codes])


def narrowband_heads_volumes(bands, evaluate, mini, maxi, tau: float, quirk_period: int = 0, evaluate_quirk=None):
    """:func:`narrowband_slab_volumes` on the whole grid for the S heads of ``bands`` (a :class:`_native.NarrowBandHeads`) in
    lockstep, with ``evaluate(points S x n_pad x 3 float32 CUDA) -> values S x n_pad``: the same steps in the same order, each one
    launch sequence and one count read-back for all heads, and one evaluation per round for all heads that listed something.  A
    round's rows are padded to :func:`pad_rows` of its counts.  The band runs until no head's growth step lists anything; a head
    that has closed lists nothing in the later rounds, so each head's volume is the one its single band gives.  Returns
    ``(volumes (S, res, res, res), stats)``: per head ``blocks_active``, ``voxels_evaluated``, ``growth_rounds`` (the rounds in
    which it listed voxels) and ``padded_rows`` (rows evaluated on its behalf beyond its count)."""
    if quirk_period and evaluate_quirk is None:
        raise ValueError('narrowband_heads_volumes: quirk_period > 0 needs evaluate_quirk')
    S = bands.n_heads
    vols = bands.volumes()
    evaluated, padded, rounds = [0] * S, [0] * S, [0] * S

    def run(ns, fn):
        if not any(ns):
            return
        n_pad = pad_rows(ns)
        bands.scatter(fn(bands.gather(n_pad, mini, maxi)), vols)
        for h, n in enumerate(ns):
            evaluated[h] += n
            padded[h] += n_pad - n

    ns = bands.begin(quirk_period)
    if quirk_period:
        run(ns, evaluate_quirk)
    run(bands.corners(), evaluate)
    run(bands.classify(tau, vols), evaluate)
    while True:
        ns = bands.grow(vols)
        if not any(ns):
            break
        for h, n in enumerate(ns):
            rounds[h] += n > 0
        run(ns, evaluate)
    bands.fill(vols)
    stats = [{'blocks_active': int(bands.active_blocks[h]), 'voxels_evaluated': evaluated[h], 'growth_rounds': rounds[h],
              'padded_rows': padded[h]} for h in range(S)]
    return vols, stats


def _device_meshes(verts, tris, counts, mini, maxi, resolution):
    """:func:`_device_mesh` of each head's part of :meth:`_native.NarrowBandHeads.marching_cubes`, with one host copy for all."""
    dev = verts.device
    step = (np.array(maxi) - np.array(mini)) / (resolution - 1)
    v_host, t_host = _to_host(verts), _to_host(tris).view(np.uint64)
    dev_verts = verts * torch.as_tensor(step, device=dev) + torch.as_tensor(np.asarray(mini, dtype=np.float64), device=dev)
    nv, nt = [c[0] for c in counts], [c[1] for c in counts]
    meshes = []
    for v, t, dv in zip(np.split(v_host, np.cumsum(nv)[:-1]), np.split(t_host, np.cumsum(nt)[:-1]), split_heads(dev_verts, nv)):
        vertices = v * np.expand_dims(step, axis=0)
        vertices += [mini[0], mini[1], mini[2]]
        mesh = make_mesh(vertices, t)
        if len(mesh.vertices) == dv.shape[0]:
            try:
                mesh._nphm_device_vertices = dv.to(torch.float32)
            except AttributeError:
                pass
        meshes.append(mesh)
    return meshes


def extract_meshes_narrowband(decoder, encodings, mini, maxi, resolution, nbatch_points=100000, block=4, margin=None,
                              return_stats=False, max_heads=None, sparse=False):
    """The meshes of ``extract_mesh_narrowband(decoder, encodings[h], ...)`` for S latent codes of one decoder in one band run
    (DESIGN §4.18): every step of the band one launch sequence and one read-back for all heads, each round one decoder query for
    all heads, and one marching-cubes count and emit for all.  Head h's mesh is bit for bit the single-head one (vertex ids,
    float64 positions, triangles), and so the dense ``mesh_from_logits(get_logits(...))`` mesh whenever that one is.

    ``encodings``: an ``S x D`` tensor or a list of codes.  ``decoder.training`` is honoured as in :func:`extract_mesh_narrowband`.
    Heads run in chunks of as many as half the free device memory holds, at :meth:`_native.NarrowBandHeads.device_bytes_per_head`
    plus 16 bytes of query rows per voxel, and at most ``max_heads``; chunking changes no mesh.
    Returns the list of S meshes, and with ``return_stats`` also the list of S stats dicts of :func:`extract_mesh_narrowband`, each
    with ``padded_rows``, the rows evaluated on the head's behalf beyond its voxels (0 when nothing is padded).  Decoders or
    devices without a native band query extract head by head with :func:`extract_mesh_narrowband`.

    ``sparse=True`` runs the heads in the block-sparse band of S heads (:class:`_native.SparseNarrowBandHeads`, DESIGN §4.21):
    each head's mesh and band stats are those of ``extract_mesh_narrowband(..., sparse=True)``, and ``device_bytes`` gives the
    memory of the chunk that ran the head (``'band'``, ``'mc'``, and its number of ``'heads'``).  Chunks are planned at
    :meth:`_native.SparseNarrowBandHeads.device_bytes_per_head` plus 16 bytes of query rows per voxel of that head's starting pool;
    a band that outgrows those pools (a field whose band covers much of the grid) may need a smaller ``max_heads``, and a chunk
    whose pools cannot grow raises."""
    codes = _as_codes(encodings)
    S, res = codes.shape[0], int(resolution)
    device = next(decoder.parameters()).device
    fns = _heads_evaluators(decoder, codes[:1], device)
    if fns is None:
        meshes, stats = [], []
        for h in range(S):
            m, st = extract_mesh_narrowband(decoder, codes[h:h + 1], mini, maxi, res, nbatch_points=nbatch_points, block=block,
                                            margin=margin, return_stats=True, sparse=sparse)
            meshes.append(m)
            stats.append(dict(st, padded_rows=0))
        return (meshes, stats) if return_stats else meshes
    quirk_period = 0 if (decoder.training or fns[1] is None) else int(nbatch_points)
    tau = default_margin(mini, maxi, res, block) if margin is None else float(margin)
    meshes, stats = _heads_meshes(lambda h0, h1: _heads_evaluators(decoder, codes[h0:h1], device), S, mini, maxi, res, block, tau,
                                  quirk_period, device, max_heads, sparse)
    return (meshes, stats) if return_stats else meshes


def _heads_chunk_bytes(res: int, block: int, sparse: bool) -> int:
    """Device bytes one head of a chunk is planned at: its band and marching-cubes scratch plus 16 bytes of query rows per voxel it
    may evaluate (the whole grid for dense storage, the voxels of its starting brick pool for sparse storage)."""
    if not sparse:
        return _native.NarrowBandHeads.device_bytes_per_head(res, block) + 16 * res ** 3
    slots = _native.SparseNarrowBandHeads.default_slots(res, block)
    return _native.SparseNarrowBandHeads.device_bytes_per_head(res, block, slots) + 16 * slots * block ** 3


def _heads_meshes(evaluators, S, mini, maxi, res, block, tau, quirk_period, device, max_heads, sparse):
    """The S meshes and stats of the head-batched band, in chunks of as many heads as half the free device memory holds at
    :func:`_heads_chunk_bytes` (at most ``max_heads``); ``evaluators(h0, h1)`` gives (evaluate, evaluate_quirk) of heads
    [h0, h1)."""
    budget = torch.cuda.mem_get_info(device)[0] // 2
    meshes, stats = [], []
    with torch.no_grad(), torch.cuda.device(device):
        for h0, h1 in plan_head_chunks(S, _heads_chunk_bytes(res, block, sparse), budget, max_heads):
            ev, evq = evaluators(h0, h1)
            bands = (_native.SparseNarrowBandHeads if sparse else _native.NarrowBandHeads)(res, block, device, h1 - h0)
            vols, st = narrowband_heads_volumes(bands, ev, mini, maxi, tau, quirk_period, evq)
            verts, tris, counts = bands.marching_cubes(vols)
            del vols
            meshes += _device_meshes(verts, tris, counts, mini, maxi, res)
            nb = bands.blocks_per_axis
            stats += [{'blocks_active': s['blocks_active'], 'blocks_total': nb ** 3, 'voxels_evaluated': s['voxels_evaluated'],
                       'voxels_total': res ** 3, 'growth_rounds': s['growth_rounds'], 'margin': tau, 'padded_rows': s['padded_rows']}
                      for s in st]
            if sparse:
                used = {'band': bands.device_bytes(), 'mc': bands.mc_bytes, 'heads': h1 - h0}
                for s in stats[h0 - h1:]:
                    s['device_bytes'] = dict(used)
            del bands
    return meshes, stats


# ------------------------------------------------------------------------------------------ posed meshes
def extract_posed_meshes_narrowband(decoder_shape, decoder_expr, lat_rep_shape, lat_reps_expr, mini, maxi, resolution,
                                    nbatch_points=100000, block=4, margin=None, return_stats=False, max_heads=None, sparse=False):
    """The posed meshes ``mesh_from_logits(get_logits_posed(decoder_shape, decoder_expr, lat_rep_shape, lat_reps_expr, grid,
    nbatch_points)[s], mini, maxi, resolution)`` of the S expression codes (``(S, E)``, ``(S, 1, E)`` or ``(E,)``), bit for bit
    (vertex ids, float64 positions, triangles), from the head-batched narrow band of :func:`extract_meshes_narrowband` with the
    posed query as its evaluator: the expressions are the heads, and every round runs one native posed query for all of them
    (:func:`nphm_b200.models.reconstruction.posed_evaluator`).

    The band is exact when every piece of the posed surface inside a block outside the band reaches one of its faces.  The
    default ``margin`` (:func:`default_margin`) guarantees that for a posed field with ``|grad| <= 2``; the posed field's
    gradient is ``grad sdf(xc) (I + dF_ex/dx)^-1`` at the root, so a deformation that compresses space raises it above the
    identity SDF's, and ``margin`` (SDF units) is the override for such fields.  Decoders or devices without the native posed
    query take the dense ``get_logits_posed`` and ``mesh_from_logits``.  ``return_stats``: also the S stats dicts of
    :func:`extract_meshes_narrowband`.  ``sparse=True``: the expressions are the heads of the block-sparse band of S heads (DESIGN
    §4.21), whose memory follows the band instead of the grid, as in :func:`extract_meshes_narrowband`; the meshes are the same."""
    from ..models.EnsembledDeepSDF import FastEnsembleDeepSDFMirrored
    from ..models.reconstruction import _expression_codes, get_logits_posed, posed_evaluator
    codes, _ = _expression_codes(lat_reps_expr)
    S, res = codes.shape[0], int(resolution)
    device = next(decoder_shape.parameters()).device
    fn = posed_evaluator(decoder_shape, decoder_expr, lat_rep_shape, codes[:1])
    if fn is None:
        grid = torch.from_numpy(create_grid_points_from_bounds(mini, maxi, res)).to(device, dtype=torch.float32)
        logits = get_logits_posed(decoder_shape, decoder_expr, lat_rep_shape, codes, grid[None], nbatch_points=nbatch_points)
        meshes = [mesh_from_logits(logits[s], mini, maxi, res) for s in range(S)]
        n = res ** 3
        stats = [{'blocks_active': None, 'blocks_total': None, 'voxels_evaluated': n, 'voxels_total': n, 'growth_rounds': 0,
                  'margin': None, 'padded_rows': 0} for _ in range(S)]
        return (meshes, stats) if return_stats else meshes
    quirk = not decoder_shape.training and isinstance(decoder_shape, FastEnsembleDeepSDFMirrored)
    quirk_period = int(nbatch_points) if quirk else 0
    tau = default_margin(mini, maxi, res, block) if margin is None else float(margin)

    def evaluators(h0, h1):
        fn = posed_evaluator(decoder_shape, decoder_expr, lat_rep_shape, codes[h0:h1])
        return (lambda pts: fn(pts)[0]), ((lambda pts: fn(pts, quirk=True)[0]) if quirk else None)
    meshes, stats = _heads_meshes(evaluators, S, mini, maxi, res, block, tau, quirk_period, device, max_heads, sparse)
    return (meshes, stats) if return_stats else meshes
