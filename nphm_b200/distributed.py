"""Multi-GPU mesh extraction: the grid is partitioned in contiguous x-slabs, one per rank (SURVEY.md 8e).

  * SDF query: every point is independent -> no collective.  A rank evaluates the planes its cells touch (its own
    cell layers, the closing plane, and one ghost cell layer below so that vertices shared with the previous rank
    resolve to that rank's ids); the <= 2 extra planes are recomputed rather than exchanged.
  * Marching cubes: one exchange step - ``all_gather`` of the per-rank (vertex, triangle) counts gives every rank the
    id base of its first vertex, so the concatenated result is IDENTICAL (ids, order, fp64 positions) to a single-GPU run.
  * The triangle / vertex buffers are collected on rank 0 in one batched point-to-point exchange (variable sizes; every
    buffer lands directly in its slice of the result).

One process per GPU, ``torch.distributed`` (NCCL on GPUs; the host logic is exercised with gloo on CPU in
tests/test_distributed_cpu.py).

The narrow band (``extract_mesh_narrowband_sharded``, DESIGN §4.16) is sharded in x-slabs of whole block layers instead:
the ranks swap the planes they share after every round of evaluation, and the ghost plane after the fill.  Its host driver
(slab plan, round loop, per-slab marching cubes) is the one of the one-GPU band in ``utils/reconstruction.py``, where the
one-GPU extraction is the one-slab case; this module adds the exchange between ranks (:class:`GroupExchange`).
"""
from __future__ import annotations

from typing import Callable, List, Optional, Tuple

import torch
import torch.distributed as dist

from .utils.reconstruction import _band_setup, _run_band, plan_block_slabs
# the band's host driver stays importable from here, where the callers of the multi-GPU band find it next to GroupExchange
from .utils.reconstruction import (LocalExchange, extract_mesh_narrowband_slabs, narrowband_slab_volumes,  # noqa: F401
                                   narrowband_slabs_mesh)


def plan_slabs(res: int, world: int) -> List[Tuple[int, int]]:
    """Cell layers [c0, c1) of each rank; res-1 cell layers split as evenly as possible (first ranks get the extra)."""
    n_layers = res - 1
    base, extra = divmod(n_layers, world)
    out, c = [], 0
    for r in range(world):
        n = base + (1 if r < extra else 0)
        out.append((c, c + n))
        c += n
    return out


def slab_planes(c0: int, c1: int) -> Tuple[int, int, bool]:
    """(first plane, number of planes, has ghost layer) a rank must evaluate for cell layers [c0, c1)."""
    if c1 <= c0:
        return c0, 0, False
    ghost = c0 > 0
    p0 = c0 - (1 if ghost else 0)
    return p0, c1 + 1 - p0, ghost


def exchange_counts(n_verts: int, n_tris: int, group=None, device='cpu') -> List[Tuple[int, int]]:
    world = dist.get_world_size(group)
    mine = torch.tensor([n_verts, n_tris], dtype=torch.int64, device=device)
    allc = [torch.zeros_like(mine) for _ in range(world)]
    dist.all_gather(allc, mine, group=group)
    return [(int(c[0]), int(c[1])) for c in allc]


def gather_mesh(verts: torch.Tensor, tris: torch.Tensor, counts: List[Tuple[int, int]], group=None, dst: int = 0):
    """Concatenate per-rank (verts (v,3) f64, tris (t,3) i64) on ``dst`` in rank order: ONE batched exchange
    (``batch_isend_irecv`` = one NCCL group): every sender posts its two buffers, ``dst`` receives each of them
    directly into its slice of the result at the prefix offset the count exchange gave (no staging buffers, no
    serial receive loop).  Returns (verts, tris) on ``dst`` and (None, None) elsewhere."""
    rank = dist.get_rank(group)
    world = dist.get_world_size(group)
    ops = []
    if rank != dst:
        if verts.shape[0]:
            ops.append(dist.P2POp(dist.isend, verts.contiguous(), dst, group))
        if tris.shape[0]:
            ops.append(dist.P2POp(dist.isend, tris.contiguous(), dst, group))
        if ops:
            for w in dist.batch_isend_irecv(ops):
                w.wait()
        return None, None
    tot_v = sum(c[0] for c in counts)
    tot_t = sum(c[1] for c in counts)
    all_v = torch.empty(tot_v, 3, dtype=verts.dtype, device=verts.device)
    all_t = torch.empty(tot_t, 3, dtype=tris.dtype, device=tris.device)
    ov = ot = 0
    for r in range(world):
        nv, nt = counts[r]
        if r == dst:
            all_v[ov:ov + nv] = verts
            all_t[ot:ot + nt] = tris
        else:
            if nv:
                ops.append(dist.P2POp(dist.irecv, all_v[ov:ov + nv], r, group))      # contiguous row slice
            if nt:
                ops.append(dist.P2POp(dist.irecv, all_t[ot:ot + nt], r, group))
        ov += nv
        ot += nt
    if ops:
        for w in dist.batch_isend_irecv(ops):
            w.wait()
    return all_v, all_t


class _Lap:
    """Device-side lap timer (CUDA events on the current stream); a no-op on CPU tensors / when disabled."""

    def __init__(self, sink: Optional[dict], device):
        self.sink = sink
        self.on = sink is not None and torch.device(device).type == 'cuda'
        self.marks = []
        if self.on:
            self.mark(None)

    def mark(self, name):
        if not self.on:
            return
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        self.marks.append((name, ev))

    def close(self):
        if not self.on:
            return
        torch.cuda.synchronize()
        for (_, a), (name, b) in zip(self.marks[:-1], self.marks[1:]):
            self.sink[name] = self.sink.get(name, 0.0) + a.elapsed_time(b)


def extract_mesh_sharded(slab_volume_fn: Callable[[int, int], torch.Tensor], res: int, iso: float = 0.0,
                         negate: bool = True, group=None,
                         mc_count: Optional[Callable] = None, mc_emit: Optional[Callable] = None,
                         timings: Optional[dict] = None):
    """Sharded ``get_logits`` + marching cubes.

    ``slab_volume_fn(first_plane, n_planes)`` returns this rank's SDF planes as a (n_planes, res, res) float32 tensor.
    ``mc_count`` / ``mc_emit`` default to the CUDA kernels (``nphm_b200._native``); tests inject CPU stand-ins.
    ``timings`` (optional dict) accumulates device milliseconds per phase: ``sdf_ms``, ``mc_count_ms``,
    ``count_exchange_ms``, ``mc_emit_ms``, ``gather_ms``, and ``gather_bytes`` (what this rank sent over NVLink).
    Returns (verts, tris) in global index units on rank 0, (None, None) elsewhere."""
    if mc_count is None or mc_emit is None:
        from . import _native
        mc_count, mc_emit = _native.marching_cubes_count, _native.marching_cubes_emit
    rank = dist.get_rank(group)
    world = dist.get_world_size(group)
    c0, c1 = plan_slabs(res, world)[rank]
    p0, n_planes, ghost = slab_planes(c0, c1)
    cuda = dist.get_backend(group) == 'nccl'
    device = torch.device('cuda', torch.cuda.current_device()) if cuda else torch.device('cpu')
    lap = _Lap(timings, device)
    if n_planes:
        vol = slab_volume_fn(p0, n_planes)
        lap.mark('sdf_ms')
        nv, nt, params, ws = mc_count(vol, iso, negate, x_global0=p0, ghost_lo=ghost)
        device = vol.device
    else:
        lap.mark('sdf_ms')
        vol, nv, nt, params, ws = None, 0, 0, None, None
    lap.mark('mc_count_ms')
    counts = exchange_counts(nv, nt, group, device=device)
    lap.mark('count_exchange_ms')
    base = sum(c[0] for c in counts[:rank])
    if n_planes:
        verts, tris = mc_emit(vol, params, ws, nv, nt, base)
    else:
        verts = torch.empty(0, 3, dtype=torch.float64, device=device)
        tris = torch.empty(0, 3, dtype=torch.int64, device=device)
    lap.mark('mc_emit_ms')
    out = gather_mesh(verts, tris, counts, group)
    lap.mark('gather_ms')
    lap.close()
    if timings is not None:
        timings['gather_bytes'] = 0 if rank == 0 else int(verts.numel() * 8 + tris.numel() * 8)
    return out


def ensemble_slab_fn(decoder, latent: torch.Tensor, mini, maxi, res: int, nbatch_points: int):
    """``slab_volume_fn`` for the identity ensemble: in-kernel grid generation over this rank's planes; the eval quirk
    follows the GLOBAL flat index so the result does not depend on the number of ranks."""
    eng = decoder.engine()

    def fn(first_plane: int, n_planes: int) -> torch.Tensor:
        period = 0 if decoder.training else int(nbatch_points)
        out, _ = eng.query_grid(latent, mini, maxi, res, first_plane * res * res, n_planes * res * res, period)
        return out.view(n_planes, res, res)

    return fn


# ------------------------------------------------------------------------------------------------------------------
# Point-sharded fitting of ONE head (north_star; SURVEY.md 8e, reference loop src/NPHM/models/fitting.py:197-279)
# ------------------------------------------------------------------------------------------------------------------
def shard_rows(n: int, world: int, rank: int) -> Tuple[int, int]:
    """Rows [lo, hi) of an n-row batch that `rank` evaluates (contiguous, as even as possible)."""
    base, extra = divmod(n, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def combine_surface_terms(grad: torch.Tensor, loss: torch.Tensor, n_kept: torch.Tensor, group=None):
    """The ONE collective of a sharded fitting iteration: all-reduce(SUM) of [n_r * grad_r (lat_dim), n_r * loss_r, n_r].
    Returns (global mean gradient, [n_kept, sum |sdf|]) - identical on every rank.  grad_r / loss_r are this rank's
    d(mean |sdf|)/d latent and mean |sdf| over ITS kept points (loss_r may be NaN when n_r = 0: it is not used then)."""
    n = n_kept.reshape(1).to(grad.dtype)
    payload = torch.cat([grad.reshape(-1) * n, torch.where(n > 0, loss.reshape(1) * n, torch.zeros_like(n)), n])
    dist.all_reduce(payload, op=dist.ReduceOp.SUM, group=group)
    total = payload[-1]
    mean_grad = torch.where(total > 0, payload[:-2] / total.clamp(min=1), torch.zeros_like(payload[:-2]))
    return mean_grad.contiguous(), torch.stack([total, payload[-2]]).contiguous()


class _NativeShardOps:
    """Per-rank surface term + replicated update on the native kernels (nphm_fit_surface_grad / nphm_fit_apply_gradient)."""

    def __init__(self, decoder, device):
        import ctypes
        from . import _native
        self._ct, self._native = ctypes, _native
        self.device = device
        self.engine = decoder.engine()
        self.latent = torch.zeros(decoder.lat_dim, device=device, dtype=torch.float32)
        self.m = torch.zeros_like(self.latent)
        self.v = torch.zeros_like(self.latent)
        self.terms = torch.zeros(8, device=device, dtype=torch.float32)
        self.grad = torch.zeros_like(self.latent)
        self.loss_terms = torch.zeros(8, device=device, dtype=torch.float32)

    def surface(self, points: torch.Tensor, clamp: float):
        pts = points.reshape(-1, 3).to(torch.float32).contiguous()
        if pts.shape[0] == 0:
            z = torch.zeros((), device=self.device)
            return torch.zeros_like(self.latent), z, z
        nat = self._native
        with torch.cuda.device(self.device):
            nat.check(nat.lib().nphm_fit_surface_grad(self.engine.handle, pts.data_ptr(), pts.shape[0], self.latent.data_ptr(),
                                                      None, float(clamp), self.terms.data_ptr(), self.grad.data_ptr(), None, None,
                                                      torch.cuda.current_stream(self.device).cuda_stream), 'nphm_fit_surface_grad')
        return self.grad, self.terms[0], self.terms[5]

    def apply(self, mean_grad, stats, lambdas, clamp, lr, step):
        nat = self._native
        fp = nat.FitParams(float(lambdas.get('surface', 0.0)), float(lambdas.get('reg_global', 0.0)),
                           float(lambdas.get('reg_loc', 0.0)), float(lambdas.get('reg_unobserved', 0.0)),
                           float(lambdas.get('symm_dist', 0.0)), float(clamp), float(lr), int(step))
        with torch.cuda.device(self.device):
            nat.check(nat.lib().nphm_fit_apply_gradient(self.engine.handle, self.latent.data_ptr(), self.m.data_ptr(),
                                                        self.v.data_ptr(), self._ct.byref(fp), mean_grad.data_ptr(),
                                                        stats.data_ptr(), None, 1, self.loss_terms.data_ptr(), None,
                                                        torch.cuda.current_stream(self.device).cuda_stream),
                      'nphm_fit_apply_gradient')


def inference_identity_space_sharded(decoder, all_obs, lambdas, n_steps, schedule_cfg, step_scale=1, lr_scale=1, group=None,
                                     ops=None):
    """``inference_identity_space`` (reference fitting.py:180-285) for ONE head with the sampled points of every iteration
    sharded over the ranks of ``group``.  Every rank runs the same loop on the same ``all_obs`` with the same seed, so the
    CPU-generator sampling stream (fitting.py:214-222) is replicated; the 5 x 1000 sampled points are split row-wise,
    every rank evaluates the clamped |sdf| term and its latent gradient on its rows, ONE all-reduce
    (:func:`combine_surface_terms`) makes the global mean gradient, and the regularisers + Adam update are applied
    identically everywhere - the latent stays bit-identical across ranks without a broadcast.  ``ops`` injects the per-rank
    kernels (tests use a CPU stand-in).  Returns ``(lat_rep_shape (1,1,D), anchors)`` like the reference."""
    from .models.fitting import _apply_schedule, _clamp_for_iteration, _sample_observations
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    device = all_obs[0].device
    if ops is None:
        ops = _NativeShardOps(decoder, device)
    lr = 0.01 * lr_scale
    z_prev = ops.latent.clone()
    for j in range(int(n_steps * step_scale)):
        lr = _apply_schedule(j, step_scale, schedule_cfg, lambdas, lr)
        obs, _ = _sample_observations(all_obs)                       # replicated: same generator state on every rank
        pts = obs.reshape(-1, 3)
        lo, hi = shard_rows(pts.shape[0], world, rank)
        clamp = _clamp_for_iteration(j, step_scale)
        z_prev.copy_(ops.latent)
        grad, loss, kept = ops.surface(pts[lo:hi], clamp)
        mean_grad, stats = combine_surface_terms(grad, loss, kept, group)
        ops.apply(mean_grad, stats, lambdas, clamp, lr, j + 1)
    with torch.no_grad():
        anchors = decoder.predict_anchors(z_prev.reshape(1, 1, -1)) if hasattr(decoder, 'predict_anchors') else None
    return ops.latent.reshape(1, 1, -1).clone().requires_grad_(True), anchors



# ------------------------------------------------------------------------------------------------------------------
# Narrow-band extraction sharded in x-slabs of block layers (DESIGN §4.16)
# ------------------------------------------------------------------------------------------------------------------
class GroupExchange:
    """This rank's slab in a ``torch.distributed`` group: planes go to the neighbouring ranks in one batched point-to-point
    exchange, "anything listed" is an all-reduce, the mesh is assembled by :func:`exchange_counts` and :func:`gather_mesh`.
    NCCL moves the device buffers directly; other backends (gloo) send and receive host copies."""

    def __init__(self, device, group=None):
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.ranks = [self.rank]
        self.device = torch.device(device)
        nccl = dist.get_backend(group) == 'nccl'
        self.wire = self.device if nccl else torch.device('cpu')      # where the buffers and collectives of the backend live

    def swap(self, sends, expects, nbytes):
        ops, recv = [], [None, None]
        for k, peer in ((0, self.rank - 1), (1, self.rank + 1)):
            if sends[0][k] is not None:
                ops.append(dist.P2POp(dist.isend, sends[0][k].to(self.wire), peer, self.group))
            if expects[0][k]:
                recv[k] = torch.empty(nbytes, dtype=torch.uint8, device=self.wire)
                ops.append(dist.P2POp(dist.irecv, recv[k], peer, self.group))
        if ops:
            for w in dist.batch_isend_irecv(ops):
                w.wait()
        return [tuple(None if r is None else r.to(self.device) for r in recv)]

    def any(self, counts) -> bool:
        flag = torch.tensor([int(any(c > 0 for c in counts))], dtype=torch.int64, device=self.wire)
        dist.all_reduce(flag, op=dist.ReduceOp.MAX, group=self.group)
        return bool(flag.item())

    def rows(self, rows):
        mine = torch.tensor(rows[0], dtype=torch.int64, device=self.wire)
        allr = [torch.zeros_like(mine) for _ in range(self.world)]
        dist.all_gather(allr, mine, group=self.group)
        return [r.tolist() for r in allr]

    def counts(self, counts):
        return exchange_counts(counts[0][0], counts[0][1], self.group, device=self.wire)

    def gather(self, parts, counts):
        verts, tris = gather_mesh(parts[0][0].to(self.wire), parts[0][1].to(self.wire), counts, self.group)
        return (None, None) if verts is None else (verts.to(self.device), tris.to(self.device))


def extract_mesh_narrowband_sharded(decoder, encoding, mini, maxi, resolution, nbatch_points=100000, block=4, margin=None, group=None,
                                    return_stats=False, sparse=False):
    """:func:`nphm_b200.utils.reconstruction.extract_mesh_narrowband` over the ranks of ``group``, one x-slab of block layers
    each (:func:`plan_block_slabs`); every rank holds only its slab's planes.  Rank 0 returns the mesh, bit for bit the one
    ``extract_mesh_narrowband`` gives with the same arguments for any world size; the other ranks return None.  Decoders
    without a native band query take the dense sharded path (:func:`extract_mesh_sharded`, NCCL).  ``return_stats``: also a
    dict with the per-rank ``blocks_active``, ``voxels_evaluated`` and ``bytes_exchanged`` (bytes each rank sent per plane
    exchange), ``growth_rounds``, the totals, the margin and the slab plan (rank 0; None elsewhere).  ``sparse``: every rank keeps its
    slab in block-sparse storage (DESIGN §4.17); the stats then give that rank's ``device_bytes``."""
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    res = int(resolution)
    device, fns, _, _ = _band_setup(decoder, encoding, mini, maxi, res, nbatch_points, block, margin)
    if fns is None:
        return _dense_sharded(decoder, encoding, mini, maxi, res, nbatch_points, group, device, return_stats)
    out = _run_band(decoder, encoding, mini, maxi, res, nbatch_points, block, margin, plan_block_slabs(res, block, world),
                    lambda plan: [plan[rank]], GroupExchange(device, group), True, sparse)
    mesh, stats = out if rank == 0 else (None, None)
    return (mesh, stats) if return_stats else mesh


def _dense_sharded(decoder, encoding, mini, maxi, res, nbatch_points, group, device, return_stats):
    from .models.reconstruction import get_logits
    from .utils.reconstruction import _device_mesh, create_grid_points_from_bounds
    if device.type != 'cuda' or dist.get_backend(group) != 'nccl':
        raise ValueError('extract_mesh_narrowband_sharded: a decoder without a native band query needs CUDA and NCCL')
    grid = torch.from_numpy(create_grid_points_from_bounds(mini, maxi, res)).to(device, dtype=torch.float32).view(res, res * res, 3)

    def slab_fn(p0, n):
        pts = grid[p0:p0 + n].reshape(1, -1, 3)
        return torch.from_numpy(get_logits(decoder, encoding, pts, nbatch_points=nbatch_points)).to(device).view(n, res, res)

    with torch.cuda.device(device):
        verts, tris = extract_mesh_sharded(slab_fn, res, group=group)
        mesh = None if verts is None else _device_mesh(verts, tris, mini, maxi, res)
    n = res ** 3
    stats = None if mesh is None else {'blocks_active': None, 'blocks_total': None, 'voxels_evaluated': n, 'voxels_total': n,
                                       'growth_rounds': 0, 'margin': None}
    return (mesh, stats) if return_stats else mesh


# Data-parallel training steps (DESIGN §6): defined in training_sharded.py, which uses shard_rows above
from .training_sharded import (LocalTrainGroup, clip_sparse_grad_norm_, shard_trainer, train_step_sharded,  # noqa: E402,F401
                               val_step_sharded)
# Many scans fitted over the ranks (DESIGN §6): defined in fitting_sharded.py
from .fitting_sharded import (FitPlan, fit_owner, inference_identity_space_batched_sharded,  # noqa: E402,F401
                              inference_iterative_root_finding_joint_batched_sharded, plan_fit_chunks)
