"""Fitting many scans on several GPUs: the scan-batched fitters of ``nphm_b200.models.fitting`` over the ranks of a
``torch.distributed`` group (DESIGN §6).

The subjects are cut into consecutive chunks of ``batch_size`` (:func:`plan_fit_chunks`).  The cut depends on the subject
list and ``batch_size`` only, never on the world size, because a subject's batched result depends on its batch: the ensemble
kernel's cost model splits a tile's members over CTAs at S = 1 and keeps whole tiles at larger S, so the same scan fitted in
batches of different sizes differs in the last bits.  With a fixed cut every subject's result is what one process gets from
``inference_*_batched`` on that subject's chunk, for any world size: every step of the batched fitters receives the same
inputs bit for bit.  (The results are bitwise equal where the fit is deterministic, as on the CPU; the native fitting kernels
sum gradients with float atomics, so two runs of the same batched call on the GPU already differ in the last bits.)  Chunks
go to ranks by longest-processing-time greedy.  One call:

  1. one all-gather of a digest of the arguments (subject count, every observation's point count, ``n_steps``, ``step_scale``,
     ``batch_size``, ``lambdas``): ranks called with different arguments all raise ``ValueError``;
  2. every rank walks ``_sampling_plan`` over all subjects (the index draws only): it gives each subject's generator and
     leaves torch's global CPU generator where the sequential loop leaves it;
  3. the rank fits its chunks, each from its own copy of ``lambdas``, each subject drawing from its own generator; where no
     batched fitter takes the decoder, the single-subject function runs per subject from that subject's generator state;
  4. the rank's results go into ONE flat float64 bucket (float32 and float64 results both travel exactly) whose length the plan
     fixes, so no count is exchanged; one all-gather, and every rank rebuilds the whole list in subject order.

The caller's ``lambdas`` ends as one single-subject call leaves it, as with the batched functions.  A rank without a chunk
still walks the generator and joins both collectives.
"""
from __future__ import annotations

import hashlib
import math
import time
from typing import Dict, List, NamedTuple, Optional, Sequence, Tuple

import torch
import torch.distributed as dist


class FitPlan(NamedTuple):
    """Subjects [lo, hi) of every chunk, in subject order, and the rank that fits each chunk."""
    chunks: List[Tuple[int, int]]
    owners: List[int]


def plan_fit_chunks(costs: Sequence[float], batch_size: int, world: int) -> FitPlan:
    """Consecutive chunks of ``batch_size`` subjects (the last one may be shorter) over ``world`` ranks.  ``costs[k]`` is
    subject k's cost: 1 for identity fitting, its number of expressions for joint fitting.  Longest-processing-time greedy:
    the costliest chunk first (ties: the lower chunk index) goes to the least loaded rank (ties: the lower rank)."""
    if int(batch_size) < 1 or int(world) < 1:
        raise ValueError('plan_fit_chunks: batch_size and world must be >= 1, got %r and %r' % (batch_size, world))
    n, b = len(costs), int(batch_size)
    chunks = [(lo, min(lo + b, n)) for lo in range(0, n, b)]
    cost = [sum(costs[lo:hi]) for lo, hi in chunks]
    load = [0] * int(world)
    owners = [0] * len(chunks)
    for c in sorted(range(len(chunks)), key=lambda c: (-cost[c], c)):
        r = min(range(int(world)), key=lambda r: (load[r], r))
        owners[c] = r
        load[r] += cost[c]
    return FitPlan(chunks, owners)


def fit_owner(plan: FitPlan, k: int) -> int:
    """The rank that fitted subject ``k``: meshing the subject there needs no transfer."""
    for (lo, hi), r in zip(plan.chunks, plan.owners):
        if lo <= k < hi:
            return r
    raise IndexError('fit_owner: subject %d is not in the plan' % k)


def _group(group):
    """(rank, world, NCCL?) of ``group``; without an initialised process group, ``group=None`` is a world of one."""
    if group is None and not (dist.is_available() and dist.is_initialized()):
        return 0, 1, False
    return dist.get_rank(group), dist.get_world_size(group), dist.get_backend(group) == 'nccl'


def _check_arguments(name, subjects, n_steps, step_scale, batch_size, lambdas, group, world, wire):
    desc = repr((len(subjects), [[int(o.shape[0]) for o in s] for s in subjects], float(n_steps), float(step_scale),
                 int(batch_size), sorted((str(k), float(v)) for k, v in lambdas.items())))
    digest = torch.frombuffer(bytearray(hashlib.sha256(desc.encode()).digest()), dtype=torch.int64).to(wire)
    got = [torch.empty_like(digest) for _ in range(world)]
    dist.all_gather(got, digest, group=group)
    bad = [r for r, d in enumerate(got) if not torch.equal(d, got[0])]
    if bad:
        raise ValueError('%s: ranks %s were called with other subjects, point counts, n_steps, step_scale, batch_size or '
                         'lambdas than rank 0; every rank must pass the same arguments' % (name, bad))


def _slot_code(t: torch.Tensor) -> float:
    """One float beside every result tensor in the bucket: its requires_grad flag and whether it is float64."""
    if t.dtype not in (torch.float32, torch.float64):
        raise TypeError('fitting result of dtype %s' % t.dtype)
    return float(t.requires_grad) + 2.0 * float(t.dtype == torch.float64)


def _pack(results, layouts, device):
    parts = []
    for res, layout in zip(results, layouts):
        for t, shape in zip(res, layout):
            if (t is None) != (shape is None) or (t is not None and tuple(t.shape) != shape):
                raise RuntimeError('fitting result of shape %s where %s was expected'
                                   % (None if t is None else tuple(t.shape), shape))
            if t is not None:
                parts += [t.detach().reshape(-1).to(device, torch.float64),
                          torch.full((1,), _slot_code(t), dtype=torch.float64, device=device)]
    return parts


def _unpack(seg, codes, layout, device):
    """Subject results from their bucket segment ``seg``; ``codes``: the same segment on the host."""
    out, off = [], 0
    for shape in layout:
        if shape is None:
            out.append(None)
            continue
        n = math.prod(shape)
        code = int(codes[off + n])
        dtype = torch.float64 if code & 2 else torch.float32
        out.append(seg[off:off + n].view(shape).to(device=device, dtype=dtype).clone().requires_grad_(bool(code & 1)))
        off += n + 1
    return tuple(out)


def _fit_sharded(name, subjects, costs, layout, batch_fit, fit_one, lambdas, n_steps, schedule_cfg, step_scale, group,
                 batch_size, timings: Optional[Dict[str, float]]):
    """Steps 1-4 of the module docstring.  ``layout(k)``: the shapes of subject k's results (None for a result that is
    None); ``batch_fit(chunk, gens, lambdas)``: the batched fit, or None; ``fit_one(all_obs, lambdas)``: the single-subject
    function on the global generator."""
    from .models.fitting import _apply_schedule, _sampling_plan
    rank, world, nccl = _group(group)
    device = subjects[0][0].device if subjects else torch.device('cpu')
    wire = device if nccl else torch.device('cpu')
    if world > 1:
        _check_arguments(name, subjects, n_steps, step_scale, batch_size, lambdas, group, world, wire)
    if not subjects:
        return []
    n_iters = int(n_steps * step_scale)
    if n_iters < 1:
        raise ValueError('%s: n_steps * step_scale = %r gives no iteration' % (name, n_steps * step_scale))
    plan = plan_fit_chunks(costs, batch_size, world)
    lap = time.perf_counter()

    def tick(key):
        nonlocal lap
        if timings is not None:
            if device.type == 'cuda':
                torch.cuda.synchronize(device)
            now = time.perf_counter()
            timings[key] = timings.get(key, 0.0) + now - lap
            lap = now

    gens = _sampling_plan(subjects, n_iters)
    end_state = torch.get_rng_state()
    tick('sampling_walk_s')
    start = dict(lambdas)
    results = []
    for (lo, hi), r in zip(plan.chunks, plan.owners):
        if r != rank:
            continue
        if batch_fit is not None:
            results += batch_fit(subjects[lo:hi], gens[lo:hi], dict(start))
            continue
        for k in range(lo, hi):
            torch.set_rng_state(gens[k].get_state())
            results.append(fit_one(subjects[k], dict(start)))
    torch.set_rng_state(end_state)
    tick('fit_s')

    # the bucket of every rank: its chunks' subjects in subject order, each result followed by its slot code
    sizes = [sum(math.prod(s) + 1 for s in layout(k) if s is not None) for k in range(len(subjects))]
    lengths = [0] * world
    where, mine = [None] * len(subjects), []
    for (lo, hi), r in zip(plan.chunks, plan.owners):
        for k in range(lo, hi):
            where[k] = (r, lengths[r])
            lengths[r] += sizes[k]
            if r == rank:
                mine.append(k)
    parts = _pack(results, [layout(k) for k in mine], wire)
    parts.append(torch.zeros(max(lengths) - lengths[rank], dtype=torch.float64, device=wire))
    bucket = torch.cat(parts)
    if world > 1:
        buckets = [torch.empty_like(bucket) for _ in range(world)]
        dist.all_gather(buckets, bucket, group=group)
    else:
        buckets = [bucket]
    host = [b.cpu() for b in buckets]
    out = []
    for k in range(len(subjects)):
        r, off = where[k]
        out.append(_unpack(buckets[r][off:off + sizes[k]], host[r][off:off + sizes[k]], layout(k), device))
    tick('exchange_s')

    lam = dict(start)                     # one single-subject call's schedule
    for j in range(n_iters):
        _apply_schedule(j, step_scale, schedule_cfg, lam, 1.0)
    lambdas.update(lam)
    return out


def _anchor_shape(decoder):
    """The anchors the fitters return: (1, K, 3) for the local ensemble, None for a ``DeepSDF``."""
    return (1, decoder.num_kps, 3) if hasattr(decoder, 'lat_dim_loc') else None


def inference_identity_space_batched_sharded(decoder, scans: List[List[torch.Tensor]], lambdas, n_steps, schedule_cfg: Dict,
                                             step_scale=1, lr_scale=1, group=None, batch_size: int = 8,
                                             timings: Optional[Dict[str, float]] = None):
    """:func:`nphm_b200.models.fitting.inference_identity_space_batched` over the ranks of ``group`` (a ``torch.distributed``
    group; None: the default group, or a world of one when none is initialised).  Every rank passes the same arguments, with
    the scans on its own device, and gets the whole list ``[(lat_rep_shape, anchors)]`` in scan order.  Scan k's result is
    what ``inference_identity_space_batched`` gives on its chunk of ``batch_size`` consecutive scans, from the same inputs at
    every step (the rank that fitted it: ``fit_owner(plan_fit_chunks([1] * len(scans), batch_size, world), k)``).  The global CPU generator and
    ``lambdas`` end as the sequential calls leave them.  ``timings`` (optional dict) accumulates this rank's host seconds:
    ``sampling_walk_s``, ``fit_s`` and ``exchange_s`` (each ends in a device synchronise)."""
    from .models import fitting as F
    fit = F._identity_batch_fit(decoder, scans, n_steps, schedule_cfg, step_scale, lr_scale) if scans else None

    def one(all_obs, lam):
        return F.inference_identity_space(decoder, all_obs, lam, n_steps, schedule_cfg, step_scale, lr_scale)
    D, anchors = decoder.lat_dim, _anchor_shape(decoder)
    return _fit_sharded('inference_identity_space_batched_sharded', scans, [1] * len(scans), lambda k: [(1, 1, D), anchors],
                        fit, one, lambdas, n_steps, schedule_cfg, step_scale, group, batch_size, timings)


def inference_iterative_root_finding_joint_batched_sharded(decoder, decoder_expr, subjects: List[List[torch.Tensor]], lambdas,
                                                           n_steps, schedule_cfg: Dict, step_scale=1, lr_scale=1, group=None,
                                                           batch_size: int = 8, timings: Optional[Dict[str, float]] = None):
    """:func:`nphm_b200.models.fitting.inference_iterative_root_finding_joint_batched` over the ranks of ``group``, under the
    contract of :func:`inference_identity_space_batched_sharded`: every rank gets ``[(lat_rep, lat_rep_shape, anchors)]`` in
    subject order, subject k's result that of the batched call on its chunk.  Chunks are balanced on the subjects'
    numbers of expressions: ``plan_fit_chunks([len(s) for s in subjects], batch_size, world)``."""
    from .models import fitting as F
    fit = (F._joint_batch_fit(decoder, decoder_expr, subjects, n_steps, schedule_cfg, step_scale, lr_scale)
           if subjects else None)

    def one(all_obs, lam):
        return F.inference_iterative_root_finding_joint(decoder, decoder_expr, all_obs, lam, n_steps, schedule_cfg, step_scale,
                                                        lr_scale)
    D, anchors = decoder.lat_dim, _anchor_shape(decoder)
    E = decoder_expr.lat_dim_expr if hasattr(decoder_expr, 'lat_dim_expr') else F.NPM_EXPR_DIM
    return _fit_sharded('inference_iterative_root_finding_joint_batched_sharded', subjects, [len(s) for s in subjects],
                        lambda k: [(len(subjects[k]), 1, E), (1, 1, D), anchors], fit, one, lambdas, n_steps, schedule_cfg,
                        step_scale, group, batch_size, timings)
