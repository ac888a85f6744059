"""Data-parallel training steps for the reference's ``TrainerAutoDecoder`` of both stages (``NPHM.models.training``, stage 1,
``training.py:111-139`` / ``:250-275``; ``NPHM.models.training_corresp``, stage 2, ``training_corresp.py:154-176`` /
``:292-320``), DESIGN §6.

Every rank holds the whole model, receives the WHOLE batch (the reference's loader yields it on every rank) and evaluates a
contiguous slice of its rows (:func:`nphm_b200.distributed.shard_rows`).  One step:

  1. the ranks check that they hold the same batch (``idx``, and ``subj_ind`` in stage 2);
  2. every code row of the batch is looked up once under ``no_grad``, which applies the ``Embedding``'s ``max_norm``
     renormalisation to the whole batch on every rank, so the replicated tables stay bitwise equal; the rank then reads its
     own rows without renormalising them again;
  3. the rank evaluates the existing loss on its rows (stage 1: ``actual_compute_loss(native=True)`` on CUDA, the composite
     path elsewhere; stage 2: ``compute_loss_corresp_forward`` with its native default and ``rows=``, which draws every random
     tensor for the whole batch and keeps the rank's rows), each term scaled by ``B_r / B``: every term is a mean over a set
     whose size is proportional to the rows, so the scaled terms of the ranks add up to the whole-batch term;
  4. the decoder's weight gradients, the gradient rows of the codes and the loss terms of the rank go into ONE flat bucket;
     the buckets are all-gathered and every rank adds the dense parts in rank order and lays the code rows out in batch
     order - the result does not depend on the collective's algorithm and is bitwise equal on every rank;
  5. every rank runs the reference's clipping and optimizer steps (AdamW on the decoder, SparseAdam on the codes) on the
     reduced gradients, so weights, codes and optimizer states stay equal without a broadcast.

The codes' gradient is the sparse tensor the reference's backward makes: the batch's rows as indices, in batch order, with
repeats (stage 2's ``subj_ind``; SparseAdam sums them).  ``torch.nn.utils.clip_grad_norm_`` has no kernel for a sparse
gradient in this torch, so the codes are clipped by :func:`clip_sparse_grad_norm_` (the norm of the coalesced values, the
same coefficient).

Differences from the reference, none of which changes what is trained: in stage 2 the reference accumulates gradients into
the shape codes (``latent_codes_shape.requires_grad = False`` sets a module attribute, not the parameter's flag) and into
``decoder_shape.mlp_pos``, which no optimizer steps and nothing zeroes; the validation step accumulates the decoder's
gradients, which the next training step's ``zero_grad`` drops.  The sharded steps leave those gradients untouched.

The ranks must draw the same batches: the reference's loader shuffles with torch's global CPU generator, so seed it alike on
every rank (``torch.manual_seed`` before the trainer is built).  The CUDA generator must be seeded alike as well: stage 2
draws from it, and each rank ends a step with the state of a one-process step.
"""
from __future__ import annotations

from typing import List

import torch
import torch.distributed as dist
import torch.nn.functional as F


class LocalTrainGroup:
    """The ``world`` shards of every step, run one after another in this process with the ordered reduction of the
    multi-process step, so the result is that of ``world`` processes bit for bit.  Each shard's autograd graph is freed before
    the next one starts: the batch trains at about ``1/world`` of the per-row workspace (gradient accumulation)."""

    def __init__(self, world: int):
        if int(world) < 1:
            raise ValueError('LocalTrainGroup: world must be >= 1, got %r' % (world,))
        self.world = int(world)
        self.ranks = list(range(self.world))
        self.is_main = True

    def check_batch(self, keys: torch.Tensor):
        pass                                    # one batch feeds every shard

    def gather(self, buckets: List[torch.Tensor]) -> List[torch.Tensor]:
        return buckets

    def barrier(self):
        pass


class _ProcessTrainGroup:
    """This process's rank of a ``torch.distributed`` group.  NCCL gathers the device buckets; other backends (gloo) gather
    host copies."""

    def __init__(self, group, device):
        if not dist.is_initialized():
            raise RuntimeError('train_step_sharded: torch.distributed is not initialised (use torchrun and '
                               'init_process_group, or pass a LocalTrainGroup)')
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.ranks = [self.rank]
        self.is_main = self.rank == 0
        self.device = torch.device(device)
        self.wire = self.device if dist.get_backend(group) == 'nccl' else torch.device('cpu')

    def _all_gather(self, t: torch.Tensor) -> List[torch.Tensor]:
        t = t.to(self.wire)
        out = [torch.empty_like(t) for _ in range(self.world)]
        dist.all_gather(out, t, group=self.group)
        return out

    def check_batch(self, keys: torch.Tensor):
        sizes = self._all_gather(torch.tensor([keys.numel()], dtype=torch.int64))
        if any(int(s) != int(sizes[0]) for s in sizes):
            raise ValueError('train_step_sharded: the ranks hold batches of different sizes %s; every rank must receive the '
                             'same batch (seed torch\'s global generator alike on every rank)' % [int(s) for s in sizes])
        allk = self._all_gather(keys.reshape(-1).to(torch.int64))
        bad = [r for r, k in enumerate(allk) if not torch.equal(k, allk[0])]
        if bad:
            raise ValueError('train_step_sharded: ranks %s hold a different batch (idx / subj_ind) than rank 0; every rank '
                             'must receive the same batch (seed torch\'s global generator alike on every rank)' % bad)

    def gather(self, buckets: List[torch.Tensor]) -> List[torch.Tensor]:
        return [b.to(self.device) for b in self._all_gather(buckets[0])]

    def barrier(self):
        dist.barrier(group=self.group)


def _train_group(group, device):
    return group if isinstance(group, LocalTrainGroup) else _ProcessTrainGroup(group, device)


def clip_sparse_grad_norm_(weight: torch.nn.Parameter, max_norm: float):
    """``torch.nn.utils.clip_grad_norm_(embedding.parameters(), max_norm)`` for the sparse gradient of an
    ``Embedding(sparse=True)``: the norm of the coalesced values and torch's coefficient ``min(1, max_norm / (norm + 1e-6))``."""
    g = weight.grad.coalesce()
    coef = torch.clamp(max_norm / (g.values().norm() + 1e-6), max=1.0)
    weight.grad = g * coef


class _Rows:
    """Reads rows of an ``Embedding``'s table without its ``max_norm`` renormalisation (the step renormalises the whole batch's
    rows first) and keeps what it returned: the gradient of that tensor is the code gradient of those rows."""

    def __init__(self, embedding):
        self.weight = embedding.weight
        self.out = None

    def __call__(self, idx):
        self.out = F.embedding(idx, self.weight)
        return self.out


def _is_stage2(trainer) -> bool:
    return hasattr(trainer, 'latent_codes_shape')


def _loss_keys(trainer, stage2: bool):
    """The keys of the loss dict, known to a rank that evaluates no rows."""
    if stage2:
        return ['corresp', 'lat_reg', 'loss_reg_zero']
    from .models.EnsembledDeepSDF import FastEnsembleDeepSDFMirrored
    keys = ['surf_sdf', 'normals', 'space_sdf', 'grad', 'lat_reg']
    if isinstance(trainer.decoder, FastEnsembleDeepSDFMirrored):
        keys += ['anchors', 'symm_dist', 'middle_dist']
    return keys


def _shard_losses(trainer, stage2, batch, rows, codes, shape_codes, epoch, exp_path):
    """The loss dict of batch rows [r0, r1) and the lookup of the rank's code rows."""
    from .models.loss_functions import actual_compute_loss, compute_loss_corresp_forward
    lookup = _Rows(codes)
    if stage2:
        losses = compute_loss_corresp_forward(dict(batch), trainer.decoder, trainer.decoder_shape, lookup, _Rows(shape_codes),
                                              trainer.device, epoch, exp_path, rows=rows)
        return losses, lookup
    r0, r1 = rows
    dtype = codes.weight.dtype                       # float32 as the reference's .float(); float64 codes keep float64
    part = {k: v[r0:r1].to(trainer.device).to(dtype) for k, v in batch.items() if k != 'path'}
    glob_cond = lookup(batch['idx'][r0:r1].to(trainer.device))
    native = True if torch.device(trainer.device).type == 'cuda' else None
    return actual_compute_loss(part, trainer.decoder, glob_cond, native=native), lookup


def _sharded_pass(trainer, batch, grp, codes, shape_codes, params, epoch, exp_path):
    """Steps 1-4 of the module docstring for one batch: afterwards every parameter in ``params`` and ``codes.weight`` hold the
    reduced gradients of the whole batch.  Returns (loss keys, tensor of the reduced terms followed by the total)."""
    from .distributed import shard_rows              # distributed.py re-exports this module
    stage2 = shape_codes is not None
    idx = batch['idx']
    B = idx.shape[0]
    grp.check_batch(torch.cat([idx.reshape(-1), batch['subj_ind'].reshape(-1)]) if stage2 else idx.reshape(-1))
    device = codes.weight.device
    with torch.no_grad():                            # the renormalisation of every row of the batch (max_norm)
        codes(idx.to(device))
        if stage2:
            shape_codes(batch['subj_ind'].to(device))
    keys = _loss_keys(trainer, stage2)
    lambdas = trainer.cfg['lambdas']
    dtype = codes.weight.dtype
    D = codes.weight.shape[1]
    counts = [hi - lo for lo, hi in (shard_rows(B, grp.world, r) for r in range(grp.world))]
    slot = max(counts) * D
    # each gradient's segment of the bucket starts 256 bytes in, as a tensor of its own would: the foreach kernels of the
    # clipping and the optimizers take the same path as on separately allocated gradients
    align = max(1, 256 // codes.weight.element_size())
    sizes = [-(-p.numel() // align) * align for p in params]
    n_dense = sum(sizes)
    many = len(grp.ranks) > 1
    if many:
        cpu_state = torch.get_rng_state()
        cuda_state = torch.cuda.get_rng_state(device) if device.type == 'cuda' else None
    buckets = []
    for rank in grp.ranks:
        if many:                                     # every shard starts from the step's generator state
            torch.set_rng_state(cpu_state)
            if cuda_state is not None:
                torch.cuda.set_rng_state(cuda_state, device)
        r0, r1 = shard_rows(B, grp.world, rank)
        if r1 == r0:                                 # no rows: zeros, and the random draws the other ranks make
            if stage2:
                from .models.loss_functions import corresp_forward_draws
                corresp_forward_draws(trainer.decoder, B, batch['points_neutral'].shape[1], device, dtype)
            buckets.append(torch.zeros(n_dense + len(keys) + 1 + slot, device=device, dtype=dtype))
            continue
        losses, lookup = _shard_losses(trainer, stage2, batch, (r0, r1), codes, shape_codes, epoch, exp_path)
        if list(losses) != keys:
            raise ValueError('train_step_sharded: the loss returned %s, expected %s' % (list(losses), keys))
        scale = (r1 - r0) / B
        terms = [losses[k] * scale for k in keys]
        tot = 0
        for k, t in zip(keys, terms):
            tot = tot + lambdas[k] * t
        grads = torch.autograd.grad(tot, list(params) + [lookup.out], allow_unused=True)
        for p, g in zip(params, grads):
            if g is None:
                raise ValueError('train_step_sharded: a trained decoder parameter of shape %s gets no gradient from the loss'
                                 % tuple(p.shape))
        code_rows = grads[-1].reshape(-1)
        parts = []
        for g, n in zip(grads[:-1], sizes):
            parts += [g.reshape(-1), g.new_zeros(n - g.numel())] if n > g.numel() else [g.reshape(-1)]
        parts += [t.detach().reshape(1).to(dtype) for t in terms]
        parts += [tot.detach().reshape(1).to(dtype), code_rows, code_rows.new_zeros(slot - code_rows.numel())]
        buckets.append(torch.cat(parts))
        del losses, lookup, terms, tot, grads, parts
    buckets = grp.gather(buckets)

    n_sum = n_dense + len(keys) + 1
    acc = buckets[0][:n_sum].clone()                 # rank-ordered sum: the same on every rank, whatever the collective does
    for b in buckets[1:]:
        acc += b[:n_sum]
    off = 0
    for p, n in zip(params, sizes):
        p.grad = acc[off:off + p.numel()].view_as(p)
        off += n
    values = torch.cat([b[n_sum:n_sum + c * D] for b, c in zip(buckets, counts)]).view(B, D)
    codes.weight.grad = torch.sparse_coo_tensor(idx.reshape(1, -1).to(device), values, codes.weight.shape,
                                                check_invariants=False)
    return keys, acc[off:]


def train_step_sharded(trainer, batch, epoch, group=None):
    """Drop-in for ``TrainerAutoDecoder.train_step(batch, epoch)`` of either stage: one data-parallel step over the ranks of
    ``group`` (a ``torch.distributed`` group, None = the default one, or a :class:`LocalTrainGroup`).  Every rank passes the
    same whole batch; returns the reference's dict of Python floats (the loss terms and ``loss``), equal on every rank."""
    stage2 = _is_stage2(trainer)
    grp = _train_group(group, trainer.latent_codes.weight.device)
    trainer.decoder.train()
    trainer.optimizer_encoder.zero_grad()
    trainer.optimizer_lat.zero_grad()
    params = [p for p in trainer.decoder.parameters() if p.requires_grad]
    keys, reduced = _sharded_pass(trainer, batch, grp, trainer.latent_codes,
                                  trainer.latent_codes_shape if stage2 else None, params, epoch,
                                  getattr(trainer, 'exp_path', None))
    if trainer.cfg['grad_clip'] is not None:
        torch.nn.utils.clip_grad_norm_(trainer.decoder.parameters(), max_norm=trainer.cfg['grad_clip'])
    if trainer.cfg['grad_clip_lat'] is not None:
        clip_sparse_grad_norm_(trainer.latent_codes.weight, trainer.cfg['grad_clip_lat'])
    trainer.optimizer_encoder.step()
    trainer.optimizer_lat.step()
    values = reduced.tolist()
    out = dict(zip(keys, values[:-1]))
    out['loss'] = values[-1]
    return out


def val_step_sharded(trainer, epoch, group=None):
    """Drop-in for ``TrainerAutoDecoder.compute_val_loss(epoch)``: the decoder in eval mode, every validation batch sharded as
    in :func:`train_step_sharded`, the validation codes' gradient reduced, clipped and stepped by SparseAdam.  The eval-mode
    quirk of the ensemble (the last point of each decoder call, i.e. of each batch row) stays within a rank's rows.  Returns
    the reference's dict of batch means."""
    stage2 = _is_stage2(trainer)
    grp = _train_group(group, trainer.latent_codes_val.weight.device)
    trainer.decoder.eval()
    sums = {k: 0.0 for k in trainer.cfg['lambdas']}
    sums['loss'] = 0.0
    c = 0
    for val_batch in trainer.val_data_loader:
        trainer.optimizer_lat_val.zero_grad()
        keys, reduced = _sharded_pass(trainer, val_batch, grp, trainer.latent_codes_val,
                                      trainer.latent_codes_shape_val if stage2 else None, [], None, None)
        if trainer.cfg['grad_clip_lat'] is not None:
            clip_sparse_grad_norm_(trainer.latent_codes_val.weight, trainer.cfg['grad_clip_lat'])
        trainer.optimizer_lat_val.step()
        values = reduced.tolist()
        for k, v in zip(keys, values[:-1]):
            sums[k] += v
        sums['loss'] += values[-1]
        c = c + 1
    return {k: v / c for k, v in sums.items()}


def shard_trainer(trainer, group=None):
    """Binds :func:`train_step_sharded` and :func:`val_step_sharded` onto a reference ``TrainerAutoDecoder`` of either stage,
    and makes ``save_checkpoint`` and ``log_recs`` run on rank 0 only, followed by a barrier.  The reference's ``train_model``
    loop then trains data-parallel unchanged.  Returns the trainer."""
    grp = _train_group(group, trainer.latent_codes.weight.device)
    trainer.train_step = lambda batch, epoch: train_step_sharded(trainer, batch, epoch, group)
    trainer.compute_val_loss = lambda epoch: val_step_sharded(trainer, epoch, group)

    def on_main(fn):
        def run(*args, **kwargs):
            if grp.is_main:
                fn(*args, **kwargs)
            grp.barrier()
        return run
    trainer.save_checkpoint = on_main(trainer.save_checkpoint)
    trainer.log_recs = on_main(trainer.log_recs)
    return trainer
