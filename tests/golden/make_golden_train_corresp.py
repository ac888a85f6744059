#!/usr/bin/env python
"""Generate train_corresp.npz: one stage-2 training step of the reference (compute_loss_corresp_forward,
src/NPHM/models/loss_functions.py:282-322, + backward with the nphm_def.yaml lambdas) on its own modules (torch fp32, CPU):
a seeded compress-mode DeformationNetwork in TRAIN mode (per-point compressor noise), the seeded ensemble as decoder_shape
(anchors from its mlp_pos), seeded expression / shape embeddings, B = 4 samples x 300 points.

Stores the random draws the reference made (in order), the loss terms, the full gradients of the compressor, the biases,
mlp_pos's biases and the expression / shape rows of the batch, and a seeded subsample plus the norm of every weight gradient.
tests/test_train_corresp_cpu.py replays the draws through the mirror's composite path, tests/test_gpu_train.py through the
native one.  Needs the reference modules (oracle/_ref, made by oracle/make_ref.py, or a reference checkout):

    python tests/golden/make_golden_train_corresp.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_loader as R      # noqa: E402
import corresp_common as C              # noqa: E402


def main():
    ns = R.load()
    dfn = R.make_deformation(ns).train()
    shape_dec = R.make_ensemble(ns, 0).train()
    lat_expr, lat_shape = C.make_embeddings()
    batch = C.make_batch()
    out = {'batch_' + k: v for k, v in batch.items()}
    out['weights_expr'] = lat_expr.weight.detach().numpy().copy()
    out['weights_shape'] = lat_shape.weight.detach().numpy().copy()
    torch.manual_seed(7)
    log = []
    with C.record_draws(log):
        losses = ns.loss_functions.compute_loss_corresp_forward({k: torch.from_numpy(v) for k, v in batch.items()}, dfn,
                                                                shape_dec, lat_expr, lat_shape, 'cpu')
    C.total_loss(losses).backward()
    out['draw_kinds'] = np.array([k for k, _ in log])
    for i, (_, a) in enumerate(log):
        out['draw_%d' % i] = a.astype(np.float32)
    names = sorted(losses)
    out['loss_names'] = np.array(names)
    out['loss_values'] = np.array([float(losses[k].detach()) for k in names])
    full, sampled = C.gradient_record(dfn, shape_dec, lat_expr, lat_shape, batch)
    for k, v in full.items():
        out['full_' + k] = v.astype(np.float32)
    for k, v in sampled.items():
        flat = v.reshape(-1)
        idx = C.sample_idx(k, flat.size)
        out['idx_' + k] = idx.astype(np.int64)
        out['sampled_' + k] = flat[idx].astype(np.float32)
        out['norm_' + k] = np.array(np.linalg.norm(flat.astype(np.float64)))
    path = os.path.join(HERE, 'train_corresp.npz')
    np.savez_compressed(path, **out)
    print('wrote %s (%d bytes), draws %s, losses %s' % (path, os.path.getsize(path), list(out['draw_kinds']),
                                                       dict(zip(names, out['loss_values']))))


if __name__ == '__main__':
    main()
