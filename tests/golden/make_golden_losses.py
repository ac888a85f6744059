#!/usr/bin/env python
"""Generate losses.npz: the reference's identity-space training losses (loss_functions.py:20-110, actual_compute_loss) on
its own modules (torch fp32, CPU, autograd) for the batches tests/test_losses_cpu.py and tests/test_gpu_losses.py use.

Needs the reference modules (oracle/_ref, made by oracle/make_ref.py, or a reference checkout):

    python tests/golden/make_golden_losses.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_loader as R      # noqa: E402

KEYS = ('points_face', 'points_non_face', 'sup_grad_near', 'sup_grad_far', 'normals_face', 'normals_non_face', 'gt_anchors')
GRAD_SAMPLES = 4000


def batch(rng, B, n, center, unit_normals):
    def pts(scale):
        return (rng.randn(B, n, 3) * scale + center).astype(np.float32)

    def normals():
        v = rng.randn(B, n, 3).astype(np.float32)
        return v / np.linalg.norm(v, axis=-1, keepdims=True) if unit_normals else v
    out = {'points_face': pts(0.12), 'points_non_face': pts(0.2), 'sup_grad_near': pts(0.15), 'sup_grad_far': pts(0.4),
           'normals_face': normals(), 'normals_non_face': normals(),
           'gt_anchors': (rng.randn(B, 39, 3) * 0.1).astype(np.float32)}
    out['cond'] = (rng.randn(B, 1, 1344) * 0.3).astype(np.float32)
    return out


def main():
    ns = R.load()
    ref = R.make_ensemble(ns, 0).train()
    out = {}
    for tag, seed, B, n, center, unit in (('cpu', 11, 2, 40, 0.0, False), ('gpu', 5, 3, 700, np.array([0.0, 0.05, -0.1]), True)):
        b = batch(np.random.RandomState(seed), B, n, center, unit)
        tb = {k: torch.from_numpy(b[k]) for k in KEYS}
        cond = torch.from_numpy(b['cond']).requires_grad_()
        want = ns.loss_functions.actual_compute_loss(tb, ref, cond)
        for k, v in b.items():
            out['%s_%s' % (tag, k)] = v
        names = sorted(want)
        out['%s_loss_names' % tag] = np.array(names)
        out['%s_loss_values' % tag] = np.array([float(want[k].detach()) for k in names])
        if tag == 'cpu':
            # the graph reaches the weights through the spatial gradient (double backward): d(total)/d lin1.weight, sampled
            total = sum(want[k] for k in ('surf_sdf', 'normals', 'grad'))
            g = torch.autograd.grad(total, ref.ensembled_deep_sdf.lin1.weight)[0].reshape(-1).numpy()
            idx = np.sort(np.random.RandomState(0).choice(g.size, GRAD_SAMPLES, replace=False))
            out['cpu_lin1_grad_idx'] = idx.astype(np.int64)
            out['cpu_lin1_grad'] = g[idx]
            out['cpu_lin1_grad_absmax'] = np.array(np.abs(g).max())
    path = os.path.join(HERE, 'losses.npz')
    np.savez_compressed(path, **out)
    print('wrote %s (%d bytes)' % (path, os.path.getsize(path)))


if __name__ == '__main__':
    main()
