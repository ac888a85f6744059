#!/usr/bin/env python
"""Generate train_ensemble.npz: one stage-1 training step of the reference (actual_compute_loss,
src/NPHM/models/loss_functions.py:20-110, + backward with the nphm.yaml lambdas) on its own FastEnsembleDeepSDFMirrored at
nphm.yaml size (39 local members + 1 global, 16 symmetric pairs, hidden 200, 4 layers; torch.manual_seed(0) as in
ensemble.npz), torch fp32 on CPU, B = 2 with small point sets centred on the anchors.

Stores the batch and codes, the state-dict sha256 (the mirror must initialise to the same weights), the loss terms, the
full code and mlp_pos gradients, and a seeded subsample plus the max-abs and norm of every ensembled weight and bias
gradient.  Keeps only points where the reference's |sdf| >= 1e-4 (closer to 0 the sign in the gradients of surf_sdf and
space_sdf is not resolved by an fp32 evaluation).  tests/test_train_ensemble_cpu.py checks the mirror against it.  Needs the reference modules (oracle/_ref,
made by oracle/make_ref.py, or a reference checkout):

    python tests/golden/make_golden_train_ensemble.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_loader as R      # noqa: E402
import ensemble_train_common as E       # noqa: E402
import shape_common as S                # noqa: E402


NORMALS = {'points_face': 'normals_face', 'points_non_face': 'normals_non_face'}


def select_points(net, batch):
    """Per set and batch element, the first E.SIZES points (of twice as many drawn) where the reference's |sdf| >= 1e-4."""
    codes = torch.from_numpy(batch['codes'])
    gt = torch.from_numpy(batch['gt_anchors'])
    out = dict(batch)
    with torch.no_grad():
        for name, n in zip(E.POINT_SETS, E.SIZES):
            pts = torch.from_numpy(batch[name])
            s = net(pts, codes.repeat(1, pts.shape[1], 1), gt)[0][..., 0].abs().numpy()
            keep = [np.flatnonzero(s[b] >= E.MIN_ABS_SDF)[:n] for b in range(s.shape[0])]
            assert all(k.size == n for k in keep), '%s: too few points with |sdf| >= %g' % (name, E.MIN_ABS_SDF)
            for key in (name,) + ((NORMALS[name],) if name in NORMALS else ()):
                out[key] = np.stack([batch[key][b, k] for b, k in enumerate(keep)])
    return out


def main():
    ns = R.load()
    net = R.make_ensemble(ns, 0).train()
    batch = select_points(net, E.make_batch(ns.assets['anchors_39'], sizes=[2 * n for n in E.SIZES]))
    out = {'batch_' + k: v for k, v in batch.items()}
    out['sha256'] = np.array(S.state_dict_sha256(net))
    bt = {k: torch.from_numpy(v) for k, v in batch.items() if k != 'codes'}
    codes = torch.from_numpy(batch['codes']).requires_grad_()
    losses = ns.loss_functions.actual_compute_loss(bt, net, codes)
    E.total_loss(losses).backward()
    names = sorted(losses)
    out['loss_names'] = np.array(names)
    out['loss_values'] = np.array([float(losses[k].detach()) for k in names])
    full, sampled = E.gradient_record(net, codes)
    for k, v in full.items():
        out['full_' + k] = v.astype(np.float32)
    for k, v in sampled.items():
        flat = v.reshape(-1)
        idx = S.sample_idx(k, flat.size)
        out['idx_' + k] = idx.astype(np.int64)
        out['sampled_' + k] = flat[idx].astype(np.float32)
        out['maxabs_' + k] = np.array(np.abs(flat).max(), np.float64)
        out['norm_' + k] = np.array(np.linalg.norm(flat.astype(np.float64)))
    path = os.path.join(HERE, 'train_ensemble.npz')
    np.savez_compressed(path, **out)
    print('wrote %s (%d bytes), losses %s' % (path, os.path.getsize(path), dict(zip(names, out['loss_values']))))


if __name__ == '__main__':
    main()
