#!/usr/bin/env python
"""Generate train_shape.npz: one stage-1 training step of the reference (actual_compute_loss,
src/NPHM/models/loss_functions.py:20-110, + backward with the npm.yaml lambdas) on its own DeepSDF at npm.yaml size
(lat_dim 512, hidden 1024, 8 layers, geometric init, torch.manual_seed(12) as in npm.npz), torch fp32 on CPU, B = 2 with
small point sets and unit normals.

Stores the batch and codes, the state-dict sha256 (the mirror must initialise to the same weights), the loss terms, the
full code and bias gradients, and a seeded subsample plus the max-abs and norm of every weight gradient.
tests/test_train_shape_cpu.py checks the mirror's composite path against it, tests/test_gpu_train_shape.py the native one.
Needs the reference modules (oracle/_ref, made by oracle/make_ref.py, or a reference checkout):

    python tests/golden/make_golden_train_shape.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_loader as R      # noqa: E402
import shape_common as S                # noqa: E402


def main():
    ns = R.load()
    net = S.make_decoder(ns.deepSDF.DeepSDF)
    batch = S.make_batch()
    out = {'batch_' + k: v for k, v in batch.items()}
    out['sha256'] = np.array(S.state_dict_sha256(net))
    bt = {k: torch.from_numpy(v) for k, v in batch.items() if k != 'codes'}
    codes = torch.from_numpy(batch['codes']).requires_grad_()
    losses = ns.loss_functions.actual_compute_loss(bt, net, codes)
    S.total_loss(losses).backward()
    names = sorted(losses)
    out['loss_names'] = np.array(names)
    out['loss_values'] = np.array([float(losses[k].detach()) for k in names])
    full, sampled = S.gradient_record(net, codes)
    for k, v in full.items():
        out['full_' + k] = v.astype(np.float32)
    for k, v in sampled.items():
        flat = v.reshape(-1)
        idx = S.sample_idx(k, flat.size)
        out['idx_' + k] = idx.astype(np.int64)
        out['sampled_' + k] = flat[idx].astype(np.float32)
        out['maxabs_' + k] = np.array(np.abs(flat).max(), np.float64)
        out['norm_' + k] = np.array(np.linalg.norm(flat.astype(np.float64)))
    path = os.path.join(HERE, 'train_shape.npz')
    np.savez_compressed(path, **out)
    print('wrote %s (%d bytes), losses %s' % (path, os.path.getsize(path), dict(zip(names, out['loss_values']))))


if __name__ == '__main__':
    main()
