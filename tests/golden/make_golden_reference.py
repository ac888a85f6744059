#!/usr/bin/env python
"""Generate reference_configs.npz: outputs of the UNMODIFIED reference modules (torch fp32, CPU) on BASELINE.json's
configurations, which tests/test_gpu_reference.py compares the CUDA path against.

Needs the reference modules (oracle/_ref, made by oracle/make_ref.py, or a reference checkout); run where they exist:

    python tests/golden/make_golden_reference.py

Every array is the reference's own output at a fixed, seeded set of grid indices (whole chunks where the chunked
evaluation matters), so the file stays small while the tests keep comparing value for value.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import ref_loader as R      # noqa: E402

MINI = [-.55, -.5, -.95]
MAXI = [0.55, 0.75, 0.4]
C1_SAMPLES = 4000
C2_CHUNKS = (0, 335, 500, 671)          # 25 000-point chunks of the 256^3 grid (671: the ragged last one, 2216 points)
C3_SAMPLES = 6000


def grid(ns, res):
    g = ns.utils_reconstruction.create_grid_points_from_bounds(MINI, MAXI, res)
    return torch.from_numpy(g).to(dtype=torch.float).reshape(1, -1, 3)


def fingerprint(module):
    """Per-parameter (sum, sum of squares, first 8 values) in float64: pins the reference's initialisation."""
    keys, fp = [], []
    for k, v in module.state_dict().items():
        a = v.detach().double().reshape(-1).numpy()
        head = np.zeros(8)
        head[:min(8, a.size)] = a[:8]
        keys.append(k)
        fp.append(np.concatenate([[a.sum(), (a * a).sum()], head]))
    return np.array(keys), np.array(fp)


def main():
    ns = R.load()
    torch.set_num_threads(os.cpu_count() or 1)
    out = {}
    dec = R.make_ensemble(ns, 0)
    out['ens_keys'], out['ens_fp'] = fingerprint(dec)
    out['def_keys'], out['def_fp'] = fingerprint(R.make_deformation(ns))
    lat = R.sample_latent(ns, 1)
    rng = np.random.RandomState(0)

    # configs[0]: 64^3, get_logits, eval / train, nbatch 25 000 / 20 000 - seeded points + every chunk's last index and its neighbour
    g64 = grid(ns, 64)
    n = g64.shape[1]
    for train in (False, True):
        dec.train(train)
        for nb in (25000, 20000):
            last = np.concatenate([np.arange(nb - 1, n, nb), [n - 1]])
            idx = np.unique(np.concatenate([rng.choice(n, C1_SAMPLES, replace=False), last, last - 1]))
            with torch.no_grad():
                want = ns.reconstruction.get_logits(dec, lat, g64, nbatch_points=nb)
            out['c1_%d_%d_idx' % (train, nb)] = idx.astype(np.int64)
            out['c1_%d_%d_sdf' % (train, nb)] = want[idx].astype(np.float32)

    # configs[1]: 256^3, eval, nbatch 25 000 - whole chunks (the quirk sits at each chunk's last index)
    dec.eval()
    g256 = grid(ns, 256)
    for c in C2_CHUNKS:
        pts = g256[:, c * 25000:(c + 1) * 25000]
        with torch.no_grad():
            out['c2_chunk_%d' % c] = ns.reconstruction.get_logits(dec, lat, pts, nbatch_points=25000).astype(np.float32)
    del g256

    # configs[2]: deformation field on 64^3 (seeded points) and the identity field (train mode) at the deformed points
    dfn = R.make_deformation(ns)
    torch.manual_seed(3)
    lat_ex = torch.randn(200) * 0.01
    cond = torch.cat([lat, lat_ex]).reshape(1, 1, -1)
    idx = np.sort(rng.choice(n, C3_SAMPLES, replace=False))
    pts = g64[:, idx]
    with torch.no_grad():
        _, anchors = dec(g64[:, :1], lat.reshape(1, 1, -1), None)
        off = dfn(pts, cond.repeat(1, len(idx), 1), anchors)[0]
        dec.train()
        sdf = dec(pts + off, lat.reshape(1, 1, -1).repeat(1, len(idx), 1), None)[0]
    out['c3_idx'] = idx.astype(np.int64)
    out['c3_lat_ex'] = lat_ex.numpy()
    out['c3_offsets'] = off[0].numpy()
    out['c3_sdf'] = sdf.reshape(-1).numpy()

    # get_logits_backward (models/reconstruction.py:28-56) with a DeepSDF expression decoder on 24^3
    dec.eval()
    torch.manual_seed(31)
    ex = ns.deepSDF.DeepSDF(lat_dim=100, hidden_dim=128, nlayers=6, out_dim=3).eval()
    torch.manual_seed(32)
    lat_e = torch.randn(1, 1, 100) * 0.1
    g24 = grid(ns, 24)
    want, anc = ns.reconstruction.get_logits_backward(dec, ex, lat.reshape(1, 1, -1), lat_e, g24, nbatch_points=5000,
                                                      return_anchors=True)
    want0 = ns.reconstruction.get_logits_backward(dec, ex, lat.reshape(1, 1, -1), None, g24, nbatch_points=5000)
    out['bw_lat_ex'] = lat_e.numpy()
    out['bw_sdf'] = np.asarray(want, dtype=np.float32)
    out['bw_anchors'] = anc.detach().numpy()
    out['bw_sdf_no_expr'] = np.asarray(want0, dtype=np.float32)
    ex_keys, ex_fp = fingerprint(ex)
    out['ex_keys'], out['ex_fp'] = ex_keys, ex_fp

    path = os.path.join(HERE, 'reference_configs.npz')
    np.savez_compressed(path, **out)
    print('wrote %s (%d bytes)' % (path, os.path.getsize(path)))


if __name__ == '__main__':
    main()
