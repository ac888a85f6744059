#!/usr/bin/env python
"""Narrow-band mesh extraction (extract_mesh_narrowband) against the dense path (get_logits + mesh_from_logits), in eval mode.

    python tools/bench_narrowband.py [--res 256 512] [--decoders nphm npm] [--reps 3] [--warmup 1]

Decoders: nphm = the seeded head of bench.py (tests/conftest.py make_ensemble(0), sample_latent(1), nbatch_points 25000);
npm = an NPM-size DeepSDF (515 -> 1024 x 8 -> 1, tests/narrowband_common.py make_npm_head).  Each measurement is the median
host time of whole calls (both end with the mesh on the host) over --reps after --warmup, the two paths alternating.  Prints one
JSON line per (decoder, res) with ms per mesh, the evaluated fraction, the growth rounds, whether the band mesh is identical to
the dense one (vertex ids, float64 positions, triangles), and the card, its power limit and SM clock read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np
import torch

CHUNK = 25000


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--res', type=int, nargs='+', default=[256, 512])
    ap.add_argument('--decoders', nargs='+', default=['nphm', 'npm'], choices=['nphm', 'npm'])
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_narrowband needs a CUDA device')
    from conftest import MAXI, MINI, make_ensemble, sample_latent
    from narrowband_common import make_npm_head
    from nphm_b200.models.reconstruction import get_logits
    from nphm_b200.utils.reconstruction import create_grid_points_from_bounds, extract_mesh_narrowband, mesh_from_logits
    dev = torch.device('cuda:0')
    for name in args.decoders:
        if name == 'nphm':
            dec, lat = make_ensemble(0, device=dev).eval(), sample_latent(1).to(dev)
        else:
            dec, lat = make_npm_head(dev)
        for res in args.res:
            grid = torch.from_numpy(create_grid_points_from_bounds(MINI, MAXI, res)).to(dev, dtype=torch.float32)[None]

            def dense():
                return mesh_from_logits(get_logits(dec, lat, grid, nbatch_points=CHUNK), MINI, MAXI, res)

            def band():
                return extract_mesh_narrowband(dec, lat, MINI, MAXI, res, nbatch_points=CHUNK, return_stats=True)

            times = {'dense': [], 'band': []}
            for it in range(args.warmup + args.reps):
                for key, fn in (('dense', dense), ('band', band)):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    out = fn()
                    torch.cuda.synchronize()
                    if it >= args.warmup:
                        times[key].append((time.perf_counter() - t0) * 1e3)
                    if key == 'dense':
                        ref = out
                    else:
                        mesh, stats = out
            same = (np.array_equal(np.asarray(mesh.faces), np.asarray(ref.faces))
                    and np.array_equal(np.asarray(mesh.vertices), np.asarray(ref.vertices)))
            d_ms, b_ms = float(np.median(times['dense'])), float(np.median(times['band']))
            print(json.dumps({'metric': 'narrowband_mesh', 'decoder': name, 'res': res, 'nbatch_points': CHUNK, 'card': card(),
                              'dense_ms_per_mesh': round(d_ms, 2), 'band_ms_per_mesh': round(b_ms, 2),
                              'speedup': round(d_ms / b_ms, 2), 'dense_ms_all': [round(t, 2) for t in times['dense']],
                              'band_ms_all': [round(t, 2) for t in times['band']],
                              'evaluated_fraction': round(stats['voxels_evaluated'] / stats['voxels_total'], 4),
                              'blocks_active': stats['blocks_active'], 'blocks_total': stats['blocks_total'],
                              'growth_rounds': stats['growth_rounds'], 'margin': stats['margin'],
                              'vertices': len(ref.vertices), 'identical_to_dense': bool(same)}), flush=True)
            del grid
            torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
