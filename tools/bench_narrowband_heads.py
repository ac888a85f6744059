#!/usr/bin/env python
"""Many heads in one band run (extract_meshes_narrowband) against S sequential extract_mesh_narrowband calls.

    python tools/bench_narrowband_heads.py [--res 128 256] [--heads 1 4 16] [--decoders nphm npm sphere] [--reps 2]

Heads are drawn as sample_shape_space draws them (fitting_pointclouds.py:206, randn x std x 0.85 + mean of the assets' NPHM codes,
seeds 100, 101, ...); the NPM decoder has no code statistics in the assets, so its heads are its zero code plus 0.02 randn.
Decoders: nphm = the seeded ensemble of bench.py in eval mode (nbatch_points 25000); npm = an NPM-size DeepSDF (515 -> 1024 x 8 ->
1, tests/narrowband_common.py make_npm_head); sphere = spheres of radius 0.25 + 0.01 h through an evaluate callable (torch
elementwise), whose evaluation costs next to nothing, so its time per mesh is the band's own cost at a small evaluated fraction:
the fixed per-head cost that batching amortises (loop: narrowband_volume + the one-slab marching cubes per head, as
extract_mesh_narrowband runs them; batched: narrowband_heads_volumes + NarrowBandHeads.marching_cubes).

Both paths are warmed up once per (decoder, res) and then alternate; each number is the median host time of whole calls (both end
with the meshes on the host) over --reps.  Prints one JSON line per (decoder, res, S) with ms per mesh of both paths, the mean
evaluated fraction, the padded rows, the largest number of growth rounds, the peak device memory of each path, whether every
head's mesh and stats are identical, and the card, its power limit and SM clock read in the same run."""
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


def draw_codes(name, n, dev):
    from conftest import load_golden
    if name == 'nphm':
        a = load_golden('assets.npz')
        mean, std = torch.from_numpy(a['nphm_lat_mean']), torch.from_numpy(a['nphm_lat_std'])
        out = []
        for i in range(n):
            torch.manual_seed(100 + i)
            out.append(torch.randn(mean.shape) * std * 0.85 + mean)
        return torch.stack(out).to(dev)
    g = torch.Generator().manual_seed(100)
    return (0.02 * torch.randn(n, 512, generator=g)).to(dev)


def sphere_paths(res, dev):
    """(loop, batched) for spheres of the given radii: the protocol of extract_mesh_narrowband / extract_meshes_narrowband with
    an evaluate callable in place of the decoder."""
    from conftest import MAXI, MINI
    from nphm_b200 import _native
    from nphm_b200.utils import reconstruction as R

    def dist(p):                               # elementwise, so that both paths get the same bits whatever the batch shape
        return (p[..., 0] * p[..., 0] + p[..., 1] * p[..., 1] + p[..., 2] * p[..., 2]).sqrt()

    def loop(radii):
        out = []
        with torch.no_grad():
            for r in radii:
                vol, st, band = R.narrowband_volume(lambda p, r=r: dist(p) - r, MINI, MAXI, res, dev)
                verts, tris = R._slab_mesh([band], [vol], R.LocalExchange(1), *R._mc_pair(False), dev)
                out.append((R._device_mesh(verts, tris, MINI, MAXI, res), st))
        return out

    def batched(radii):
        with torch.no_grad():
            bands = _native.NarrowBandHeads(res, 4, dev, len(radii))
            tau = R.default_margin(MINI, MAXI, res, 4)
            vols, st = R.narrowband_heads_volumes(bands, lambda p: dist(p) - radii[:, None], MINI, MAXI, tau)
            meshes = R._device_meshes(*bands.marching_cubes(vols), MINI, MAXI, res)
        nb = bands.blocks_per_axis
        return meshes, [dict(s, blocks_total=nb ** 3, voxels_total=res ** 3, margin=tau) for s in st]
    return loop, batched


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--res', type=int, nargs='+', default=[128, 256])
    ap.add_argument('--heads', type=int, nargs='+', default=[1, 4, 16])
    ap.add_argument('--decoders', nargs='+', default=['nphm', 'npm', 'sphere'], choices=['nphm', 'npm', 'sphere'])
    ap.add_argument('--reps', type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_narrowband_heads needs a CUDA device')
    from conftest import MAXI, MINI, make_ensemble
    from narrowband_common import make_npm_head
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband, extract_meshes_narrowband
    dev = torch.device('cuda:0')
    for name in args.decoders:
        if name == 'sphere':
            all_codes = 0.25 + 0.01 * torch.arange(max(args.heads), device=dev, dtype=torch.float32)
        else:
            dec = make_ensemble(0, device=dev).eval() if name == 'nphm' else make_npm_head(dev)[0]
            all_codes = draw_codes(name, max(args.heads), dev)
        for res in args.res:
            if name == 'sphere':
                loop, batched = sphere_paths(res, dev)
            else:
                def loop(codes):
                    return [extract_mesh_narrowband(dec, c, MINI, MAXI, res, nbatch_points=CHUNK, return_stats=True) for c in codes]

                def batched(codes):
                    return extract_meshes_narrowband(dec, codes, MINI, MAXI, res, nbatch_points=CHUNK, return_stats=True)

            loop(all_codes[:1])
            batched(all_codes[:2])
            for S in args.heads:
                codes = all_codes[:S]
                times, peak = {'loop': [], 'batched': []}, {}
                for it in range(args.reps):
                    for key, fn in (('loop', loop), ('batched', batched)):
                        torch.cuda.synchronize()
                        torch.cuda.reset_peak_memory_stats(dev)
                        t0 = time.perf_counter()
                        out = fn(codes)
                        torch.cuda.synchronize()
                        times[key].append((time.perf_counter() - t0) * 1e3 / S)
                        peak[key] = torch.cuda.max_memory_allocated(dev)
                        if key == 'loop':
                            ref = out
                        else:
                            meshes, stats = out
                same = all(np.array_equal(np.asarray(m.faces), np.asarray(r.faces))
                           and np.array_equal(np.asarray(m.vertices), np.asarray(r.vertices))
                           and {k: v for k, v in st.items() if k != 'padded_rows'} == rst
                           for m, st, (r, rst) in zip(meshes, stats, ref))
                l_ms, b_ms = float(np.median(times['loop'])), float(np.median(times['batched']))
                print(json.dumps({'metric': 'narrowband_heads', 'decoder': name, 'res': res, 'heads': S, 'nbatch_points': CHUNK,
                                  'card': card(), 'loop_ms_per_mesh': round(l_ms, 2), 'batched_ms_per_mesh': round(b_ms, 2),
                                  'speedup': round(l_ms / b_ms, 3),
                                  'loop_ms_all': [round(t, 2) for t in times['loop']],
                                  'batched_ms_all': [round(t, 2) for t in times['batched']],
                                  'evaluated_fraction': round(float(np.mean([s['voxels_evaluated'] for s in stats])) / res ** 3, 4),
                                  'voxels_evaluated': sum(s['voxels_evaluated'] for s in stats),
                                  'padded_rows': sum(s['padded_rows'] for s in stats),
                                  'growth_rounds_max': max(s['growth_rounds'] for s in stats),
                                  'peak_mib_loop': round(peak['loop'] / 2 ** 20), 'peak_mib_batched': round(peak['batched'] / 2 ** 20),
                                  'identical': bool(same)}), flush=True)
                del ref, meshes, stats, out
                torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
