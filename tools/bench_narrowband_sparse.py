#!/usr/bin/env python
"""The narrow band in block-sparse storage (extract_mesh_narrowband(..., sparse=True), DESIGN §4.17) against the dense-storage band,
in eval mode: ms per mesh and peak device memory.

    python tools/bench_narrowband_sparse.py [--res 256 512 1024] [--sparse-only 2048] [--decoders nphm npm sphere] [--reps 3]
                                            [--warmup 1] [--deform 1024]

Decoders: nphm = the seeded head of bench.py (tests/conftest.py make_ensemble(0), sample_latent(1), nbatch_points 25000); npm = the
NPM-size DeepSDF of tests/narrowband_common.py; sphere = the float32 SDF sqrt(x^2 + y^2 + z^2) - 0.5 on [-1, 1]^3 (through
narrowband_volume, since it is no decoder).  For --res both storages run, alternating, and each line says whether the meshes are
identical; for --sparse-only the sparse band runs alone (the dense storage does not fit).  Time: median host time of whole calls
(ending with the mesh on the host) over --reps after --warmup; memory: torch.cuda.max_memory_allocated over one call above what was
allocated before it, decoder weights excluded.  In eval mode the band also evaluates the voxels of get_logits' last-point quirk and
the blocks around them: quirk_voxels says how many, quirk_blocks how many more blocks are active with the quirk than without it,
quirk_share the share of the evaluated voxels the quirk adds (a second run with the quirk off).  --deform poses the sparse nphm mesh of that res with deform_mesh.  Every line carries the card, its power
limit and SM clock read in the same run."""
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
CUBE = ([-1.0] * 3, [1.0] * 3)


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name(0)


def sphere(p):
    out = torch.empty(p.shape[0], device=p.device, dtype=torch.float32)
    for i in range(0, p.shape[0], 1 << 24):
        q = p[i:i + (1 << 24)]
        out[i:i + (1 << 24)] = torch.sqrt(q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1] + q[:, 2] * q[:, 2]) - 0.5
    return out


def measure(fn, dev):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3, torch.cuda.max_memory_allocated(dev) - base


def runner(name, res, sparse, dev, heads):
    from conftest import MAXI, MINI
    from nphm_b200.utils.reconstruction import (LocalExchange, _device_mesh, _mc_pair, _slab_mesh, _sparse_bytes,
                                                extract_mesh_narrowband, narrowband_volume)
    if name == 'sphere':
        def fn():
            with torch.no_grad():
                vol, st, band = narrowband_volume(sphere, *CUBE, res, dev, sparse=sparse)
                v, t = _slab_mesh([band], [vol], LocalExchange(1), *_mc_pair(sparse), dev)
                if sparse:
                    st['device_bytes'] = _sparse_bytes(band)
                return _device_mesh(v, t, *CUBE, res), st
        return fn
    dec, lat = heads[name]
    return lambda: extract_mesh_narrowband(dec, lat, MINI, MAXI, res, nbatch_points=CHUNK, return_stats=True, sparse=sparse)


def same(a, b):
    return bool(np.array_equal(np.asarray(a.faces), np.asarray(b.faces)) and np.array_equal(np.asarray(a.vertices), np.asarray(b.vertices)))


def quirk_share(res, dev, heads):
    """(quirk voxels, extra active blocks, share of the evaluated voxels the quirk adds) for the nphm head in eval mode."""
    from conftest import MAXI, MINI
    from nphm_b200.utils.reconstruction import _band_evaluators, narrowband_volume
    dec, lat = heads['nphm']
    ev, evq = _band_evaluators(dec, lat, dev)
    with torch.no_grad():
        _, on, band = narrowband_volume(ev, MINI, MAXI, res, dev, quirk_period=CHUNK, evaluate_quirk=evq, sparse=True)
        del band
        _, off, band = narrowband_volume(ev, MINI, MAXI, res, dev, sparse=True)
        del band
    n_quirk = -(-res ** 3 // CHUNK)
    return n_quirk, on['blocks_active'] - off['blocks_active'], round(1 - off['voxels_evaluated'] / on['voxels_evaluated'], 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--res', type=int, nargs='*', default=[256, 512, 1024])
    ap.add_argument('--sparse-only', type=int, nargs='*', default=[2048])
    ap.add_argument('--decoders', nargs='+', default=['nphm', 'npm', 'sphere'], choices=['nphm', 'npm', 'sphere'])
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--deform', type=int, nargs='*', default=[1024])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_narrowband_sparse needs a CUDA device')
    from conftest import load_golden, make_deformation, make_ensemble, sample_latent
    from narrowband_common import make_npm_head
    from nphm_b200._native import NativeError
    dev = torch.device('cuda:0')
    heads = {'nphm': (make_ensemble(0, device=dev).eval(), sample_latent(1).to(dev)), 'npm': make_npm_head(dev)}
    jobs = [(res, True) for res in args.res] + [(res, False) for res in args.sparse_only]
    for name in args.decoders:
        for res, both in jobs:
            kinds = ('dense', 'sparse') if both else ('sparse',)
            times, peak, out = {k: [] for k in kinds}, {}, {}
            try:
                for it in range(args.warmup + args.reps):
                    for k in kinds:
                        (mesh, st), ms, pk = measure(runner(name, res, k == 'sparse', dev, heads), dev)
                        out[k] = (mesh, st)
                        peak[k] = max(peak.get(k, 0), pk)
                        if it >= args.warmup:
                            times[k].append(ms)
            except NativeError as e:                  # e.g. a band larger than the u32 brick indices allow
                print(json.dumps({'metric': 'narrowband_sparse_mesh', 'decoder': name, 'res': res, 'card': card(),
                                  'error': str(e)}), flush=True)
                torch.cuda.empty_cache()
                continue
            mesh, st = out['sparse']
            line = {'metric': 'narrowband_sparse_mesh', 'decoder': name, 'res': res, 'card': card(),
                    'sparse_ms_per_mesh': round(float(np.median(times['sparse'])), 1),
                    'sparse_peak_gb': round(peak['sparse'] / 1e9, 3), 'sparse_ms_all': [round(t, 1) for t in times['sparse']],
                    'band_device_gb': round(st['device_bytes']['band'] / 1e9, 3) if 'device_bytes' in st else None,
                    'evaluated_fraction': round(st['voxels_evaluated'] / st['voxels_total'], 5), 'blocks_active': st['blocks_active'],
                    'growth_rounds': st['growth_rounds'], 'vertices': len(mesh.vertices)}
            if both:
                line.update({'dense_storage_ms_per_mesh': round(float(np.median(times['dense'])), 1),
                             'dense_storage_peak_gb': round(peak['dense'] / 1e9, 3),
                             'dense_storage_ms_all': [round(t, 1) for t in times['dense']],
                             'identical_to_dense_storage': same(mesh, out['dense'][0]) and all(
                                 st[k] == out['dense'][1][k] for k in ('blocks_active', 'voxels_evaluated', 'growth_rounds'))})
            if name == 'nphm':
                line['quirk_voxels'], line['quirk_blocks'], line['quirk_share'] = quirk_share(res, dev, heads)
            print(json.dumps(line), flush=True)
            del out, mesh
    from nphm_b200.models.reconstruction import deform_mesh
    d = load_golden('deform.npz')
    dfn = make_deformation(dev)
    for res in args.deform:
        dec, lat = heads['nphm']
        from conftest import MAXI, MINI
        from nphm_b200.utils.reconstruction import extract_mesh_narrowband

        def pose():
            mesh = extract_mesh_narrowband(dec, lat, MINI, MAXI, res, nbatch_points=CHUNK, sparse=True)
            posed = deform_mesh(mesh, dfn, torch.from_numpy(d['z_ex']).to(dev).reshape(1, 1, -1),
                                torch.from_numpy(d['anchors']).to(dev).unsqueeze(0),
                                lat_rep_shape=torch.from_numpy(d['latent_id']).to(dev).reshape(1, 1, -1))
            return mesh, posed
        (mesh, posed), ms, pk = measure(pose, dev)
        moved = float(np.abs(np.asarray(posed.vertices) - np.asarray(mesh.vertices)).max())
        print(json.dumps({'metric': 'narrowband_sparse_posed', 'decoder': 'nphm', 'res': res, 'card': card(), 'ms': round(ms, 1),
                          'peak_gb': round(pk / 1e9, 3), 'vertices': len(posed.vertices), 'faces': len(posed.faces),
                          'max_offset': round(moved, 5), 'finite': bool(np.isfinite(np.asarray(posed.vertices)).all())}), flush=True)


if __name__ == '__main__':
    main()
