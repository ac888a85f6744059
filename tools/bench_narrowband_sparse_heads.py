#!/usr/bin/env python
"""The block-sparse band of S heads (extract_meshes_narrowband / extract_posed_meshes_narrowband with sparse=True, DESIGN §4.21)
against the head-by-head sparse loop and the dense-storage head band, in eval mode: ms per mesh, peak device memory, band bytes
per head and padded rows.

    python tools/bench_narrowband_sparse_heads.py [--res 256 512 1024] [--heads 1 4 16] [--posed-res 256 512 1024]
                                                  [--posed-heads 1 4] [--thin 2048] [--reps 2] [--warmup 1] [--no-dense]

Canonical rows: the seeded ensemble of bench.py (tests/conftest.py make_ensemble(0), codes sample_latent(1 .. S), nbatch_points
25000), batched sparse against extract_mesh_narrowband(..., sparse=True) per head and against the dense-storage head band.  Posed
rows: the same ensemble with the tests' seeded `compress` deformation network, S expressions (seed 8, x 0.1), sparse against
dense storage, default margin.  Thin rows: two translation fields over the analytic sphere sqrt(x^2 + y^2 + z^2) - 0.5 on
[-1, 1]^3 (the posed SDF of a translation t is sdf(p - t), as test_posed_logits_of_a_translation checks), evaluated in closed form
and meshed in sparse storage only, so that the band is thin.  Time: median host time of whole calls (meshes on the host) over --reps after --warmup, the variants alternated; memory:
torch.cuda.max_memory_allocated over one call above what was allocated before it.  Every line says whether each head's mesh and
band stats were identical to the path it is compared with, and carries the card, its power limit and SM clock read in the same
run."""
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
BAND_STATS = ('blocks_active', 'voxels_evaluated', 'growth_rounds')


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name(0)


def measure(fn, dev):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3, torch.cuda.max_memory_allocated(dev) - base


def same(a, b):
    return bool(np.array_equal(np.asarray(a.faces), np.asarray(b.faces)) and np.array_equal(np.asarray(a.vertices), np.asarray(b.vertices)))


def identical(out, ref):
    (ma, sa), (mb, sb) = out, ref
    return all(same(x, y) for x, y in zip(ma, mb)) and all({k: x[k] for k in BAND_STATS} == {k: y[k] for k in BAND_STATS}
                                                           for x, y in zip(sa, sb))


def run(variants, reps, warmup, dev):
    """{name: fn} alternated: (outputs, median ms, all ms, peak bytes) per name."""
    times, peak, out = {k: [] for k in variants}, {}, {}
    for it in range(warmup + reps):
        for k, fn in variants.items():
            o, ms, pk = measure(fn, dev)
            out[k] = o
            peak[k] = max(peak.get(k, 0), pk)
            if it >= warmup:
                times[k].append(ms)
    return {k: (out[k], float(np.median(times[k])), [round(t, 1) for t in times[k]], peak[k]) for k in variants}


def summary(line, S, res, res_out):
    (meshes, stats), ms, all_ms, pk = res_out['sparse_heads']
    nb = stats[0]['device_bytes']
    line.update({'sparse_heads_ms_per_mesh': round(ms / S, 1), 'sparse_heads_ms_all': all_ms, 'sparse_heads_peak_gb': round(pk / 1e9, 3),
                 'band_gb_per_head': round(nb['band'] / nb['heads'] / 1e9, 3), 'heads_per_chunk': nb['heads'],
                 'evaluated_fraction': round(float(np.mean([s['voxels_evaluated'] for s in stats])) / res ** 3, 4),
                 'padded_rows_per_evaluated': round(sum(s['padded_rows'] for s in stats) / sum(s['voxels_evaluated'] for s in stats), 5),
                 'growth_rounds': [s['growth_rounds'] for s in stats], 'vertices': [len(m.vertices) for m in meshes]})
    for k, (o, ms_k, all_k, pk_k) in res_out.items():
        if k == 'sparse_heads':
            continue
        line.update({k + '_ms_per_mesh': round(ms_k / S, 1), k + '_ms_all': all_k, k + '_peak_gb': round(pk_k / 1e9, 3),
                     'identical_to_' + k: identical(res_out['sparse_heads'][0], o)})
    return line


def canonical(args, dev):
    from conftest import MAXI, MINI, make_ensemble, sample_latent
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband, extract_meshes_narrowband
    dec = make_ensemble(0, device=dev).eval()
    for res in args.res:
        for S in args.heads:
            codes = torch.stack([sample_latent(1 + h).to(dev) for h in range(S)]).reshape(S, -1)
            kw = dict(nbatch_points=CHUNK, return_stats=True)

            def loop():
                out = [extract_mesh_narrowband(dec, codes[h:h + 1], MINI, MAXI, res, sparse=True, **kw) for h in range(S)]
                return [m for m, _ in out], [s for _, s in out]
            variants = {'sparse_heads': lambda: extract_meshes_narrowband(dec, codes, MINI, MAXI, res, sparse=True, **kw),
                        'sparse_loop': loop}
            if not args.no_dense:
                variants['dense_storage_heads'] = lambda: extract_meshes_narrowband(dec, codes, MINI, MAXI, res, **kw)
            out = run(variants, args.reps, args.warmup, dev)
            print(json.dumps(summary({'metric': 'sparse_heads_canonical', 'heads': S, 'res': res, 'card': card()}, S, res, out)),
                  flush=True)
            del out
            torch.cuda.empty_cache()


def posed(args, dev):
    from conftest import MAXI, MINI, make_deformation, make_ensemble, sample_latent
    from nphm_b200.utils.reconstruction import extract_posed_meshes_narrowband
    dec = make_ensemble(0, device=dev).eval()
    dfn = make_deformation(dev)
    lat = sample_latent(1).to(dev)
    for res in args.posed_res:
        for S in args.posed_heads:
            torch.manual_seed(8)
            z_ex = torch.randn(S, 200, device=dev) * 0.1
            kw = dict(nbatch_points=CHUNK, return_stats=True)
            variants = {'sparse_heads': lambda: extract_posed_meshes_narrowband(dec, dfn, lat, z_ex, MINI, MAXI, res, sparse=True, **kw)}
            if not args.no_dense:
                variants['dense_storage_heads'] = lambda: extract_posed_meshes_narrowband(dec, dfn, lat, z_ex, MINI, MAXI, res, **kw)
            out = run(variants, args.reps, args.warmup, dev)
            print(json.dumps(summary({'metric': 'sparse_heads_posed', 'heads': S, 'res': res, 'card': card()}, S, res, out)), flush=True)
            del out
            torch.cuda.empty_cache()


def thin(args, dev):
    """Translation fields over the analytic sphere: the posed value at p is sdf(p - t_s), the exact root of x + t_s = p, evaluated
    in closed form; the S expressions run through narrowband_heads_volumes with the sparse band of S heads, and each head's mesh
    (index units, ids, triangles) and stats are checked against the single sparse band of the same field."""
    from nphm_b200 import _native
    from nphm_b200.utils.reconstruction import (LocalExchange, _mc_pair, _slab_mesh, default_margin, narrowband_heads_volumes,
                                                narrowband_volume)
    lo, hi = [-1.0] * 3, [1.0] * 3
    shifts = torch.tensor([[0.03, -0.02, 0.05], [-0.04, 0.01, 0.02]], device=dev)
    S = shifts.shape[0]

    def evaluate(pts):                                   # S x n x 3 -> S x n
        out = torch.empty(pts.shape[:2], device=dev, dtype=torch.float32)
        for i in range(0, pts.shape[1], 1 << 23):
            q = pts[:, i:i + (1 << 23)] - shifts[:, None]
            out[:, i:i + (1 << 23)] = torch.sqrt((q * q).sum(-1)) - 0.5
        return out

    for res in args.thin:
        tau = default_margin(lo, hi, res)

        def fn():
            with torch.no_grad():
                bands = _native.SparseNarrowBandHeads(res, 4, dev, S)
                vols, st = narrowband_heads_volumes(bands, evaluate, lo, hi, tau)
                v, t, counts = bands.marching_cubes(vols)
                return (v, t, counts), st, bands.device_bytes()
        ((v, t, counts), st, band_bytes), ms, pk = measure(fn, dev)
        ok, vo, to = True, 0, 0
        for s in range(S):                               # each head against the single sparse band of its shifted sphere
            f = lambda p, s=s: evaluate(p[None].expand(S, -1, 3).contiguous())[s]      # noqa: E731
            with torch.no_grad():
                vol, st1, band = narrowband_volume(f, lo, hi, res, dev, margin=tau, sparse=True)
                v1, t1 = _slab_mesh([band], [vol], LocalExchange(1), *_mc_pair(True), dev)
            nv, nt = counts[s]
            ok &= (torch.equal(v1, v[vo:vo + nv]) and torch.equal(t1, t[to:to + nt]) and
                   all(st1[k] == st[s][k] for k in BAND_STATS))
            vo, to = vo + nv, to + nt
            del band, vol, v1, t1
        print(json.dumps({'metric': 'sparse_heads_posed_thin', 'heads': S, 'res': res, 'card': card(), 'ms_per_mesh': round(ms / S, 1),
                          'peak_gb': round(pk / 1e9, 3), 'band_gb_per_head': round(band_bytes / S / 1e9, 3),
                          'evaluated_fraction': [round(s['voxels_evaluated'] / res ** 3, 5) for s in st],
                          'vertices': [c[0] for c in counts], 'identical_to_single_sparse_band': bool(ok)}), flush=True)
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--res', type=int, nargs='*', default=[256, 512, 1024])
    ap.add_argument('--heads', type=int, nargs='*', default=[1, 4, 16])
    ap.add_argument('--posed-res', type=int, nargs='*', default=[256, 512, 1024])
    ap.add_argument('--posed-heads', type=int, nargs='*', default=[1, 4])
    ap.add_argument('--thin', type=int, nargs='*', default=[2048])
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--no-dense', action='store_true', help='skip the dense-storage head band (it does not fit at large res x S)')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_narrowband_sparse_heads needs a CUDA device')
    dev = torch.device('cuda:0')
    canonical(args, dev)
    posed(args, dev)
    thin(args, dev)


if __name__ == '__main__':
    main()
