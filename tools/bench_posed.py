#!/usr/bin/env python
"""Posed queries on the seeded decoders: the compacting Broyden search against the dense one, the dense posed grid against the
posed narrow band, and, for context, the canonical band followed by deform_mesh.

    python tools/bench_posed.py [--res 128 256] [--scale 1 80] [--reps 2] [--out FILE]

Decoders: the seeded ensemble of the tests (tests/conftest.py make_ensemble(0), code sample_latent(1)) in eval mode with
nbatch_points 25000, and the seeded 'compress' DeformationNetwork (make_deformation) with its output layer times --scale (x 80 is
the search fixture's: large deformations, slow and failing searches); one expression code, 0.1 randn (seed 7).

search: J0^-1 and the Broyden search over the whole grid in get_logits_posed's pieces of 2^20 rows, dense
(nphm_mlp_broyden_search) and compacting (nphm_mlp_broyden_search_compact), alternating, both with the early exit; time summed
over the pieces (device events), steps of the first piece, live rows after each step (from searches cut at k steps, first piece),
and whether both give the same bits.  mesh: get_logits_posed + mesh_from_logits against extract_posed_meshes_narrowband (host
time of whole calls, median over --reps, the first call warmed up), the band's evaluated fraction, peak device memory of each,
and whether the meshes are identical; canonical: extract_mesh_narrowband + deform_mesh.  One JSON line per (res, scale), with the
card, its power limit and SM clocks read in the same run."""
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
PIECE = 1 << 20


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name(0)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def search_numbers(eng, cond, grid):
    """dense / compact search time over the pieces, steps and live rows of the first piece, bitwise agreement."""
    total = {False: 0.0, True: 0.0}
    same, steps = True, None
    for a in range(0, grid.shape[1], PIECE):
        pts = grid[:, a:a + PIECE].contiguous()
        _, j0 = eng.inverse_jacobian(pts, cond)
        outs = {}
        for compact in (False, True):
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            outs[compact] = eng.broyden_search(pts, cond, pts, j0, compact=compact)
            end.record()
            end.synchronize()
            total[compact] += start.elapsed_time(end) / 1e3
        same &= all(torch.equal(u, v) for u, v in zip(outs[False][:3], outs[True][:3]))
        if steps is None:
            steps = outs[True][3]
            prev, live = pts, []
            for k in range(1, 16):
                x = eng.broyden_search(pts, cond, pts, j0, max_steps=k, early_exit=False, compact=True)[0]
                live.append(int((x != prev).any(-1).sum()))
                prev = x
    return {'dense_s': total[False], 'compact_s': total[True], 'steps_first_piece': steps, 'moved_rows_per_step': live,
            'rows_first_piece': min(PIECE, grid.shape[1]), 'identical': bool(same)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--res', type=int, nargs='+', default=[128, 256])
    ap.add_argument('--scale', type=float, nargs='+', default=[1.0, 80.0])
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_posed: needs a CUDA device')
    from conftest import MAXI, MINI, make_deformation, make_ensemble, sample_latent
    from nphm_b200.models import reconstruction as R
    from nphm_b200.models.iterative_root_finding import _fused_search_condition
    from nphm_b200.utils.reconstruction import (create_grid_points_from_bounds, extract_mesh_narrowband,
                                                extract_posed_meshes_narrowband, mesh_from_logits)
    dev = torch.device('cuda:0')
    dec = make_ensemble(0, device=dev).eval()
    lat = sample_latent(1).to(dev)
    torch.manual_seed(7)
    z_ex = (torch.randn(1, 200) * 0.1).to(dev)
    rows = []
    for scale in a.scale:
        dfn = make_deformation(dev)
        with torch.no_grad():
            dfn.defDeepSDF.lin6.weight.mul_(scale)
            dfn.defDeepSDF.lin6.bias.mul_(scale)
        eng = dfn.defDeepSDF.engine()
        anchors = dec.engine().anchors(lat.reshape(1, -1))
        cond = _fused_search_condition(dfn, torch.zeros(1, 1, 3, device=dev), torch.cat([lat.reshape(1, -1), z_ex], -1)[:, None],
                                       anchors[:, None])
        for res in a.res:
            grid = torch.from_numpy(create_grid_points_from_bounds(MINI, MAXI, res)).to(dev, torch.float32)[None]
            row = {'res': res, 'scale': scale, 'card': card(), 'search': search_numbers(eng, cond, grid)}

            def dense():
                return mesh_from_logits(R.get_logits_posed(dec, dfn, lat, z_ex, grid, nbatch_points=CHUNK)[0], MINI, MAXI, res)

            def band():
                return extract_posed_meshes_narrowband(dec, dfn, lat, z_ex, MINI, MAXI, res, nbatch_points=CHUNK,
                                                       return_stats=True)

            def canonical():
                m = extract_mesh_narrowband(dec, lat, MINI, MAXI, res, nbatch_points=CHUNK)
                return R.deform_mesh(m, dfn, z_ex.reshape(1, 1, -1), anchors,
                                     lat_rep_shape=lat.reshape(1, 1, -1)) if len(m.vertices) else m

            m_dense, (m_band, st) = dense(), band()
            canonical()
            times = {'dense': [], 'band': [], 'canonical_deform': []}
            for _ in range(a.reps):
                for name, fn in (('dense', dense), ('band', band), ('canonical_deform', canonical)):
                    times[name].append(timed(fn)[0])
            m_band = m_band[0]
            row['mesh'] = {k + '_s': float(np.median(v)) for k, v in times.items()}
            row['mesh'].update({
                'evaluated_fraction': st[0]['voxels_evaluated'] / res ** 3,
                'peak_bytes_dense': peak(dense), 'peak_bytes_band': peak(band), 'peak_bytes_canonical_deform': peak(canonical),
                'identical': bool(np.array_equal(np.asarray(m_dense.faces), np.asarray(m_band.faces))
                                  and np.array_equal(np.asarray(m_dense.vertices), np.asarray(m_band.vertices))),
                'triangles': int(len(m_band.faces))})
            print(json.dumps(row), flush=True)
            rows.append(row)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
