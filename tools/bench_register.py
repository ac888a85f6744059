"""Global registration cost on one GPU (DESIGN.md §4.25): the head volume build (``head_volume``, one decoder grid query) and the
two-stage search (``register_observations``) timed separately with CUDA events, for the ensemble and NPM heads, O = 1, 16 and
64 observations of 4000 points (near-surface grid points, turned and scaled to millimetres), unknown and known scale.  Repetitions of the two parts alternate; medians are reported, with
hypothesis-point-iterations per second of the search.  One JSON line per configuration, with the card and its power limit.

    python tools/bench_register.py [--reps 5] [--resolution 128]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        out = torch.cuda.get_device_name(0) + ', power limit not read'
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--resolution', type=int, default=128)
    ap.add_argument('--obs', type=int, nargs='+', default=[1, 16, 64])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_register.py measures on a CUDA device; none found')
    from conftest import MAXI, MINI, make_ensemble, make_npm
    from nphm_b200.models import registration as G
    dev = torch.device('cuda:0')
    gpu = card()
    for name, dec in (('ensemble', make_ensemble(0, device=dev).train()), ('npm', make_npm(dev))):
        vol = G.head_volume(dec, None, args.resolution, MINI, MAXI, dev)
        if not bool((vol.abs() < 0.01).any()):
            # the seeded NPM head's zero level set lies outside the box: search its level set at the 5 % quantile instead,
            # since the search's cost depends on the sizes, not on the field
            vol = vol - torch.quantile(vol[::97].float(), 0.05)
        near = torch.nonzero(vol.abs() < 0.01).reshape(-1)
        grid = G.Grid(args.resolution, MINI, MAXI).coordinates(dev)
        base = grid[near].float()
        g = torch.Generator().manual_seed(0)
        for n_obs in args.obs:
            obs = []
            for o in range(n_obs):
                pts = base[torch.randint(0, base.shape[0], (4000,), generator=g).to(dev)]
                R = G.quaternion_matrices(G.rotation_set(n_obs + 7)[o:o + 1]).to(dev)[0].float()
                obs.append((pts @ R.T) * 1000.0 + 37.0)
            for known in (False, True):
                kw = dict(log_scale=-float(np.log(1000.0))) if known else {}
                times = {'volume': [], 'search': []}
                for rep in range(args.reps + 1):                     # the first repetition warms up
                    for part in ('volume', 'search'):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        torch.cuda.synchronize()
                        e0.record()
                        if part == 'volume':
                            G.head_volume(dec, None, args.resolution, MINI, MAXI, dev)
                        else:
                            G.register_observations(vol, MINI, MAXI, [obs], **kw)
                        e1.record()
                        torch.cuda.synchronize()
                        if rep:
                            times[part].append(e0.elapsed_time(e1))
                n_s = 1 if known else len(G.SCALE_SEEDS)
                c, f = G.COARSE, G.FINE
                work = n_obs * (G.N_ROTATIONS * n_s * min(4000, c['points']) * (c['iters'] + 1)
                                + f['top_k'] * min(4000, f['points']) * (f['iters'] + 1))
                med = {k: float(np.median(v)) for k, v in times.items()}
                print(json.dumps({'decoder': name, 'observations': n_obs, 'points': 4000, 'scale': 'known' if known else 'unknown',
                                  'resolution': args.resolution, 'volume_ms': round(med['volume'], 3),
                                  'search_ms': round(med['search'], 3),
                                  'hypothesis_point_iterations_per_s': float('%.4g' % (work / (med['search'] * 1e-3))),
                                  'reps': args.reps, 'gpu': gpu}), flush=True)


if __name__ == '__main__':
    main()
