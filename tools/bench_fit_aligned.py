#!/usr/bin/env python
"""Fitting with and without observation poses (DESIGN.md §4.24).

    python tools/bench_fit_aligned.py [--scans 1 16] [--iters 30] [--reps 3]

For the NPHM ensemble (tests/conftest.py make_ensemble + make_deformation) and the NPM baseline's DeepSDF pair
(tests/npm_fit_common.py), identity and joint fitting: the batched fitter's step on S scans of 3 observations (5 x 1000 sampled
points per scan) without poses and with poses (one shared table), alternating --reps times, CUDA events, median.  One JSON line
per (decoder, mode, S) with scan-iterations/s of both, and, for the ensemble's identity fitter, the posed route with frozen
poses (surface_grad + apply_gradient, pose apply and gradient, no pose update), which isolates the route switch.
Each line carries the card and its power limit."""
import argparse, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np
import torch

LAMBDAS = {'surface': 2.0, 'reg_expr': 0.01, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name(0)


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--scans', type=int, nargs='+', default=[1, 16])
    ap.add_argument('--iters', type=int, default=30)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_fit_aligned needs a CUDA device')
    from conftest import make_deformation, make_ensemble
    from npm_fit_common import make_decoders
    from nphm_b200.models import fitting as F
    from nphm_b200.models.deepSDF import DeepSDF
    from nphm_b200.models.pose import ObservationPoses
    dev = torch.device('cuda:0')
    decoders = {'nphm': (make_ensemble(0, device=dev).train(), make_deformation(dev)), 'npm': make_decoders(DeepSDF, dev)}
    gpu = card()
    for name, (dec, dfn) in decoders.items():
        for S in args.scans:
            scans = []
            for k in range(S):
                rng = np.random.RandomState(100 + k)
                scans.append([torch.from_numpy((rng.randn(2500, 3) * 0.12 + np.array([0.0, 0.05, -0.1])).astype(np.float32))
                              .to(dev) for _ in range(3)])
            torch.manual_seed(0)
            sample = [F._sample_observations(s) for s in scans]
            obs = [o for o, _ in sample]
            idx = [i.long().to(dev) for _, i in sample]
            rows = torch.cat([i + 3 * k for k, i in enumerate(idx)]).to(torch.int32)
            for mode in ('identity', 'joint'):
                def fitter(poses):
                    if mode == 'identity':
                        cls = F.BatchedNpmIdentityFitter if name == 'npm' else F.BatchedIdentityFitter
                        f = cls(dec, S, dev, poses)
                        return lambda: f.step(obs, dict(LAMBDAS), 0.1, 0.01, obs_idx=None if poses is None else rows)
                    cls = F.BatchedNpmJointFitter if name == 'npm' else F.BatchedJointFitter
                    f = cls(dec, dfn, [3] * S, dev, poses=poses)
                    return lambda: f.step(obs, idx, dict(LAMBDAS), 0.1, 0.01)
                runs = {'plain': fitter(None), 'posed': fitter(ObservationPoses(3 * S, dev))}
                if mode == 'identity' and name == 'nphm':
                    runs['route_only'] = fitter(ObservationPoses(3 * S, dev, lr=(0.0, 0.0, 0.0)))
                times = {k: [] for k in runs}
                for fn in runs.values():
                    timed(fn, 3)
                for _ in range(args.reps):
                    for k, fn in runs.items():
                        times[k].append(timed(fn, args.iters))
                line = {'decoder': name, 'mode': mode, 'S': S, 'gpu': gpu}
                for k, ts in times.items():
                    line['%s_scan_it_per_s' % k] = round(S * 1000.0 / float(np.median(ts)), 1)
                print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
