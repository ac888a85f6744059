#!/usr/bin/env python
"""Joint fitting in each deformation mode the native fitters take (compress, glob_only, expr_only), native against the
autograd mirror (NPHM_JOINT_AUTOGRAD=1), on one GPU.

    python tools/bench_fit_modes.py [--modes compress glob_only expr_only] [--S 16] [--iters 10] [--reps 2]

Per mode, three whole calls of --iters iterations (host sampling, schedule and the steps), each printed as one JSON line with
the card, its power limit and SM clock:
  single    inference_iterative_root_finding_joint on 3 observations of 2500 points, iterations/s;
  batched   inference_iterative_root_finding_joint_batched on S subjects of 3 observations (the mirror fits them one after
            another), subject-iterations/s;
  fixed     inference_expression_space with a fixed identity code on the same 3 observations, iterations/s.
Seeded random weights; the deformation field's output layer is scaled down as in tools/bench_joint.py so that the searches
converge.  The two paths alternate --reps times in one process; host clock after a device synchronise, median."""
import argparse, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np
import torch

LAMBDAS = {'surface': 2.0, 'reg_expr': 0.01, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
SCHEDULE = {'lr': {200: 2, 400: 2, 600: 2, 800: 2}, 'symm_dist': {200: 10, 500: 9999}, 'reg_glob': {200: 3, 600: 10},
            'reg_loc': {500: 3, 600: 10}, 'reg_expr': {600: 10}}


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader',
                          '-i', '0'], capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name(0)


def observations(seed, dev, n=3):
    rng = np.random.RandomState(seed)
    return [torch.from_numpy((rng.randn(2500, 3) * 0.12 + np.array([0.0, 0.05, -0.1])).astype(np.float32)).to(dev)
            for _ in range(n)]


def wall(fn, autograd):
    if autograd:
        os.environ['NPHM_JOINT_AUTOGRAD'] = '1'
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0
    finally:
        os.environ.pop('NPHM_JOINT_AUTOGRAD', None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--modes', nargs='+', default=['compress', 'glob_only', 'expr_only'])
    ap.add_argument('--S', type=int, default=16)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--reps', type=int, default=2)
    args = ap.parse_args()
    from conftest import make_ensemble, mean_anchors, sample_latent
    from fit_modes_common import make_deformation
    from nphm_b200.models import fitting as F
    os.environ.pop('NPHM_JOINT_AUTOGRAD', None)
    dev = torch.device('cuda:0')
    gpu = card()
    dec = make_ensemble(0, device=dev).train()
    z_id = sample_latent(3).to(dev).reshape(1, 1, -1)
    obs = observations(100, dev)
    subjects = [observations(200 + k, dev) for k in range(args.S)]
    n_steps = args.iters * 100
    for mode in args.modes:
        dfn = make_deformation(mode, mean_anchors(), device=dev)
        with torch.no_grad():                     # a usable deformation field from random weights (tools/bench_joint.py)
            dfn.defDeepSDF.lin6.weight.mul_(0.05)
            dfn.defDeepSDF.lin6.bias.mul_(0.05)
        assert F._native_joint(dec, dfn, dev), mode
        runs = {
            'single': (1, lambda: F.inference_iterative_root_finding_joint(dec, dfn, obs, dict(LAMBDAS), n_steps, SCHEDULE,
                                                                           0.01)),
            'batched': (args.S, lambda: F.inference_iterative_root_finding_joint_batched(dec, dfn, subjects, dict(LAMBDAS),
                                                                                         n_steps, SCHEDULE, 0.01)),
            'fixed': (1, lambda: F.inference_expression_space(dec, dfn, z_id, obs, dict(LAMBDAS), n_steps, SCHEDULE, 0.01)),
        }
        for what, (scans, fn) in runs.items():
            for autograd in (False, True):
                wall(fn, autograd)                # warm-up: weights, workspaces
            times = {False: [], True: []}
            for _ in range(args.reps):
                for autograd in (False, True):
                    times[autograd].append(wall(fn, autograd))
            rate = {a: scans * args.iters / float(np.median(t)) for a, t in times.items()}
            print(json.dumps({'metric': 'fit_modes_' + what, 'mode': mode, 'gpu': gpu, 'subjects': scans,
                              'iterations': args.iters, 'points': '5 x 1000 sampled per subject and iteration',
                              'native_it_per_s': round(rate[False], 2), 'autograd_it_per_s': round(rate[True], 2),
                              'speedup': round(rate[False] / rate[True], 2)}), flush=True)


if __name__ == '__main__':
    main()
