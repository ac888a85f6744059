#!/usr/bin/env python
"""Joint identity + expression fitting (reference `inference_iterative_root_finding_joint`, SURVEY §8 a11): iteration rate
and, with --profile, where one iteration's time goes (torch profiler, top CUDA ops + number of launches).

    python tools/bench_joint.py --steps 50 [--profile] [--obs 3]
    python tools/bench_joint.py --decoder npm --steps 10 [--iters 5]

Synthetic scan: `--obs` observations x 2500 points; every iteration samples 5 x 1000 points like the reference.
`--decoder npm`: the NPM baseline of fitting_npm.yaml (DeepSDF identity 515 -> 1024 x 8 -> 1, expression 715 -> 1024 x 8 -> 3,
seeded as in tests/npm_fit_common.py).  Native (NpmJointFitter) and composite (autograd) runs of `--iters` iterations
alternate `--steps` times in one process; reports the median ms per iteration of each, with the card and its power limit."""
import argparse, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np
import torch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--obs', type=int, default=3)
    ap.add_argument('--profile', action='store_true')
    ap.add_argument('--decoder', choices=('nphm', 'npm'), default='nphm')
    ap.add_argument('--iters', type=int, default=5, help='--decoder npm: iterations per timed run')
    args = ap.parse_args()
    if args.decoder == 'npm':
        return bench_npm(args)
    from conftest import make_ensemble, make_deformation
    from nphm_b200.models.fitting import inference_iterative_root_finding_joint
    dev = torch.device('cuda', 0)
    dec = make_ensemble(0, device=dev).train()               # fitting_pointclouds.py:268
    dfn = make_deformation(device=dev)
    with torch.no_grad():                                   # small deformations, like a trained field near the neutral pose
        dfn.defDeepSDF.lin6.weight.mul_(0.05); dfn.defDeepSDF.lin6.bias.mul_(0.05)
    rng = np.random.RandomState(7)
    obs = [torch.from_numpy((rng.randn(2500, 3) * 0.12 + np.array([0.0, 0.05, -0.1])).astype(np.float32)).to(dev)
           for _ in range(args.obs)]
    lambdas = {'surface': 2.0, 'reg_expr': 0.05, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
    schedule = {'lr': {200: 2, 400: 2}, 'symm_dist': {200: 10, 500: 9999}, 'reg_glob': {200: 3}, 'reg_loc': {500: 3}}

    def run(n):
        np.random.seed(0); torch.manual_seed(0)
        return inference_iterative_root_finding_joint(dec, dfn, obs, dict(lambdas), n_steps=n, schedule_cfg=schedule)

    run(3)
    torch.cuda.synchronize(); t0 = time.perf_counter()
    z_ex, z_id, _ = run(args.steps)
    torch.cuda.synchronize(); dt = time.perf_counter() - t0
    out = {'metric': 'joint_fit', 'iterations': args.steps, 'observations': args.obs, 'ms_per_iter': 1e3 * dt / args.steps,
           'iters_per_s': args.steps / dt, 'finite': bool(torch.isfinite(z_ex).all() and torch.isfinite(z_id).all())}
    print(json.dumps(out))
    if args.profile:
        from torch.profiler import profile, ProfilerActivity
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            run(3)
            torch.cuda.synchronize()
        print(prof.key_averages().table(sort_by='cuda_time_total', row_limit=30, max_name_column_width=60))
        ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        print('cuda kernel launches per iteration: %.0f   cuda time per iteration: %.2f ms'
              % (len(ev) / 3.0, sum(e.device_time for e in ev) / 3e3))


def alternate(runs, steps, iters):
    """Times ``runs`` (name -> fn(n_iterations)) alternately, ``steps`` times each after one warm-up call; median ms per
    iteration of each (CUDA events around every call)."""
    for fn in runs.values():
        fn(2)
    times = {k: [] for k in runs}
    for _ in range(steps):
        for name, fn in runs.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            fn(iters)
            b.record()
            torch.cuda.synchronize()
            times[name].append(a.elapsed_time(b) / iters)
    return {k: float(np.median(v)) for k, v in times.items()}


def bench_npm(args):
    from bench_train import gpu_info
    from npm_fit_common import LAMBDAS_JOINT, SCHEDULE, make_decoders
    from nphm_b200.models import fitting as F
    from nphm_b200.models.deepSDF import DeepSDF
    dev = torch.device('cuda', torch.cuda.current_device())
    dec, expr = make_decoders(DeepSDF, dev)
    assert F._native_npm_joint(dec, expr, dev) and not os.environ.get('NPHM_JOINT_AUTOGRAD')
    rng = np.random.RandomState(7)
    obs = [torch.from_numpy((rng.randn(2500, 3) * 0.1 + np.array([0.0, 0.05, -0.1])).astype(np.float32)).to(dev)
           for _ in range(args.obs)]

    def run(fn):
        def go(n):
            np.random.seed(0); torch.manual_seed(0)
            return fn(dec, expr, obs, dict(LAMBDAS_JOINT), n, SCHEDULE)
        return go

    name, power = gpu_info()
    ms = alternate({'native': run(F.inference_iterative_root_finding_joint), 'composite': run(F._inference_joint_autograd)},
                   args.steps, args.iters)
    print(json.dumps({'metric': 'joint_fit_npm', 'gpu': name, 'power_limit': power, 'points': '5 x 1000 per iteration',
                      'observations': args.obs, 'runs': args.steps, 'iterations_per_run': args.iters,
                      'native_ms_per_iter': ms['native'], 'composite_ms_per_iter': ms['composite'],
                      'speedup': ms['composite'] / ms['native'],
                      'timing': 'median over runs of CUDA-event time per iteration, native and composite alternated'}))


if __name__ == '__main__':
    main()
