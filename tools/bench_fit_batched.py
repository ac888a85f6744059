#!/usr/bin/env python
"""Scan-batched fitting on one GPU: S scans in one launch sequence per iteration against the sequential native path.

    python tools/bench_fit_batched.py [--decoder {nphm,npm}] [--scans 1 2 4 8 16] [--iters 50] [--reps 3] [--profile DIR]

Identity: BatchedIdentityFitter.step on S scans of 5 x 1000 points vs S IdentityFitter.step calls.  Joint:
BatchedJointFitter.step on S subjects (3 observations each, 5 x 1000 sampled points) vs S JointFitter.step calls.
--decoder npm: the NPM baseline's DeepSDF decoders (515 -> 1024 x 8 -> 1 and 715 -> 1024 x 8 -> 3, tests/npm_fit_common.py)
with BatchedNpmIdentityFitter / BatchedNpmJointFitter against NpmIdentityFitter / NpmJointFitter; its JSON lines carry
"decoder": "npm".  The points
are sampled once per configuration (host sampling is the same for both paths and not timed).  Batched and sequential runs of
`--iters` iterations alternate `--reps` times; CUDA events, median.  Prints one JSON line per (mode, S): scan-iterations/s of
both paths, peak device memory of the batched run, the card and its power limit.  --profile DIR: a torch.profiler kernel table
of 10 batched identity and joint iterations at S = 4 (a run of its own, after the timings)."""
import argparse, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np
import torch

LAMBDAS = {'surface': 2.0, 'reg_expr': 0.01, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name(0)


def subjects(S, dev):
    out = []
    for k in range(S):
        rng = np.random.RandomState(100 + k)
        out.append([torch.from_numpy((rng.randn(2500, 3) * 0.12 + np.array([0.0, 0.05, -0.1])).astype(np.float32)).to(dev)
                    for _ in range(3)])
    return out


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
    ap.add_argument('--decoder', choices=['nphm', 'npm'], default='nphm')
    ap.add_argument('--scans', type=int, nargs='+', default=[1, 2, 4, 8, 16])
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--profile', default=None)
    args = ap.parse_args()
    from conftest import make_deformation, make_ensemble
    from nphm_b200.models.fitting import (BatchedIdentityFitter, BatchedJointFitter, BatchedNpmIdentityFitter,
                                          BatchedNpmJointFitter, IdentityFitter, JointFitter, NpmIdentityFitter, NpmJointFitter,
                                          _sample_observations)
    dev = torch.device('cuda:0')
    if args.decoder == 'npm':
        import npm_fit_common
        from nphm_b200.models.deepSDF import DeepSDF
        dec, dfn = npm_fit_common.make_decoders(DeepSDF, dev)
        BId, Id, BJoint, Joint = BatchedNpmIdentityFitter, NpmIdentityFitter, BatchedNpmJointFitter, NpmJointFitter
    else:
        dec = make_ensemble(0, device=dev).train()
        dfn = make_deformation(dev)
        BId, Id, BJoint, Joint = BatchedIdentityFitter, IdentityFitter, BatchedJointFitter, JointFitter
    tag = {'decoder': 'npm'} if args.decoder == 'npm' else {}
    name = card()

    def setups(S):
        subs = subjects(S, dev)
        torch.manual_seed(0)
        samples = [_sample_observations(s) for s in subs]
        obs = [o for o, _ in samples]
        idx = [i.long().to(dev) for _, i in samples]
        bf = BId(dec, S, dev)
        singles = [Id(dec, dev) for _ in range(S)]
        bj = BJoint(dec, dfn, [3] * S, dev)
        jsingles = [Joint(dec, dfn, 3, dev) for _ in range(S)]
        return {
            'identity': (lambda: bf.step(obs, LAMBDAS, 0.1, 0.01),
                         lambda: [f.step(o, LAMBDAS, 0.1, 0.01) for f, o in zip(singles, obs)]),
            'joint': (lambda: bj.step(obs, idx, LAMBDAS, 0.1, 0.01),
                      lambda: [f.step(o, i, LAMBDAS, 0.1, 0.01) for f, o, i in zip(jsingles, obs, idx)]),
        }

    for S in args.scans:
        runs = setups(S)
        for mode, (batched, sequential) in runs.items():
            batched(); sequential()                                   # warm-up: workspaces, packed weights, modules
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            tb, ts = [], []
            for _ in range(args.reps):
                tb.append(timed(batched, args.iters))
                ts.append(timed(sequential, args.iters))
            peak_b = torch.cuda.max_memory_allocated(dev)
            mb, ms = float(np.median(tb)), float(np.median(ts))
            print(json.dumps({**tag, 'mode': mode, 'scans': S, 'batched_ms_per_iter': round(mb, 4),
                              'sequential_ms_per_iter': round(ms, 4),
                              'batched_scan_it_per_s': round(1000.0 * S / mb, 1),
                              'sequential_scan_it_per_s': round(1000.0 * S / ms, 1),
                              'speedup': round(ms / mb, 3), 'peak_mem_gb': round(peak_b / 1e9, 3),
                              'spread_batched_ms': [round(min(tb), 4), round(max(tb), 4)], 'card': name}), flush=True)
        del runs
        torch.cuda.empty_cache()

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(args.profile, exist_ok=True)
        runs = setups(4)
        for mode, (batched, _) in runs.items():
            batched(); torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                for _ in range(10):
                    batched()
                torch.cuda.synchronize()
            prefix = 'fit_batched_npm' if args.decoder == 'npm' else 'fit_batched'
            with open(os.path.join(args.profile, '%s_%s_S4.txt' % (prefix, mode)), 'w') as f:
                f.write('%s, 10 batched iterations at S = 4\n' % ', '.join([name] + list(tag.values())))
                f.write(prof.key_averages().table(sort_by='cuda_time_total', row_limit=30))


if __name__ == '__main__':
    main()
