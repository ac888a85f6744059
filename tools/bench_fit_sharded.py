#!/usr/bin/env python
"""Many scans fitted over several GPUs (nphm_b200.fitting_sharded): the chunk plan, each rank's fit time, subjects per hour,
peak memory and the host time of the sampling walk.

    torchrun --nproc_per_node 8 tools/bench_fit_sharded.py --mode joint --subjects 32 --batch-size 8 --iters 100
    python tools/bench_fit_sharded.py --world 8 --mode joint --subjects 32 --batch-size 8 --iters 100
    python tools/bench_fit_sharded.py --world 1 --mode joint --subjects 16 --batch-size 8 --iters 100 --reps 3

Subjects are synthetic (--expressions observations of --points points each, seeded); the work does not depend on the values.
--iters iterations of the reference's schedule (fitting_pointclouds.py's 1000 steps at step_scale = iters / 1000).
--decoder npm: the NPM baseline's DeepSDF decoders (tests/npm_fit_common.py) instead of the NPHM ensemble.

Under torchrun every rank fits its chunks on its own GPU over NCCL (`timings=` of the sharded call).  --world N > 1 runs the
N ranks' chunks one after another in this process: each rank's time is that of `inference_*_batched` on its chunks, which is
what the rank computes.  --world 1 alternates, --reps times, the sharded call at world 1 against the existing batched call
on the same chunks (one call per chunk of --batch-size subjects) and reports both with the largest difference of their
results (the native fitting kernels sum with float atomics, so two runs of either differ in the last bits).  Subjects per
hour take the slowest rank's time, the sampling walk and the exchange included.  Rank 0 prints
one JSON line with the card, its power limit and its SM clock."""
import argparse, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np
import torch
import torch.distributed as dist

LAMBDAS = {'surface': 2.0, 'reg_expr': 0.01, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
SCHEDULE = {'lr': {200: 2, 400: 2, 600: 2, 800: 2}, 'symm_dist': {200: 10, 500: 9999}, 'reg_glob': {200: 3, 600: 10},
            'reg_loc': {500: 3, 600: 10}, 'reg_expr': {600: 10}}


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader',
                          '-i', str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name()


def make_subjects(n, expressions, points, dev):
    out = []
    for k in range(n):
        rng = np.random.RandomState(100 + k)
        out.append([torch.from_numpy((rng.randn(points, 3) * 0.12 + np.array([0.0, 0.05, -0.1])).astype(np.float32)).to(dev)
                    for _ in range(expressions)])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--mode', choices=['identity', 'joint'], default='joint')
    ap.add_argument('--decoder', choices=['nphm', 'npm'], default='nphm')
    ap.add_argument('--subjects', type=int, default=16)
    ap.add_argument('--expressions', type=int, default=3)
    ap.add_argument('--points', type=int, default=2500)
    ap.add_argument('--batch-size', type=int, default=8)
    ap.add_argument('--iters', type=int, default=100)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--world', type=int, default=0, help='N > 0: the N ranks in this process instead of torchrun ranks')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_fit_sharded.py needs a CUDA device')
    from nphm_b200 import fitting_sharded as S
    from nphm_b200.models import fitting as F
    from conftest import make_deformation, make_ensemble

    if args.world:
        rank, world = 0, args.world
        dev = torch.device('cuda', torch.cuda.current_device())
    else:
        rank = int(os.environ.get('LOCAL_RANK', 0))
        dev = torch.device('cuda', rank)
        torch.cuda.set_device(dev)
        dist.init_process_group('nccl', device_id=dev)
        rank, world = dist.get_rank(), dist.get_world_size()
    if args.decoder == 'npm':
        import npm_fit_common
        from nphm_b200.models.deepSDF import DeepSDF
        dec, dfn = npm_fit_common.make_decoders(DeepSDF, dev)
    else:
        dec, dfn = make_ensemble(0, device=dev).train(), make_deformation(dev)
    subjects = make_subjects(args.subjects, args.expressions, args.points, dev)
    lam0 = LAMBDAS if args.mode == 'joint' else {k: v for k, v in LAMBDAS.items() if k != 'reg_expr'}
    step_scale = args.iters / 1000.0
    costs = [len(s) for s in subjects] if args.mode == 'joint' else [1] * len(subjects)

    def batched(chunk):
        if args.mode == 'joint':
            return F.inference_iterative_root_finding_joint_batched(dec, dfn, chunk, dict(lam0), 1000, SCHEDULE, step_scale)
        return F.inference_identity_space_batched(dec, chunk, dict(lam0), 1000, SCHEDULE, step_scale)

    def sharded(group, timings):
        if args.mode == 'joint':
            return S.inference_iterative_root_finding_joint_batched_sharded(dec, dfn, subjects, dict(lam0), 1000, SCHEDULE,
                                                                            step_scale, group=group,
                                                                            batch_size=args.batch_size, timings=timings)
        return S.inference_identity_space_batched_sharded(dec, subjects, dict(lam0), 1000, SCHEDULE, step_scale, group=group,
                                                          batch_size=args.batch_size, timings=timings)

    def clock(fn):
        torch.cuda.synchronize(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize(dev)
        return out, time.perf_counter() - t0, torch.cuda.max_memory_allocated(dev)

    plan = S.plan_fit_chunks(costs, args.batch_size, world)
    walks = []
    for n_iters in (args.iters, 1000):                                # this run's walk, and the reference's 1000 iterations
        t0 = time.perf_counter()
        F._sampling_plan(subjects, n_iters)
        walks.append(time.perf_counter() - t0)
    walk_s = walks[0]
    batched(subjects[:min(2, len(subjects))])                        # warm-up: modules, packed weights, workspaces
    res = {'metric': 'fit_%s_sharded' % args.mode, 'decoder': args.decoder, 'card': card(), 'world': world,
           'subjects': args.subjects, 'expressions': args.expressions, 'points': args.points, 'batch_size': args.batch_size,
           'iters': args.iters, 'plan': [[lo, hi, r] for (lo, hi), r in zip(plan.chunks, plan.owners)],
           'sampling_walk_s': round(walk_s, 4), 'sampling_walk_1000_iters_s': round(walks[1], 4)}
    if not args.world:
        tm = {}
        _, total, peak = clock(lambda: sharded(None, tm))
        ranks = [None] * world
        dist.all_gather_object(ranks, dict(tm, total_s=total, peak_gib=peak / 2 ** 30))
        res.update(group='NCCL, one GPU per rank', ranks=ranks,
                   subjects_per_hour=round(3600 * args.subjects / max(r['total_s'] for r in ranks), 1))
    elif world == 1:
        times = {'sharded': [], 'batched': []}
        peaks = {}
        for _ in range(args.reps):
            tm = {}
            a, t, peaks['sharded'] = clock(lambda: (torch.manual_seed(0), sharded(None, tm))[1])
            times['sharded'].append(dict(tm, total_s=t))
            b, t, peaks['batched'] = clock(lambda: (torch.manual_seed(0),
                                                    [r for lo, hi in plan.chunks for r in batched(subjects[lo:hi])])[1])
            times['batched'].append(t)
        diff = max(float((x - y).detach().abs().max()) for ra, rb in zip(a, b) for x, y in zip(ra, rb) if x is not None)
        med = float(np.median([t['total_s'] for t in times['sharded']]))
        med_b = float(np.median(times['batched']))
        res.update(group='world 1, no process group', sharded_s=[round(t['total_s'], 4) for t in times['sharded']],
                   batched_s=[round(t, 4) for t in times['batched']], sharded_median_s=round(med, 4),
                   batched_median_s=round(med_b, 4), difference_s=round(med - med_b, 4),
                   sharded_timings=[{k: round(v, 4) for k, v in t.items()} for t in times['sharded']],
                   peak_gib={k: round(v / 2 ** 30, 3) for k, v in peaks.items()}, max_abs_diff=diff,
                   subjects_per_hour=round(3600 * args.subjects / med, 1))
    else:
        ranks = []
        for r in range(world):
            mine = [(lo, hi) for (lo, hi), o in zip(plan.chunks, plan.owners) if o == r]
            _, t, peak = clock(lambda: [batched(subjects[lo:hi]) for lo, hi in mine])
            ranks.append({'rank': r, 'chunks': mine, 'fit_s': round(t, 4), 'peak_gib': round(peak / 2 ** 30, 3)})
        slowest = max(r['fit_s'] for r in ranks) + walk_s
        res.update(group='%d ranks in one process, one after another' % world, ranks=ranks,
                   subjects_per_hour=round(3600 * args.subjects / slowest, 1))
    if rank == 0:
        print(json.dumps(res), flush=True)
    if not args.world:
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
