#!/usr/bin/env python
"""BASELINE.json configs[3]: identity fitting of a batch of scans, ONE SCAN PER GPU (replicas only, no collective).

    python tools/bench_fit.py --steps 200                                   # 1 GPU
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port P tools/bench_fit.py

Every rank fits its own synthetic scan (3 observations x 2500 points, seed 100 + rank) with the reference's loop
(`inference_identity_space`, 5 x 1000 sampled points per iteration, reference schedule) on the fused fitting kernels.
Prints one JSON line on rank 0: iterations/s and scans/hour over all ranks (time = max over ranks).

    python tools/bench_fit.py --decoder npm --steps 10 [--iters 20]

The NPM baseline of fitting_npm.yaml (DeepSDF 515 -> 1024 x 8 -> 1, seeded as in tests/npm_fit_common.py) on one GPU: native
(NpmIdentityFitter) and composite (autograd) runs of `--iters` iterations alternate `--steps` times; median ms per iteration
of each, with the card and its power limit.

    python tools/bench_fit.py --eval --steps 10 [--iters 20]

The same comparison for the NPHM ensemble left in eval mode: the native fitter with the eval-mode quirk rows against the
autograd fallback (`_inference_identity_space_autograd`) that such a decoder took before."""
import argparse, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np
import torch
import torch.distributed as dist


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=1000)
    ap.add_argument('--sharded', action='store_true',
                    help='ONE head, the sampled points of every iteration sharded over the ranks, one all-reduce per iteration '
                         '(nphm_b200.distributed.inference_identity_space_sharded) instead of one scan per GPU')
    ap.add_argument('--decoder', choices=('nphm', 'npm'), default='nphm')
    ap.add_argument('--iters', type=int, default=20, help='--decoder npm / --eval: iterations per timed run')
    ap.add_argument('--eval', action='store_true',
                    help='one GPU, the NPHM ensemble in eval mode: native fitter against the autograd fallback')
    args = ap.parse_args()
    if args.eval:
        if args.decoder != 'nphm' or args.sharded:
            ap.error('--eval: the NPHM ensemble on one GPU only')
        return bench_eval(args)
    if args.decoder == 'npm':
        return bench_npm(args)
    from conftest import make_ensemble
    from nphm_b200.models.fitting import inference_identity_space
    world = int(os.environ.get('WORLD_SIZE', '1')); rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    if world > 1:
        dist.init_process_group('nccl', device_id=dev)
    dec = make_ensemble(0, device=dev).train()
    rng = np.random.RandomState(100 + (0 if args.sharded else rank))
    obs = [torch.from_numpy((rng.randn(2500, 3) * 0.12 + np.array([0.0, 0.05, -0.1])).astype(np.float32)).to(dev) for _ in range(3)]
    lambdas = {'surface': 2.0, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
    schedule = {'lr': {200: 2, 400: 2, 600: 2, 800: 2}, 'symm_dist': {200: 10, 500: 9999}, 'reg_glob': {200: 3, 600: 10},
                'reg_loc': {500: 3, 600: 10}}
    if args.sharded:
        from nphm_b200.distributed import inference_identity_space_sharded
        if world == 1 and not dist.is_initialized():
            if 'MASTER_ADDR' in os.environ and 'RANK' in os.environ:
                dist.init_process_group('nccl', device_id=dev)
            else:
                dist.init_process_group('nccl', device_id=dev, init_method='tcp://127.0.0.1:29533', rank=0, world_size=1)

        def fit(n):
            return inference_identity_space_sharded(dec, obs, dict(lambdas), n_steps=n, schedule_cfg=schedule)
    else:
        def fit(n):
            return inference_identity_space(dec, obs, dict(lambdas), n_steps=n, schedule_cfg=schedule)
    np.random.seed(0); torch.manual_seed(0)
    fit(5)                                                                                        # warm-up
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize(); t0 = time.perf_counter()
    np.random.seed(0); torch.manual_seed(0)
    z, _ = fit(args.steps)
    torch.cuda.synchronize(); dt = torch.tensor([time.perf_counter() - t0], device=dev)
    if world > 1:
        dist.all_reduce(dt, op=dist.ReduceOp.MAX)
    if rank == 0:
        print(json.dumps({'metric': 'identity_fit', 'n_gpus': world, 'iterations': args.steps, 's_per_scan': dt.item(),
                          'iters_per_s_total': world * args.steps / dt.item(), 'scans_per_hour': world * 3600 / dt.item(),
                          'finite': bool(torch.isfinite(z).all()),
                          'scaling': ('strong: one head, points sharded, 1 all-reduce of lat_dim + 2 floats per iteration; '
                                      'iters_per_s_total / n_gpus = iterations/s of that head') if args.sharded
                          else 'replicas (one scan per GPU, no collective)'}))
    if dist.is_initialized():
        dist.destroy_process_group()


def bench_eval(args):
    """inference_identity_space with the NPHM ensemble in eval mode: the native fitter (the fused step with the eval-mode quirk
    rows) against the autograd fallback it replaces, 5 x 1000 points per iteration."""
    from bench_joint import alternate
    from bench_train import gpu_info
    from conftest import make_ensemble
    from nphm_b200.models import fitting as F
    dev = torch.device('cuda', torch.cuda.current_device())
    dec = make_ensemble(0, device=dev).eval()
    assert F._fused_identity(dec)
    lambdas = {'surface': 2.0, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
    schedule = {'lr': {200: 2, 400: 2, 600: 2, 800: 2}, 'symm_dist': {200: 10, 500: 9999},
                'reg_glob': {200: 3, 600: 10}, 'reg_loc': {500: 3, 600: 10}}
    rng = np.random.RandomState(100)
    obs = [torch.from_numpy((rng.randn(2500, 3) * 0.1 + np.array([0.0, 0.05, -0.1])).astype(np.float32)).to(dev) for _ in range(3)]

    def run(fn):
        def go(n):
            np.random.seed(0); torch.manual_seed(0)
            return fn(dec, obs, dict(lambdas), n, schedule)
        return go

    name, power = gpu_info()
    ms = alternate({'native': run(F.inference_identity_space), 'composite': run(F._inference_identity_space_autograd)},
                   args.steps, args.iters)
    print(json.dumps({'metric': 'identity_fit_eval_mode', 'gpu': name, 'power_limit': power,
                      'points': '5 x 1000 per iteration', 'runs': args.steps, 'iterations_per_run': args.iters,
                      'native_ms_per_iter': ms['native'], 'composite_ms_per_iter': ms['composite'],
                      'native_iters_per_s': 1000.0 / ms['native'], 'composite_iters_per_s': 1000.0 / ms['composite'],
                      'speedup': ms['composite'] / ms['native'],
                      'timing': 'median over runs of CUDA-event time per iteration, native and composite alternated'}))


def bench_npm(args):
    from bench_joint import alternate
    from bench_train import gpu_info
    from npm_fit_common import LAMBDAS_IDENTITY, SCHEDULE, make_decoders
    from nphm_b200.models import fitting as F
    from nphm_b200.models.deepSDF import DeepSDF
    dev = torch.device('cuda', torch.cuda.current_device())
    dec, _ = make_decoders(DeepSDF, dev)
    assert F._native_npm_decoder(dec, 1)
    rng = np.random.RandomState(100)
    obs = [torch.from_numpy((rng.randn(2500, 3) * 0.1 + np.array([0.0, 0.05, -0.1])).astype(np.float32)).to(dev) for _ in range(3)]

    def run(fn):
        def go(n):
            np.random.seed(0); torch.manual_seed(0)
            return fn(dec, obs, dict(LAMBDAS_IDENTITY), n, SCHEDULE)
        return go

    name, power = gpu_info()
    ms = alternate({'native': run(F.inference_identity_space), 'composite': run(F._inference_identity_space_autograd)},
                   args.steps, args.iters)
    print(json.dumps({'metric': 'identity_fit_npm', 'gpu': name, 'power_limit': power, 'points': '5 x 1000 per iteration',
                      'runs': args.steps, 'iterations_per_run': args.iters, 'native_ms_per_iter': ms['native'],
                      'composite_ms_per_iter': ms['composite'], 'speedup': ms['composite'] / ms['native'],
                      'timing': 'median over runs of CUDA-event time per iteration, native and composite alternated'}))


if __name__ == '__main__':
    main()
