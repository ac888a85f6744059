#!/usr/bin/env python
"""Data-parallel training steps (nphm_b200.training_sharded.train_step_sharded) at the tools/bench_train.py settings, on the
native paths: stage 1 of the NPHM ensemble at the nphm.yaml batch (32 x (750 + 50 + 800 + 93) points, --decoder nphm) or of
the NPM DeepSDF (--decoder npm), stage 2 with the `compress` deformation network and the `-mode npm` DeepSDF (32 x (1000 +
100) points).  Seeded weights, codes and batches (tests/train_sharded_common.py); the work does not depend on the values.

    torchrun --nproc_per_node 8 tools/bench_train_sharded.py --stage 1 --decoder nphm --steps 10 --warmup 2
    python tools/bench_train_sharded.py --local 8 --stage 1 --decoder nphm --steps 10 --warmup 2

Under torchrun every rank trains on its own GPU over NCCL; --local N runs LocalTrainGroup(N) on one GPU (the N shards in
sequence).  Per rank (rank 0 prints one JSON line): the median step time (CUDA events), the median time of the gradient
collective (the all-gather of the buckets; zero in one process), the peak device memory of the timed steps (torch's
allocator), and the largest difference, over the decoder's tensors and the codes, between the first step's reduced gradients
and those of the one-process native step on the same batch (max |sharded - one-process| / max |one-process|).  The one-process
peak memory is reported beside it."""
import argparse, json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import torch
import torch.distributed as dist


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--stage', type=int, choices=(1, 2), default=1)
    ap.add_argument('--decoder', choices=('nphm', 'npm'), default='nphm', help='stage 1: the ensemble or the NPM DeepSDF')
    ap.add_argument('--mode', choices=('compress', 'npm'), default='compress', help='stage 2: the expression decoder')
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--local', type=int, default=0, help='N > 0: LocalTrainGroup(N) in this process instead of torchrun ranks')
    args = ap.parse_args()
    if args.steps < 1:
        ap.error('--steps must be >= 1')
    if not torch.cuda.is_available():
        sys.exit('bench_train_sharded.py needs a CUDA device')
    import train_sharded_common as T
    from bench_train import gpu_info
    from nphm_b200 import training_sharded as S

    if args.local:
        group, rank, world = S.LocalTrainGroup(args.local), 0, args.local
        dev = torch.device('cuda', torch.cuda.current_device())
    else:
        rank = int(os.environ.get('LOCAL_RANK', 0))
        dev = torch.device('cuda', rank)
        torch.cuda.set_device(dev)
        dist.init_process_group('nccl', device_id=dev)
        group, rank, world = None, dist.get_rank(), dist.get_world_size()

    kind = ('nphm' if args.decoder == 'nphm' else 'npm') if args.stage == 1 else ('compress' if args.mode == 'compress' else 'expr_npm')

    def batch(step):
        return T.make_batch(kind, args.batch, step, sizes=(750, 50, 800, 93), n_points=1000)

    # the collective's time: CUDA events around the all-gather of the process group (none in one process)
    gather_ms = []
    orig_gather = S._ProcessTrainGroup.gather

    def timed_gather(self, buckets):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        out = orig_gather(self, buckets)
        ev[1].record()
        gather_ms.append(ev)
        return out
    S._ProcessTrainGroup.gather = timed_gather

    # first step's gradients against the one-process native step on the same batch and state (clipping off)
    grads = {}
    for name, world_run in (('one_process', None), ('sharded', group)):
        tr = T.make_trainer(kind, device=dev, dtype=torch.float32, big=True)
        tr.cfg = dict(tr.cfg, grad_clip=1e30, grad_clip_lat=1e30)
        torch.manual_seed(0)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        if world_run is None and name == 'one_process':
            tr.train_step(batch(0), 0)
        else:
            S.train_step_sharded(tr, batch(0), 0, group)
        torch.cuda.synchronize()
        grads[name] = (T.reduced_grads(tr), torch.cuda.max_memory_allocated(dev))
        del tr
        torch.cuda.empty_cache()
    diff = max(T.rel_err(grads['sharded'][0][k], v) for k, v in grads['one_process'][0].items())

    tr = T.make_trainer(kind, device=dev, dtype=torch.float32, big=True)
    torch.manual_seed(0)
    times = []
    gather_ms.clear()
    peak = 0
    for step in range(args.warmup + args.steps):
        b = batch(step)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        n_before = len(gather_ms)
        ev[0].record()
        S.train_step_sharded(tr, b, step, group)
        ev[1].record()
        torch.cuda.synchronize()
        if step >= args.warmup:
            times.append(ev[0].elapsed_time(ev[1]))
            peak = max(peak, torch.cuda.max_memory_allocated(dev))
        else:
            del gather_ms[n_before:]
    coll = [a.elapsed_time(b) for a, b in gather_ms]
    name, power = gpu_info()
    res = {'rank': rank, 'ms_step': float(torch.tensor(times).median()),
           'ms_gradient_collective': float(torch.tensor(coll).median()) if coll else 0.0,
           'peak_memory_gib': peak / 2 ** 30, 'one_process_peak_memory_gib': grads['one_process'][1] / 2 ** 30,
           'first_step_grad_max_rel_diff': diff}
    if args.local:
        per_rank = [res]
    else:
        per_rank = [None] * world
        dist.all_gather_object(per_rank, res)
    if rank == 0:
        print(json.dumps({'metric': 'stage%d_%s_train_step_sharded' % (args.stage, kind), 'gpu': name, 'power_limit': power,
                          'world': world, 'group': 'LocalTrainGroup(%d), one GPU' % world if args.local else 'NCCL, one GPU per rank',
                          'batch': args.batch, 'steps': args.steps, 'timing': 'median of CUDA-event times per step',
                          'ranks': per_rank}))
    if not args.local:
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
