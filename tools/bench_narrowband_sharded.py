#!/usr/bin/env python
"""Narrow-band mesh extraction sharded in x-slabs (extract_mesh_narrowband_sharded) against the one-GPU band
(extract_mesh_narrowband), in eval mode.

    torchrun --nproc_per_node 1 tools/bench_narrowband_sharded.py [--res 256 512] [--decoders nphm npm] [--slabs 2 4 8]
                                                                  [--reps 3] [--warmup 1]

One process per GPU (NCCL); without torchrun it runs as a world of one.  Per (decoder, res) it times, alternating, the one-GPU
band, the sharded path on the torchrun world, and every slab count of --slabs driven by rank 0 alone on its GPU
(extract_mesh_narrowband_slabs: the exchange protocol and the per-slab launches without a second GPU, i.e. its overhead).  Each
number is the median host time of whole calls (all end with the mesh on the host of rank 0) over --reps after --warmup.  Rank 0
prints one JSON line per (decoder, res) with the times, their ratio to the one-GPU band, the stats of tools/bench_narrowband.py,
the bytes each rank sent per plane exchange, whether every mesh is identical to the one-GPU band's, and the card, its power
limit and SM clock read in the same run.  Decoders as in tools/bench_narrowband.py."""
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
import torch.distributed as dist

CHUNK = 25000


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader', '-i',
                          str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--res', type=int, nargs='+', default=[256, 512])
    ap.add_argument('--decoders', nargs='+', default=['nphm', 'npm'], choices=['nphm', 'npm'])
    ap.add_argument('--slabs', type=int, nargs='*', default=[2, 4, 8])
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_narrowband_sharded needs a CUDA device')
    for k, v in (('RANK', '0'), ('WORLD_SIZE', '1'), ('LOCAL_RANK', '0'), ('MASTER_ADDR', '127.0.0.1'), ('MASTER_PORT', '29533')):
        os.environ.setdefault(k, v)
    dev = torch.device('cuda', int(os.environ['LOCAL_RANK']))
    torch.cuda.set_device(dev)
    dist.init_process_group('nccl', device_id=dev)
    rank, world = dist.get_rank(), dist.get_world_size()
    try:
        run(args, dev, rank, world)
    finally:
        dist.destroy_process_group()


def run(args, dev, rank, world):
    from conftest import MAXI, MINI, make_ensemble, sample_latent
    from narrowband_common import make_npm_head
    from nphm_b200.distributed import extract_mesh_narrowband_sharded
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband, extract_mesh_narrowband_slabs
    for name in args.decoders:
        if name == 'nphm':
            dec, lat = make_ensemble(0, device=dev).eval(), sample_latent(1).to(dev)
        else:
            dec, lat = make_npm_head(dev)
        for res in args.res:
            kw = dict(nbatch_points=CHUNK, return_stats=True)
            paths = [('band', True, lambda: extract_mesh_narrowband(dec, lat, MINI, MAXI, res, **kw)),
                     ('sharded', False, lambda: extract_mesh_narrowband_sharded(dec, lat, MINI, MAXI, res, **kw))]
            paths += [('slabs%d' % k, True, (lambda k=k: extract_mesh_narrowband_slabs(dec, lat, MINI, MAXI, res, k, **kw)))
                      for k in args.slabs]
            times = {key: [] for key, _, _ in paths}
            outs = {}
            for it in range(args.warmup + args.reps):
                for key, rank0_only, fn in paths:
                    if rank0_only and rank != 0:
                        continue
                    torch.cuda.synchronize()
                    if not rank0_only:
                        dist.barrier()
                    t0 = time.perf_counter()
                    outs[key] = fn()
                    torch.cuda.synchronize()
                    if it >= args.warmup:
                        times[key].append((time.perf_counter() - t0) * 1e3)
            dist.barrier()
            if rank == 0:
                ref, st = outs['band']
                line = {'metric': 'narrowband_sharded_mesh', 'decoder': name, 'res': res, 'nbatch_points': CHUNK, 'world': world,
                        'card': card(), 'evaluated_fraction': round(st['voxels_evaluated'] / st['voxels_total'], 4),
                        'blocks_active': st['blocks_active'], 'blocks_total': st['blocks_total'],
                        'growth_rounds': st['growth_rounds'], 'margin': st['margin'], 'vertices': len(ref.vertices)}
                band_ms = float(np.median(times['band']))
                for key, _, _ in paths:
                    ms = float(np.median(times[key]))
                    mesh, s = outs[key]
                    line[key + '_ms_per_mesh'] = round(ms, 2)
                    line[key + '_ms_all'] = [round(t, 2) for t in times[key]]
                    if key != 'band':
                        line[key + '_vs_band'] = round(ms / band_ms, 4)
                        line[key + '_identical'] = bool(np.array_equal(np.asarray(mesh.faces), np.asarray(ref.faces))
                                                        and np.array_equal(np.asarray(mesh.vertices), np.asarray(ref.vertices)))
                        line[key + '_voxels_evaluated'] = s['voxels_evaluated']
                        line[key + '_blocks_active'] = s['blocks_active']
                        line[key + '_growth_rounds'] = s['growth_rounds']
                        line[key + '_bytes_exchanged'] = s['bytes_exchanged']
                print(json.dumps(line), flush=True)
            outs.clear()
            torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
