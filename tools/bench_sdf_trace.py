#!/usr/bin/env python
"""Sphere tracing (render_sdf_views, csrc/sdf_trace.cu) against meshing plus rasterizing, on the seeded ensemble head.

    python tools/bench_sdf_trace.py [--reps 3] [--warmup 1] [--out results/bench_sdf_trace.jsonl]

Measured, each as the median of --reps calls that alternate between the arms (host clock around calls that end in a
synchronise, after --warmup calls of every arm), with the card and its power limit read in the same run:
  * trace, one 512 x 512 view and the 10 evaluation views at 1280 x 960 (scale 4): ms, rays/s, steps per ray (mean, p99);
  * mesh path, the same images: extract_mesh_narrowband at 256^3 and at 1024^3 (sparse) plus render_views;
  * posed (compress deformation network, 2 expressions, the 512 x 512 view): ms per expression.
Prints one JSON line per measurement."""
import argparse, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np
import torch


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name(0)


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_sdf_trace needs a CUDA device')
    from conftest import MAXI, MINI, make_ensemble, sample_latent
    import posed_common as P
    from nphm_b200.evaluation.render_utils import KK, render_cameras, render_sdf_views, render_views
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband
    dev = torch.device('cuda:0')
    dec = make_ensemble(0, device=dev).train()
    lat = sample_latent(1).to(dev)
    _, poses = render_cameras(10)
    K512 = np.array([[1000.0, 0, 256], [0, 1000.0, 256], [0, 0, 1]])
    cases = {'1x512x512': ([poses[0]], K512, (512, 512)), '10x1280x960': (poses, KK, (1280, 960))}
    info = card()
    lines = []

    def emit(d):
        d['card'] = info
        print(json.dumps(d), flush=True)
        lines.append(d)

    def mesh_arm(res, sparse, views):
        def run():
            m = extract_mesh_narrowband(dec, lat.reshape(1, 1, -1), MINI, MAXI, res, sparse=sparse)
            return render_views(np.asarray(m.vertices) / 4, m.faces, views[0], views[1], views[2])
        return run

    for name, views in cases.items():
        arms = {'trace': lambda v=views: render_sdf_views(dec, lat, v[0], v[1], v[2], scale=4.0, return_stats=True),
                'mesh256+render': mesh_arm(256, False, views), 'mesh1024sparse+render': mesh_arm(1024, True, views)}
        times = {k: [] for k in arms}
        for _ in range(a.warmup):
            for fn in arms.values():
                timed(fn)
        stats = None
        for _ in range(a.reps):
            for k, fn in arms.items():
                ms, out = timed(fn)
                times[k].append(ms)
                if k == 'trace':
                    stats = out[2]
        n_rays = len(views[0]) * views[2][0] * views[2][1]
        tr = float(np.median(times['trace']))
        emit(dict(case=name, arm='trace', ms=tr, rays_per_s=n_rays / tr * 1e3, steps_mean=stats['steps_mean'],
                  steps_p99=stats['steps_p99'], n_hit=stats['n_hit'], n_out_of_steps=stats['n_out_of_steps'], reps=times['trace']))
        for k in ('mesh256+render', 'mesh1024sparse+render'):
            emit(dict(case=name, arm=k, ms=float(np.median(times[k])), reps=times[k]))

    dec_p, dfn, lat_p, z_ex, _, _ = P.ensemble_case(dev, training=True)
    v = cases['1x512x512']
    fn = lambda: render_sdf_views(dec_p, lat_p, v[0], v[1], v[2], scale=4.0, decoder_expr=dfn, lat_reps_expr=z_ex,  # noqa: E731
                                  return_stats=True)
    for _ in range(a.warmup):
        timed(fn)
    ts = []
    for _ in range(a.reps):
        ms, out = timed(fn)
        ts.append(ms)
    st = out[2]
    emit(dict(case='posed-1x512x512', arm='trace', expressions=int(z_ex.shape[0]), ms=float(np.median(ts)),
              ms_per_expression=float(np.median(ts)) / z_ex.shape[0], steps_mean=st['steps_mean'], steps_p99=st['steps_p99'],
              n_hit=st['n_hit'], n_invalid=st['n_invalid'], n_out_of_steps=st['n_out_of_steps'], reps=ts))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            for d in lines:
                f.write(json.dumps(d) + '\n')


if __name__ == '__main__':
    main()
