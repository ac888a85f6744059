#!/usr/bin/env python
"""Expression fitting with a fixed identity code on one GPU.

    python tools/bench_fit_expression.py [--decoder {nphm,npm}] [--scans 1 4 16] [--iters 20] [--reps 3]

Three measurements, each printed as one JSON line with the card and its power limit:
  single    inference_expression_space against inference_iterative_root_finding_joint on the same 3 observations of 2500
            points (whole calls of --iters iterations: host sampling, schedule and the native steps), iterations/s;
  batched   the fixed-identity BatchedJointFitter (BatchedNpmJointFitter) step on S subjects of 3 observations against S
            fixed-identity JointFitter (NpmJointFitter) steps, points sampled once and not timed, scan-iterations/s;
  surface   (NPHM only) nphm_fit_surface_grad_batched with the point gradient, with and without the identity-code gradient,
            at S = 1 and 16 scans of 5 x 1000 points, ms per call.
Paths alternate --reps times in one process; CUDA events or a host clock after a device synchronise, median."""
import argparse, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np
import torch

LAMBDAS = {'surface': 2.0, 'reg_expr': 0.01, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
SCHEDULE = {'lr': {200: 2, 400: 2, 600: 2, 800: 2}, 'symm_dist': {200: 10, 500: 9999}, 'reg_glob': {200: 3, 600: 10},
            'reg_loc': {500: 3, 600: 10}, 'reg_expr': {600: 10}}


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name(0)


def observations(seed, dev, n=3):
    rng = np.random.RandomState(seed)
    return [torch.from_numpy((rng.randn(2500, 3) * 0.12 + np.array([0.0, 0.05, -0.1])).astype(np.float32)).to(dev)
            for _ in range(n)]


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--decoder', choices=['nphm', 'npm'], default='nphm')
    ap.add_argument('--scans', type=int, nargs='+', default=[1, 4, 16])
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    from nphm_b200 import _native
    from nphm_b200.models import fitting as F
    dev = torch.device('cuda:0')
    gpu = card()
    if args.decoder == 'nphm':
        from conftest import make_deformation, make_ensemble, sample_latent
        dec, expr = make_ensemble(0, device=dev).train(), make_deformation(dev)
        with torch.no_grad():                     # a usable deformation field from random weights (tools/bench_joint.py)
            expr.defDeepSDF.lin6.weight.mul_(0.05)
            expr.defDeepSDF.lin6.bias.mul_(0.05)
        z_id = sample_latent(3).to(dev).reshape(1, 1, -1)
        single_cls, batched_cls = F.JointFitter, F.BatchedJointFitter
    else:
        import npm_fit_common as N
        from nphm_b200.models.deepSDF import DeepSDF
        dec, expr = N.make_decoders(DeepSDF, dev)
        z_id = (torch.randn(dec.lat_dim, generator=torch.Generator().manual_seed(41)) * 0.05).to(dev).reshape(1, 1, -1)
        single_cls, batched_cls = F.NpmJointFitter, F.BatchedNpmJointFitter
    common = {'decoder': args.decoder, 'gpu': gpu, 'points': '5 x 1000 sampled per subject and iteration'}

    # ---------------------------------------------------------------- whole calls
    obs = observations(100, dev)
    n_steps = args.iters * 100
    runs = {'expression': lambda: F.inference_expression_space(dec, expr, z_id, obs, dict(LAMBDAS), n_steps, SCHEDULE, 0.01),
            'joint': lambda: F.inference_iterative_root_finding_joint(dec, expr, obs, dict(LAMBDAS), n_steps, SCHEDULE, 0.01)}
    for fn in runs.values():
        fn()                                      # warm-up: weights, workspaces
    times = {k: [] for k in runs}
    for _ in range(args.reps):
        for k, fn in runs.items():
            times[k].append(wall(fn))
    it_s = {k: args.iters / float(np.median(v)) for k, v in times.items()}
    print(json.dumps(dict(common, metric='fit_expression_single', iterations=args.iters,
                          expression_it_per_s=round(it_s['expression'], 2), joint_it_per_s=round(it_s['joint'], 2),
                          speedup=round(it_s['expression'] / it_s['joint'], 3))), flush=True)

    # ---------------------------------------------------------------- batched against sequential steps
    for S in args.scans:
        subjects = [observations(200 + k, dev) for k in range(S)]
        torch.manual_seed(0)
        samples = [F._sample_observations(s) for s in subjects]
        o_list, i_list = [o for o, _ in samples], [i.long().to(dev) for _, i in samples]
        bf = batched_cls(dec, expr, [3] * S, dev, fixed_identity=True)
        bf.z_id.copy_(z_id.reshape(1, -1).expand(S, -1))
        singles = []
        for _ in range(S):
            f = single_cls(dec, expr, 3, dev, fixed_identity=True)
            f.z_id.copy_(z_id.reshape(-1))
            singles.append(f)
        step_b = lambda: bf.step(o_list, i_list, LAMBDAS, 0.1, 0.01)
        step_s = lambda: [f.step(o, i, LAMBDAS, 0.1, 0.01) for f, o, i in zip(singles, o_list, i_list)]
        step_b(); step_s()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        tb, ts = [], []
        for _ in range(args.reps):
            tb.append(timed(step_b, args.iters))
            ts.append(timed(step_s, args.iters))
        mb, ms = float(np.median(tb)), float(np.median(ts))
        print(json.dumps(dict(common, metric='fit_expression_batched', S=S, batched_ms_per_iter=round(mb, 3),
                              sequential_ms_per_iter=round(ms, 3), batched_scan_it_per_s=round(1e3 * S / mb, 1),
                              sequential_scan_it_per_s=round(1e3 * S / ms, 1), speedup=round(ms / mb, 3),
                              peak_gb=round(torch.cuda.max_memory_allocated() / 1e9, 2))), flush=True)

    # ---------------------------------------------------------------- the surface term with and without the latent gradient
    if args.decoder != 'nphm':
        return
    eng, lib = dec.engine(), _native.lib()
    stream = torch.cuda.current_stream(dev).cuda_stream
    for S in (1, 16):
        n = 5000
        gen = torch.Generator().manual_seed(7)
        pts = (torch.randn(S, n, 3, generator=gen) * 0.12 + torch.tensor([0.0, 0.05, -0.1])).to(dev).contiguous()
        mask = torch.ones(S, n, dtype=torch.uint8, device=dev)
        z = z_id.reshape(1, -1).expand(S, -1).contiguous()
        ws = torch.empty(lib.nphm_fit_batch_workspace_bytes(eng.handle, S, n), dtype=torch.uint8, device=dev)
        terms, g_lat, g_pts = torch.empty(S, 8, device=dev), torch.empty(S, dec.lat_dim, device=dev), torch.empty_like(pts)

        def call(gl):
            _native.check(lib.nphm_fit_surface_grad_batched(eng.handle, pts.data_ptr(), mask.data_ptr(), S, n, z.data_ptr(), 0.1,
                                                            terms.data_ptr(), _native._ptr(gl), g_pts.data_ptr(),
                                                            ws.data_ptr(), ws.numel(), stream), 'nphm_fit_surface_grad_batched')
        with_lat, without = (lambda: call(g_lat)), (lambda: call(None))
        with_lat(); without()
        tw, tn = [], []
        for _ in range(args.reps):
            tw.append(timed(with_lat, 200))
            tn.append(timed(without, 200))
        mw, mn = float(np.median(tw)), float(np.median(tn))
        print(json.dumps(dict(common, metric='fit_surface_grad_latent', S=S, points_per_scan=n, with_latent_ms=round(mw, 4),
                              without_latent_ms=round(mn, 4), saved_fraction=round(1 - mn / mw, 3))), flush=True)


if __name__ == '__main__':
    main()
