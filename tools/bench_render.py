#!/usr/bin/env python
"""Native depth / normal rendering (nphm_render_depth_normals) at 1280 x 960, the size of gen_render_samples.

    python tools/bench_render.py [--reps 20] [--warmup 3] [--res 256]

Meshes, all scaled by 1/4 as gen_render_samples scales them, seen from its 10 cameras:
  (a) head: the zero level set of the golden ensemble (tests/conftest.py make_ensemble) at res^3;
  (b) (a) plus, behind the head, one quad that covers the first view's whole viewport (and much of the others');
  (b10) (a) plus one such quad per view;
  (c) a UV sphere of about 10 M triangles, standing in for a raw scan.
For each: one view, and the 10-view launch of gen_render_samples - median over --reps of CUDA-event times after --warmup calls,
triangles per second (faces x views / time), peak device memory of the 10-view call.  Then sample_surface_points end to end on
(a) (render, post-processing, slicing, nearest neighbours, the copy to the host; host clock around the synchronous call).  Prints
one JSON line per measurement, with the card and its power limit read in the same run."""
import argparse, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np
import torch


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name(0)


def head(res, dev):
    from conftest import MAXI, MINI, make_ensemble, sample_latent
    from nphm_b200.models.reconstruction import get_logits
    from nphm_b200.utils.reconstruction import create_grid_points_from_bounds, mesh_from_logits
    dec = make_ensemble(0, device=dev).eval()
    grid = torch.from_numpy(create_grid_points_from_bounds(MINI, MAXI, res)).to(dev, dtype=torch.float).reshape(1, -1, 3)
    mesh = mesh_from_logits(get_logits(dec, sample_latent(1).to(dev), grid, nbatch_points=1 << 22), MINI, MAXI, res)
    return np.asarray(mesh.vertices) / 4, np.asarray(mesh.faces).astype(np.int64)


def backdrops(v, f, cams):
    """One 10 x 10 quad per given camera, facing it, 0.6 behind the origin: full viewport in that camera's view."""
    V, F = [v], [f]
    n = len(v)
    for c in cams:
        c = np.asarray(c)
        u = np.cross([0.0, 1.0, 0.0], c); u /= np.linalg.norm(u)
        w = np.cross(c, u)
        o = -0.6 * c
        V.append(np.stack([o - 5 * u - 5 * w, o + 5 * u - 5 * w, o + 5 * u + 5 * w, o - 5 * u + 5 * w]))
        F.append(np.array([(0, 1, 2), (0, 2, 3)]) + n)
        n += 4
    return np.concatenate(V), np.concatenate(F)


def uv_sphere(n_tri, radius=0.2):
    k = int(np.sqrt(n_tri / 2))
    th, ph = np.meshgrid(np.linspace(0, np.pi, k + 1), np.linspace(0, 2 * np.pi, k + 1), indexing='ij')
    v = radius * np.stack([np.sin(th) * np.cos(ph), np.cos(th), np.sin(th) * np.sin(ph)], -1).reshape(-1, 3)
    i, j = np.meshgrid(np.arange(k), np.arange(k), indexing='ij')
    a = (i * (k + 1) + j).reshape(-1); b = a + 1; c = a + k + 1; d = c + 1
    return v, np.concatenate([np.stack([a, c, b], 1), np.stack([b, c, d], 1)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--res', type=int, default=256)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_render needs a CUDA device')
    from nphm_b200 import _native
    from nphm_b200.evaluation import render_utils as ru
    from nphm_b200.evaluation import sampling
    from nphm_b200.utils.mesh import SimpleMesh
    dev = torch.device('cuda:0')
    gpu = card()
    cams, poses = ru.render_cameras(10)
    w2e = torch.from_numpy(np.stack([np.linalg.inv(p)[:3] for p in poses]))
    k = ru.KK.astype(np.float64)
    intr = torch.from_numpy(np.tile([k[0][0], k[1][1], k[0][2], k[1][2]], (10, 1)))
    hv, hf = head(args.res, dev)
    scenes = {'a_head_%d' % args.res: (hv, hf), 'b_head_plus_fullview_quad': backdrops(hv, hf, cams[:1]),
              'b10_head_plus_quad_per_view': backdrops(hv, hf, cams), 'c_uv_sphere_10M': uv_sphere(10_000_000)}
    times = {}
    for name, (v, f) in scenes.items():
        vt = torch.from_numpy(v.astype(np.float32)).to(dev)
        ft = torch.from_numpy(f.astype(np.int32)).to(dev)
        for views in (1, 10):
            call = lambda: _native.render_depth_normals(vt, ft, w2e[:views], intr[:views], 1280, 960)   # noqa: E731
            for _ in range(args.warmup):
                call()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            base = torch.cuda.memory_allocated(dev)
            ms = []
            for _ in range(args.reps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(); call(); b.record(); b.synchronize()
                ms.append(a.elapsed_time(b))
            t = float(np.median(ms))
            times[(name, views)] = t
            print(json.dumps({'scene': name, 'faces': len(f), 'views': views, 'size': [1280, 960], 'ms_median': round(t, 3),
                              'ms_min': round(min(ms), 3), 'ms_max': round(max(ms), 3),
                              'triangles_per_s': float('%.4g' % (len(f) * views / t * 1e3)),
                              'peak_mem_gb': round((torch.cuda.max_memory_allocated(dev) - base) / 1e9, 3), 'gpu': gpu}), flush=True)
    for b in ('b_head_plus_fullview_quad', 'b10_head_plus_quad_per_view'):
        for views in (1, 10):
            print(json.dumps({'ratio_over_a': round(times[(b, views)] / times[('a_head_%d' % args.res, views)], 3), 'scene': b,
                              'views': views, 'gpu': gpu}), flush=True)
    rng = np.random.RandomState(0)
    flame = SimpleMesh(hv[rng.choice(len(hv), 5023, replace=False)] * 4, np.zeros((0, 3), np.int64))
    nrm = rng.randn(5023, 3)
    flame.vertex_normals = nrm / np.linalg.norm(nrm, axis=1, keepdims=True)
    mesh = SimpleMesh(hv * 4, hf)
    face_idx = np.arange(0, 5023, 2)
    for _ in range(args.warmup):
        sampling.sample_surface_points(mesh, flame, face_idx, 250000)
    ms = []
    for _ in range(max(3, args.reps // 4)):
        torch.cuda.synchronize(); t0 = time.perf_counter()
        out = sampling.sample_surface_points(mesh, flame, face_idx, 250000)
        ms.append(1e3 * (time.perf_counter() - t0))
    print(json.dumps({'sample_surface_points_ms_median': round(float(np.median(ms)), 2), 'ms_min': round(min(ms), 2),
                      'faces': len(hf), 'num_samps': 250000, 'points_face': len(out[2]), 'gpu': gpu}), flush=True)


if __name__ == '__main__':
    main()
