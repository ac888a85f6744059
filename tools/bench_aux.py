#!/usr/bin/env python
"""Secondary paths of the hot path on one GPU: deformation-field query (config 3 ingredient), identity fitting
iterations/s (config 4 ingredient).  Prints one JSON line.   python tools/bench_aux.py [--res 128]"""
import argparse, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np
import torch
from conftest import MAXI, MINI, load_golden, make_deformation, make_ensemble, sample_latent
from nphm_b200.models.fitting import IdentityFitter
from nphm_b200.utils.reconstruction import create_grid_points_from_bounds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--res', type=int, default=128)
    ap.add_argument('--fit-iters', type=int, default=200)
    ap.add_argument('--joint-res', type=int, default=256)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    out = {}
    # ---- deformation query on a grid
    dfn = make_deformation(dev)
    dec = make_ensemble(0, device=dev).eval()
    lat = sample_latent(1).to(dev)
    torch.manual_seed(11)
    z_ex = (torch.randn(200) * 0.1).to(dev)
    pts = torch.from_numpy(create_grid_points_from_bounds(MINI, MAXI, args.res)).to(dev, dtype=torch.float).reshape(1, -1, 3)
    with torch.no_grad():
        _, anchors = dec(torch.zeros(1, 1, 3, device=dev), lat.reshape(1, 1, -1), None)
        cond = torch.cat([lat, z_ex]).reshape(1, 1, -1)
        for _ in range(2):
            off, _ = dfn(pts, cond, anchors)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(3):
            off, _ = dfn(pts, cond, anchors)
        e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 3
    n = pts.shape[1]
    out['deformation_query'] = {'res': args.res, 'ms': ms, 'points_per_s': n / (ms * 1e-3),
                                'tflops_dense': 2.624e6 * n / (ms * 1e-3) / 1e12}
    # ---- joint query (BASELINE.json configs[2]): identity SDF + forward deformation on the same grid
    R = args.joint_res
    gp = torch.from_numpy(create_grid_points_from_bounds(MINI, MAXI, R)).to(dev, dtype=torch.float).reshape(1, -1, 3)
    vol = torch.empty(R ** 3, device=dev)
    with torch.no_grad():
        for _ in range(2):
            dec.engine().query_grid(lat, MINI, MAXI, R, 0, R ** 3, 25000, out=vol)
            off, _ = dfn(gp, cond, anchors)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(3):
            dec.engine().query_grid(lat, MINI, MAXI, R, 0, R ** 3, 25000, out=vol)
            off, _ = dfn(gp, cond, anchors)
        e1.record(); torch.cuda.synchronize()
    jms = e0.elapsed_time(e1) / 3
    out['joint_query'] = {'res': R, 'ms': jms, 'points_per_s': R ** 3 / (jms * 1e-3),
                          'tflops_dense': 12.24e6 * R ** 3 / (jms * 1e-3) / 1e12}
    del gp, off
    # ---- identity fitting: 5 x 1000 points per iteration
    rng = np.random.RandomState(0)
    obs = torch.from_numpy((rng.randn(5000, 3) * 0.12).astype(np.float32)).to(dev)
    dec.train()
    fitter = IdentityFitter(dec, dev)
    lam = {'surface': 2.0, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
    for _ in range(5):
        fitter.step(obs, lam, 0.1, 0.01)
    torch.cuda.synchronize(); t0 = time.perf_counter()
    for _ in range(args.fit_iters):
        fitter.step(obs, lam, 0.1, 0.01)
    torch.cuda.synchronize(); dt = time.perf_counter() - t0
    out['identity_fit'] = {'points_per_iter': 5000, 'iters_per_s': args.fit_iters / dt, 'ms_per_iter': 1e3 * dt / args.fit_iters}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
