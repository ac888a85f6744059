#!/usr/bin/env python
"""Golden fixture for the posed SDF (get_logits_posed), from the UNMODIFIED reference: the composition of its joint fitter
(src/NPHM/models/fitting.py:59-114) on whole point sets,

    _, anchors = decoder_shape(zeros(1, 1, 3), lat_rep_shape, None)                       (ensemble only)
    glob_cond  = cat([lat_rep_shape, z_ex[s]], -1)
    xc, res    = search(chunk, glob_cond.repeat(1, n, 1), decoder_expr, anchors | None, multi_corresp=False)
    sdf, _     = decoder_shape(xc, lat_rep_shape [.repeat(1, n, 1) for a DeepSDF], None)

    python tests/golden/make_golden_posed.py          # needs /root/reference

ensemble: the seeded ensemble and 'compress' DeformationNetwork of make_golden_search.py (output layer x 80, so that some rows
need many Broyden steps and some fail) on the 16^3 grid of create_grid_points_from_bounds(MINI, MAXI, 16), two expressions,
nbatch_points = 1500 (a ragged last chunk of 1096 rows), the identity decoder in train and in eval mode (the search does not
depend on it).  npm: the NPM pair of tests/npm_fit_common.py on 300 points, two expressions.  Writes posed.npz."""
import os
import sys

import numpy as np
import torch

import make_golden as G            # stubs the unused third-party imports and puts the reference on sys.path
from NPHM.models.deepSDF import DeepSDF, DeformationNetwork
from NPHM.models.iterative_root_finding import search

sys.path.insert(0, os.path.dirname(G.HERE))
import npm_fit_common as C         # noqa: E402

OUT_SCALE = 80.0
RES = 16
NBATCH = 1500


def posed(decoder_shape, decoder_expr, lat_rep_shape, z_ex, points, nbatch, modes=(True,)):
    """sdf[mode][s] and valid[s] of the composition above, chunk by chunk."""
    ensemble = hasattr(decoder_shape, 'lat_dim_loc')
    anchors = None
    if ensemble:
        with torch.no_grad():
            _, anchors = decoder_shape(torch.zeros([1, 1, 3]), lat_rep_shape, None)
    sdf = {m: np.empty((z_ex.shape[0], points.shape[1]), np.float32) for m in modes}
    valid = np.empty((z_ex.shape[0], points.shape[1]), bool)
    for s in range(z_ex.shape[0]):
        glob_cond = torch.cat([lat_rep_shape, z_ex[s].reshape(1, 1, -1)], dim=-1)
        for a in range(0, points.shape[1], nbatch):
            chunk = points[:, a:a + nbatch]
            n = chunk.shape[1]
            xc, res = search(chunk, glob_cond.repeat(1, n, 1), decoder_expr,
                             None if anchors is None else anchors.clone().unsqueeze(1).repeat(1, n, 1, 1), multi_corresp=False)
            xc = xc.detach()
            valid[s, a:a + n] = res['valid_ids'].reshape(-1).numpy()
            for m in modes:
                decoder_shape.train(m)
                with torch.no_grad():
                    out, _ = decoder_shape(xc, lat_rep_shape if ensemble else lat_rep_shape.repeat(1, n, 1), None)
                sdf[m][s, a:a + n] = out.reshape(-1).numpy()
    return sdf, valid


def main():
    torch.set_num_threads(os.cpu_count())
    anchors64 = np.load(os.path.join(G.REF, 'assets', 'anchors_39.npy'))
    anchors = torch.from_numpy(anchors64).float().unsqueeze(0).unsqueeze(0)
    lat_mean = np.load(os.path.join(G.REF, 'assets', 'nphm_lat_mean.npy'))
    lat_std = np.load(os.path.join(G.REF, 'assets', 'nphm_lat_std.npy'))
    dec = G.make_ensemble(0, anchors)
    lat = G.sample_latent(1, torch.from_numpy(lat_mean), torch.from_numpy(lat_std)).reshape(1, 1, -1)
    torch.manual_seed(10)
    dfn = DeformationNetwork(mode='compress', lat_dim_expr=200, lat_dim_id=32, lat_dim_glob_shape=64,
                             lat_dim_loc_shape=32, n_loc=39, anchors=anchors, hidden_dim=512, nlayers=6,
                             out_dim=3, input_dim=3)
    dfn.eval()
    with torch.no_grad():
        dfn.defDeepSDF.lin6.weight.mul_(OUT_SCALE)
        dfn.defDeepSDF.lin6.bias.mul_(OUT_SCALE)
    torch.manual_seed(41)
    z_ex = torch.randn(2, 200) * 0.1
    grid = G.create_grid_points_from_bounds(G.MINI, G.MAXI, RES).astype(np.float32)
    sdf, valid = posed(dec, dfn, lat, z_ex, torch.from_numpy(grid)[None], NBATCH, modes=(True, False))
    print('ensemble: valid %d / %d' % (valid.sum(), valid.size))

    npm_dec, npm_expr = C.make_decoders(DeepSDF)
    torch.manual_seed(42)
    npm_zid = torch.randn(1, 1, 512) * 0.05
    npm_zex = torch.randn(2, 200) * 0.05
    npm_pts = (np.random.RandomState(43).randn(1, 300, 3) * 0.1 + np.array([0.0, 0.05, -0.1])).astype(np.float32)
    npm_sdf, npm_valid = posed(npm_dec, npm_expr, npm_zid, npm_zex, torch.from_numpy(npm_pts), 1000)
    print('npm: valid %d / %d' % (npm_valid.sum(), npm_valid.size))
    np.savez_compressed(os.path.join(G.HERE, 'posed.npz'), out_scale=np.float32(OUT_SCALE), res=np.int64(RES),
                        nbatch_points=np.int64(NBATCH), latent_id=lat.numpy().reshape(-1), z_ex=z_ex.numpy(), grid=grid,
                        sdf_train=sdf[True], sdf_eval=sdf[False], valid=valid,
                        npm_latent_id=npm_zid.numpy().reshape(-1), npm_z_ex=npm_zex.numpy(), npm_points=npm_pts,
                        npm_sdf=npm_sdf[True], npm_valid=npm_valid)


if __name__ == '__main__':
    main()
