"""Shared by test_posed_cpu.py and test_gpu_posed.py: the decoders, codes and points of tests/golden/posed.npz (made by
tests/golden/make_golden_posed.py), and the comparison against it."""
import numpy as np
import torch

from conftest import load_golden, make_deformation, make_ensemble
import npm_fit_common as C

# the tolerance test_device_broyden_search_matches_reference_and_oracle takes for the roots: the search stops at |residual|
# < 1e-6, so two runs agree to a few 1e-6 times |J^-1|; the SDF at the roots inherits it times |grad sdf|
SDF_TOL = 5e-5
VALID_AGREE = 0.97


def ensemble_case(device='cpu', training=True):
    """(decoder_shape, decoder_expr, lat_rep_shape (1, 1, D), z_ex (2, 200), grid (1, N, 3), golden)."""
    g = load_golden('posed.npz')
    dec = make_ensemble(0, device=device).train(training)
    dfn = make_deformation(device)
    with torch.no_grad():
        dfn.defDeepSDF.lin6.weight.mul_(float(g['out_scale']))
        dfn.defDeepSDF.lin6.bias.mul_(float(g['out_scale']))
    lat = torch.from_numpy(g['latent_id']).reshape(1, 1, -1).to(device)
    z_ex = torch.from_numpy(g['z_ex']).to(device)
    grid = torch.from_numpy(g['grid']).reshape(1, -1, 3).to(device)
    return dec, dfn, lat, z_ex, grid, g


def npm_case(device='cpu'):
    """The NPM pair: (decoder_shape, decoder_expr, lat_rep_shape, z_ex (2, 200), points (1, 300, 3), golden)."""
    from nphm_b200.models.deepSDF import DeepSDF
    g = load_golden('posed.npz')
    dec, expr = C.make_decoders(DeepSDF, device)
    lat = torch.from_numpy(g['npm_latent_id']).reshape(1, 1, -1).to(device)
    return dec, expr, lat, torch.from_numpy(g['npm_z_ex']).to(device), torch.from_numpy(g['npm_points']).to(device), g


def check_against_golden(sdf, valid, sdf_ref, valid_ref, tol=SDF_TOL):
    """valid agrees on >= 97 % of the rows and sdf to ``tol`` on the rows both mark valid."""
    assert sdf.shape == sdf_ref.shape and valid.shape == valid_ref.shape and valid.dtype == bool
    assert (valid == valid_ref).mean() >= VALID_AGREE
    both = valid & valid_ref
    assert both.sum() > 0.9 * both.size
    err = float(np.abs(sdf[both] - sdf_ref[both]).max())
    assert err < tol, err
    return err
