"""Dense grid queries skip the members whose blend terms fp32 rounding absorbs (den + w == den and w |s| < ulp(|num|) / 4 at
every valid point of a tile, DESIGN 4.1); the outputs must not change a bit.  Each case runs with the skip on and off
(NPHM_ENS_ABSORB=0) in one build: the bench bounds at 64^3 and 128^3 for three latents, a wide grid, an x-slab with ghost
planes, a chunk with the reference's quirk rows, a head with doubled weights (larger member outputs) and a head scaled so that
num passes near zero on the surface."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))

CHUNK = 256 ** 3 // 8


def run(eng, lat, mini, maxi, res, first, count, quirk, absorb):
    old = os.environ.get('NPHM_ENS_ABSORB')
    os.environ['NPHM_ENS_ABSORB'] = '1' if absorb else '0'
    try:
        out = eng.query_grid(lat, mini, maxi, res, first, count, quirk, impl='tc')[0].clone()
        torch.cuda.synchronize()
        return out
    finally:
        if old is None:
            del os.environ['NPHM_ENS_ABSORB']
        else:
            os.environ['NPHM_ENS_ABSORB'] = old


def head(dev, scale=1.0):
    from conftest import make_ensemble, sample_latent
    from nphm_b200 import _native
    dec = make_ensemble(0, scale=scale, device=dev).eval()
    eng = _native.EnsembleEngine(dec)
    eng.refresh(dec)
    lat = torch.stack([sample_latent(s).reshape(-1) for s in (1, 2, 3)]).to(dev)
    return eng, lat


def both_equal(eng, lat, *args):
    on = run(eng, lat, *args, absorb=True)
    off = run(eng, lat, *args, absorb=False)
    assert torch.equal(on.view(torch.int32), off.view(torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize('res', [64, 128])
@pytest.mark.parametrize('latent', [0, 1, 2])
def test_bench_bounds(cuda_device, res, latent):
    from conftest import MAXI, MINI
    eng, lat = head(cuda_device)
    both_equal(eng, lat[latent], MINI, MAXI, res, 0, res ** 3, CHUNK)


@pytest.mark.gpu
def test_wide_grid_slab_and_quirk(cuda_device):
    import make_golden_ensemble_zero_skip as M
    from conftest import MAXI, MINI
    eng, lat = head(cuda_device)
    both_equal(eng, lat[0], M.WIDE_MIN, M.WIDE_MAX, 64, 0, 64 ** 3, 0)
    both_equal(eng, lat[2], MINI, MAXI, 128, 47 * 128 ** 2, 34 * 128 ** 2, CHUNK)        # x-slab with ghost planes
    both_equal(eng, lat[1], MINI, MAXI, 96, 0, 96 ** 3, 4097)                          # quirk rows in many tiles


@pytest.mark.gpu
@pytest.mark.parametrize('scale', [2.0, 0.25])
def test_scaled_heads(cuda_device, scale):
    from conftest import MAXI, MINI
    eng, lat = head(cuda_device, scale)
    both_equal(eng, lat[0], MINI, MAXI, 128, 0, 128 ** 3, CHUNK)
