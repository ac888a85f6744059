"""The absorption certificate per point (DESIGN 4.1): the producer warp skips member k on a tile when, at every valid point
with w_k != 0, w_k * B_k < ulp(L) / 4 with L the point's own |num| two evaluated positions back minus the lag term of the
member in between.  Outputs with the skip on and off (NPHM_ENS_ABSORB=0) must be bit-identical in one build.  The cases are
those where the per-point rule certifies members the tile-wide rule did not (tools/absorbed_member_tiles.py): a head scaled
by 0.25, whose num crosses zero inside many tiles; an x-slab with ghost planes; a chunk with quirk rows in many tiles; a
wide grid whose far tiles keep only the global member; and several latents and chunkings of the scaled head."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))

from test_gpu_ensemble_absorb import CHUNK, both_equal, head  # noqa: E402


@pytest.mark.gpu
@pytest.mark.parametrize('latent', [0, 1, 2])
def test_quarter_head_crosses_zero(cuda_device, latent):
    from conftest import MAXI, MINI
    eng, lat = head(cuda_device, 0.25)
    both_equal(eng, lat[latent], MINI, MAXI, 128, 0, 128 ** 3, CHUNK)


@pytest.mark.gpu
def test_quarter_head_slab_and_quirk(cuda_device):
    from conftest import MAXI, MINI
    eng, lat = head(cuda_device, 0.25)
    both_equal(eng, lat[1], MINI, MAXI, 128, 47 * 128 ** 2, 34 * 128 ** 2, CHUNK)        # x-slab with ghost planes
    both_equal(eng, lat[0], MINI, MAXI, 96, 0, 96 ** 3, 4097)                          # quirk rows in many tiles
    both_equal(eng, lat[2], MINI, MAXI, 80, 1000, 80 ** 3 - 2000, 0)                     # a chunk inside planes


@pytest.mark.gpu
def test_slab_quirk_and_global_only_tiles(cuda_device):
    import make_golden_ensemble_zero_skip as M
    from conftest import MAXI, MINI
    eng, lat = head(cuda_device)
    both_equal(eng, lat[1], M.WIDE_MIN, M.WIDE_MAX, 96, 0, 96 ** 3, 0)                  # far tiles: only the global member
    both_equal(eng, lat[0], MINI, MAXI, 160, 61 * 160 ** 2, 38 * 160 ** 2, 8191)          # x-slab with ghost planes and quirk rows
    both_equal(eng, lat[2], MINI, MAXI, 256, 120 * 256 ** 2, 3 * 256 ** 2, CHUNK)         # planes of the benchmark grid
