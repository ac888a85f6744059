"""The narrow-band extraction restated in numpy (oracle/band_oracle.py) gives the dense mesh of the C marching-cubes oracle on
analytic SDFs, grows along a surface that leaves the initial band, and misses a sub-block blob only at a small margin."""
import numpy as np
import pytest

from narrowband_common import analytic_volume
from oracle import band_oracle as BO
from oracle import nphm_oracle as O

LO, HI = [-1.0] * 3, [1.0] * 3


def _mesh(vol, res):
    return O.mesh_from_logits(vol.copy(), LO, HI, res)


def _same(a, b):
    return a[0].shape == b[0].shape and np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


@pytest.mark.parametrize('name,res', [('sphere', 33), ('sphere', 65), ('torus', 49), ('two_spheres', 65), ('thin_plate', 65)])
def test_band_mesh_equals_dense(name, res):
    dense, h = analytic_volume(name, res)
    r = BO.band_volume(dense, block=4, tau=4 * np.sqrt(3) * h)
    ref = _mesh(dense, res)
    assert len(ref[0]) > 0
    assert _same(_mesh(r['volume'], res), ref)
    assert np.array_equal(r['volume'][r['evaluated']], dense[r['evaluated']])
    assert r['voxels_evaluated'] < res ** 3
    if name == 'thin_plate':
        assert r['growth_rounds'] >= 2                 # the plate leaves the initial band; the band follows it


def test_quirk_voxels_are_evaluated_with_their_blocks():
    dense, h = analytic_volume('torus', 33)
    # spurious positive values, like get_logits' last point of every chunk in eval mode: bubbles the band must reproduce
    period = 97
    g = np.union1d(np.arange(period - 1, 33 ** 3, period), [33 ** 3 - 1])
    dense.reshape(-1)[g] = 1.0
    r = BO.band_volume(dense, block=4, tau=4 * np.sqrt(3) * h, quirk_period=period)
    assert r['evaluated'].reshape(-1)[g].all()
    assert _same(_mesh(r['volume'], 33), _mesh(dense, 33))


def test_infinite_margin_is_dense():
    dense, _ = analytic_volume('sphere', 33)
    r = BO.band_volume(dense, block=4, tau=np.inf)
    assert r['active'].all() and r['evaluated'].all()
    assert np.array_equal(r['volume'], dense)


def test_sub_block_blob_needs_the_margin():
    """The documented limit: a blob between block corners that are all farther than tau from 0 is not seen."""
    res, B = 65, 4
    h = 2.0 / (res - 1)
    c = -1.0 + 34 * h                                  # the centre voxel of block (8, 8, 8)
    ax = np.linspace(-1.0, 1.0, res)
    X, Y, Z = np.meshgrid(ax, ax, ax, indexing='ij')
    dense = (np.sqrt((X - c) ** 2 + (Y - c) ** 2 + (Z - c) ** 2) - 1.3 * h).astype(np.float32)
    ref = _mesh(dense, res)
    assert len(ref[0]) > 0
    small = BO.band_volume(dense, block=B, tau=1.0 * h)
    assert small['active'].sum() == 0 and len(_mesh(small['volume'], res)[0]) == 0
    large = BO.band_volume(dense, block=B, tau=4.0 * h)        # > the corner distance B h sqrt(3) / 2 minus the radius
    assert _same(_mesh(large['volume'], res), ref)
