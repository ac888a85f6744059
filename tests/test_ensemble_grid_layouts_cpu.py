"""The layout matrix of tests/test_gpu_ensemble_grid_layouts.py on the CPU: tools/zero_member_tiles.py (the restatement of
tc_ensemble_launch's tile choice that the replay tests and the GPU test's tile-count check use) gives every case the layout
the table names, its tiles cover each grid index of the range exactly once, the 3 % rule puts the boundary cases on the
side the table claims, and the table reaches every kind of range it is meant to (ragged blocks, partial planes, cubes that
start off a multiple of 8 planes, sharded x-slabs, the pruned kernel on a grid ragged in x, y and z)."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(HERE), 'tools'))

from test_gpu_ensemble_grid_layouts import CASES, mirror_tiles  # noqa: E402
from zero_member_tiles import tile_layout, tile_points  # noqa: E402


def _ratio(res, first, count, block):
    """Tiles of blocks `block` over the x-planes of the range, over its linear 128-point tiles."""
    rr = res * res
    px0, px1 = first // rr, (first + count - 1) // rr
    tbx, tby, tbz = block
    blocked = ((px1 - px0 + tbx) // tbx) * -(-res // tby) * -(-res // tbz)
    return blocked, -(-count // 128)


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_case_reaches_its_layout(case):
    label, layout, res, first, count, impl = case
    assert 0 <= first and first + count <= res ** 3, label
    name, kind, block = mirror_tiles(res, first, count, impl)
    assert name == layout, (label, name)


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_tiles_cover_the_range_once(case):
    """Over the valid rows of tile_points, every grid index of [first, first + count) once and nothing else; invalid rows
    carry in-grid coordinates (the kernel loads the axes there).  A range that ends inside an x-plane leaves the blocks past
    its end without a valid row."""
    label, layout, res, first, count, impl = case
    name, kind, block = mirror_tiles(res, first, count, impl)
    ix, iy, iz, valid = tile_points(res, first, count, kind, block)
    assert ix.shape[1] == 128
    for c in (ix, iy, iz):
        assert c.min() >= 0 and c.max() < res, label
    g = ((ix * res + iy) * res + iz)[valid]
    assert g.size == count, (label, g.size, count)
    assert np.array_equal(np.sort(g), np.arange(first, first + count, dtype=np.int64)), label


def test_three_percent_boundary():
    """The dense rule keeps blocks while they add at most 3 % tiles (blocked * 100 <= linear * 103)."""
    # 264^3, 3 x-planes in 1 x 16 x 8 blocks: 3 * 17 * 33 = 1683 tiles against 1634 linear ones, 102.999 %
    first, count = 130 * 264 ** 2, 3 * 264 ** 2
    blocked, linear = _ratio(264, first, count, (1, 16, 8))
    assert (blocked, linear) == (1683, 1634) and blocked * 100 <= linear * 103 < blocked * 100 + 103
    assert tile_layout(264, first, count, 'auto') == ('blocked', (1, 16, 8))
    # 134^3 in 8 x 4 x 4 blocks: 8 planes 102.94 % (in), 128 planes 103.007 % (out: linear tiles)
    blocked, linear = _ratio(134, 0, 8 * 134 ** 2, (8, 4, 4))
    assert (blocked, linear) == (1156, 1123) and blocked * 100 <= linear * 103
    assert tile_layout(134, 0, 8 * 134 ** 2, 'auto') == ('blocked', (8, 4, 4))
    blocked, linear = _ratio(134, 0, 128 * 134 ** 2, (8, 4, 4))
    assert (blocked, linear) == (18496, 17956) and blocked * 100 > linear * 103
    assert tile_layout(134, 0, 128 * 134 ** 2, 'auto') == ('linear', None)
    # the pruned kernel's cubes ignore the rule: 37^3 in cubes is 1.36 x the linear tiles
    blocked, linear = _ratio(37, 0, 37 ** 3, (8, 4, 4))
    assert blocked * 100 > linear * 103 and tile_layout(37, 0, 37 ** 3, '8x4x4') == ('blocked', (8, 4, 4))


def _kinds(case):
    label, layout, res, first, count, impl = case
    name, kind, block = mirror_tiles(res, first, count, impl)
    rr = res * res
    px0, px1 = first // rr, (first + count - 1) // rr
    k = {layout}
    if block is not None:
        tbx, tby, tbz = block
        if res % tby or res % tbz:
            k.add(layout + ' ragged')
        if (px1 - px0 + 1) % tbx:
            k.add(layout + ' ragged x')
    if first % rr or (first + count) % rr:
        k.add(layout + ' partial planes')
    if layout == 'cube' and px0 % 8:
        k.add('cube off 8')
    if label.startswith('shard'):
        k.add('sharded')
    if impl == 'tc_pruned':
        k |= {'pruned ' + x for x in k}
    return k


def test_matrix_reaches_every_kind_of_range():
    kinds = set().union(*(_kinds(c) for c in CASES))
    for want in ('cube', 'cube ragged', 'cube off 8', 'plane', 'plane ragged', 'plane partial planes', 'linear',
                 'linear partial planes', 'sharded', 'pruned cube ragged', 'pruned cube ragged x'):
        assert want in kinds, (want, sorted(kinds))
    # every range distributed.slab_planes issues at 128^3 (2, 3, 8 ranks) and 256^3 (8 ranks)
    from nphm_b200.distributed import plan_slabs, slab_planes
    got = {(c[2], c[3], c[4]) for c in CASES if c[0].startswith('shard')}
    for res, world in ((128, 2), (128, 3), (128, 8), (256, 8)):
        for c0, c1 in plan_slabs(res, world):
            p0, n, _ = slab_planes(c0, c1)
            assert (res, p0 * res * res, n * res * res) in got, (res, world, c0, c1)
    # the sharded ranges carry ghost planes and take plane blocks
    assert all(c[1] == 'plane' for c in CASES if c[0].startswith('shard'))
