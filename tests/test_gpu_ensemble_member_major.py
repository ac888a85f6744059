"""Dense grid queries member by member (DESIGN 4.1): the edges of the member-major path against the tile-major kernel.

With the fp32-absorption skip on, a dense grid query runs per member a pass that blends quirk rows, skips the rows whose
term fp32 rounding absorbs and lists the rest, then the ensemble kernel on 128-row tiles of that list.  Absorb off
(NPHM_ENS_ABSORB=0) runs the tile-major kernel on every non-zero member.  Both must give the same bits:
  * across the 2^24-row chunk boundary of the per-row state (264^3: two chunks);
  * where some member's last listed tile holds a single row;
  * with no write outside the range and every point of it written (sentinel buffer);
  * where some member's list is empty;
  * for two back-to-back queries of different sizes on one stream (the counters start from zero each time);
  * at res 2048 over 16 x-slabs of 32-plane sub-boxes: 65 536 sub-box bounds per member, more than a grid dimension other
    than x may hold (its planes against the same planes queried alone).
And the listed rows, on the benchmark head at 64^3 and 128^3: per member exactly the pairs tools/absorbed_member_tiles.py
predicts on the CPU (tests/golden/ensemble_member_major.npz), at most 128 per tile whose pre-pass mask has the member, and
fewer listed tiles (sum over members of ceil(rows / 128)) than member-tiles the tile-major kernel evaluates.
"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from test_gpu_ensemble_absorb_replay import CHUNK, bits, debug_array, head, lib, query  # noqa: E402
from test_gpu_ensemble_grid_layouts import SENTINEL, check_writes  # noqa: E402

HEAD = 'seed:0:1'                   # the benchmark's head


class absorb_on:
    """NPHM_ENS_ABSORB=1 inside the block, the caller's setting after it."""
    def __enter__(self):
        self.old = os.environ.get('NPHM_ENS_ABSORB')
        os.environ['NPHM_ENS_ABSORB'] = '1'

    def __exit__(self, *exc):
        if self.old is None:
            del os.environ['NPHM_ENS_ABSORB']
        else:
            os.environ['NPHM_ENS_ABSORB'] = self.old


def pair_counts(eng, M):
    """Rows listed per (chunk, member) by the last query: n_chunks x M (0 x M when it ran tile-major)."""
    from nphm_b200 import _native
    L = _native.lib()
    f = L.nphm_debug_ens_pair_counts
    f.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong, ctypes.POINTER(ctypes.c_longlong)]
    n = ctypes.c_longlong(0)
    _native.check(f(eng.handle, None, 0, ctypes.byref(n)), 'pair counts')
    buf = np.zeros(n.value, np.uint32)
    _native.check(f(eng.handle, buf.ctypes.data_as(ctypes.c_void_p), n.value, ctypes.byref(n)), 'pair counts')
    return buf.reshape(-1, M).astype(np.int64)


def on_off(eng, z, res, first, count, quirk=CHUNK):
    from conftest import MAXI, MINI
    on, _ = query(eng, z, MINI, MAXI, res, first, count, quirk, absorb=True)
    counts = pair_counts(eng, eng.n_loc + 1)
    off, _ = query(eng, z, MINI, MAXI, res, first, count, quirk, absorb=False)
    n = int((on.view(torch.int32) != off.view(torch.int32)).sum())
    assert n == 0, '%d of %d outputs differ between member-major and tile-major (%d^3, [%d, +%d))' % (n, count, res, first, count)
    return counts


@pytest.fixture(scope='module')
def eng_z(cuda_device):
    from conftest import sample_latent
    _, eng = head(HEAD, cuda_device)
    return eng, sample_latent(1).reshape(-1).to(cuda_device)


@pytest.mark.gpu
def test_chunk_boundary(eng_z):
    eng, z = eng_z
    counts = on_off(eng, z, 264, 0, 264 ** 3)
    assert counts.shape[0] == 2, 'a 264^3 grid runs in two chunks of per-row state'
    print('  264^3: rows listed per chunk %s' % counts.sum(axis=1).tolist())


@pytest.mark.gpu
def test_single_row_last_tile(eng_z):
    """Ranges until some member's list ends with a one-row tile; every range on against off."""
    eng, z = eng_z
    found = []
    for res in (40, 48, 56, 64, 72, 80, 88, 96):
        for first_planes in (0, 3):
            first = first_planes * res * res
            counts = on_off(eng, z, res, first, res ** 3 - first)
            hit = np.nonzero(counts[0] % 128 == 1)[0]
            if hit.size:
                found.append((res, first, int(hit[0])))
        if found:
            break
    print('  one-row last tiles: %s' % found)
    assert found, 'no range with a one-row last tile'


@pytest.mark.gpu
def test_writes_stay_in_range(eng_z):
    from conftest import MAXI, MINI
    eng, z = eng_z
    bad = []
    for res, first, count in ((64, 0, 64 ** 3), (100, 777, 100 ** 3 - 5000), (128, 40 * 128 ** 2, 16 * 128 ** 2)):
        pad = 2 * res * res + 256
        buf = torch.full((count + 2 * pad,), SENTINEL, dtype=torch.int32, device=z.device).view(torch.float32)
        with absorb_on():
            eng.query_grid(z, MINI, MAXI, res, first, count, CHUNK, impl='tc', out=buf[pad:pad + count])
            torch.cuda.synchronize()
        assert pair_counts(eng, eng.n_loc + 1).shape[0] == 1, 'the query did not run member by member'
        check_writes(buf, pad, count, '%d^3 [%d, +%d)' % (res, first, count), bad)
    assert not bad, bad


@pytest.mark.gpu
def test_empty_member_list(eng_z):
    """Thin x-slabs at the edges of the grid until some member lists no row there (its weight is zero or absorbed at every
    point); every range on against off."""
    eng, z = eng_z
    found = []
    for res, first, count in ((128, 0, 2 * 128 ** 2), (128, 126 * 128 ** 2, 2 * 128 ** 2), (256, 0, 256 ** 2),
                              (256, 255 * 256 ** 2, 256 ** 2), (64, 0, 64 ** 3)):
        counts = on_off(eng, z, res, first, count)
        empty = np.nonzero(counts[0] == 0)[0]
        if empty.size:
            found.append((res, first, count, empty.tolist()))
            break
    print('  members with an empty list: %s' % found)
    assert found, 'no range with an empty member list'


@pytest.mark.gpu
def test_many_sub_boxes(eng_z):
    """x-planes 31 .. 480 of the 2048^3 grid (1.9 G points, 7.5 GB of output) touch x-slabs 0 .. 15 of the 32^3-point
    sub-boxes: 16 x 64 x 64 = 65 536 sub-boxes.  The first, a middle and the last plane must equal the same planes queried
    alone, which equal the tile-major kernel."""
    from conftest import MAXI, MINI
    eng, z = eng_z
    res, rr = 2048, 2048 ** 2
    x0, x1 = 31, 480
    with absorb_on():
        big, _ = eng.query_grid(z, MINI, MAXI, res, x0 * rr, (x1 - x0 + 1) * rr, CHUNK, impl='tc')
        torch.cuda.synchronize()
    assert pair_counts(eng, eng.n_loc + 1).shape[0] > 1, 'the query did not run member by member'
    for x in (x0, 256, x1):
        one = on_off(eng, z, res, x * rr, rr)
        assert one.shape[0] == 1
        plane, _ = query(eng, z, MINI, MAXI, res, x * rr, rr, CHUNK, absorb=True)
        got = big[(x - x0) * rr:(x - x0 + 1) * rr]
        assert torch.equal(got.view(torch.int32), plane.view(torch.int32)), 'plane %d differs from the plane alone' % x
    del big


@pytest.mark.gpu
def test_back_to_back_queries(eng_z):
    """A large query and a small one on one stream without a synchronize in between, then the same in reverse."""
    from conftest import MAXI, MINI
    eng, z = eng_z
    sizes = [(128, 0, 128 ** 3), (48, 5 * 48 * 48, 20 * 48 * 48)]
    ref = [query(eng, z, MINI, MAXI, r, f, c, CHUNK, absorb=False)[0] for r, f, c in sizes]
    for order in (sizes, sizes[::-1]):
        with absorb_on():
            outs = [eng.query_grid(z, MINI, MAXI, r, f, c, CHUNK, impl='tc')[0] for r, f, c in order]
            torch.cuda.synchronize()
        for (r, f, c), out in zip(order, outs):
            want = ref[sizes.index((r, f, c))]
            assert torch.equal(out.view(torch.int32), want.view(torch.int32)), (r, f, c)


@pytest.mark.gpu
@pytest.mark.parametrize('res', [64, 128])
def test_listed_rows(eng_z, res):
    """Listed rows per member: the predictor's, within the tiles whose mask has the member, and in fewer compact tiles
    than the member-tiles the tile-major kernel evaluates (its skip log)."""
    from conftest import MAXI, MINI, load_golden
    eng, z = eng_z
    M = eng.n_loc + 1
    counts = on_off(eng, z, res, 0, res ** 3)[0]
    want = load_golden('ensemble_member_major.npz')['pairs_%d' % res]
    diff = np.nonzero(counts != want)[0]
    print('  %d^3: %d rows listed, the predictor %d; members that differ %s: %s against %s' % (
        res, counts.sum(), want.sum(), diff.tolist(), counts[diff].tolist(), want[diff].tolist()))
    assert diff.size == 0, 'listed rows differ from the predictor'
    masks = bits(debug_array(eng, 'nphm_debug_ens_tile_masks', np.uint64), M)
    assert np.all(counts <= 128 * masks.sum(axis=0)), 'more rows listed than the masked tiles hold'
    assert counts[M - 1] > 0, 'the global member listed no row'
    L = lib()
    L.nphm_debug_ens_skip_log(eng.handle, 1)
    try:
        query(eng, z, MINI, MAXI, res, 0, res ** 3, CHUNK)
        assert pair_counts(eng, M).shape[0] == 0, 'a query with the skip log must run tile-major'
        masks = bits(debug_array(eng, 'nphm_debug_ens_tile_masks', np.uint64), M)
        skipped = bits(debug_array(eng, 'nphm_debug_ens_skipped', np.uint64), M)
    finally:
        L.nphm_debug_ens_skip_log(eng.handle, 0)
    tile_major = int((masks & ~skipped).sum())
    member_major = int(((counts + 127) // 128).sum())
    print('  %d^3: %d member-tiles tile-major, %d member by member (%d rows listed)'
          % (res, tile_major, member_major, int(counts.sum())))
    assert member_major < tile_major
