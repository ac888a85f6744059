"""The dense ensemble kernel hands tiles out on demand (a device counter that the last CTA resets) and takes each tile's
member mask from a pre-pass.  Every point must be written exactly once, whatever the number of tiles against the number of
SMs, and back-to-back launches on one stream must each start from a reset counter.  The pre-pass masks of the benchmark's
head must keep exactly the members tools/zero_member_tiles.py predicts."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools'))

CHUNK = 25000


@pytest.fixture(scope='module')
def eng_lat(cuda_device):
    from conftest import make_ensemble, sample_latent
    from nphm_b200 import _native
    dec = make_ensemble(0, device=cuda_device).eval()
    eng = _native.EnsembleEngine(dec)
    eng.refresh(dec)
    lat = torch.stack([sample_latent(s).reshape(-1) for s in (1, 2, 3)]).to(cuda_device)
    return eng, lat


def n_sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def grid_nan(eng, lat, res, first, count, impl='tc', mini=None, maxi=None):
    from conftest import MAXI, MINI
    out = torch.full((count,), float('nan'), device=lat.device)
    eng.query_grid(lat, MINI if mini is None else mini, MAXI if maxi is None else maxi, res, first, count, 0,
                   impl=impl, out=out)
    return out


def xyz_nan(eng, xyz, lat, impl='tc'):
    """nphm_ensemble_query into an output filled with NaN (EnsembleEngine.query allocates its own)."""
    from nphm_b200 import _native
    B, N, _ = xyz.shape
    xyz = xyz.contiguous().float()
    lat = lat.contiguous().float()
    sdf = torch.full((B, N, 1), float('nan'), device=xyz.device)
    anchors = torch.empty(B, eng.n_loc, 3, device=xyz.device)
    _native.check(_native.lib().nphm_ensemble_query(eng.handle, xyz.data_ptr(), lat.data_ptr(), B, N, 0, sdf.data_ptr(),
                                                    anchors.data_ptr(), _native.impl_code(impl),
                                                    torch.cuda.current_stream(xyz.device).cuda_stream),
                  'nphm_ensemble_query')
    return sdf


def grid_xyz(res, first, count, dev, mini=None, maxi=None):
    from conftest import MAXI, MINI
    lo, hi = MINI if mini is None else mini, MAXI if maxi is None else maxi
    axes = [torch.from_numpy(np.linspace(lo[a], hi[a], res).astype(np.float32)) for a in range(3)]
    xyz = torch.stack(torch.meshgrid(*axes, indexing='ij'), dim=-1).reshape(-1, 3)[first:first + count]
    return xyz.reshape(1, -1, 3).to(dev)


def shuffled_query(eng, xyz, lat, impl='tc'):
    """The same points in a random order (other tiles, other masks), put back in place."""
    perm = torch.randperm(xyz.shape[1], generator=torch.Generator().manual_seed(3)).to(xyz.device)
    s = xyz_nan(eng, xyz[:, perm], lat, impl)
    back = torch.empty_like(s)
    back[:, perm] = s
    return back


def assert_all_written(t):
    assert not torch.isnan(t).any(), '%d points not written' % int(torch.isnan(t).sum())


@pytest.mark.gpu
@pytest.mark.parametrize('case', ['fewer_tiles_than_sms', 'sms_k_plus_1', 'slab_ghost_planes', 'full_grid'])
def test_grid_every_point_once(eng_lat, case):
    eng, lat = eng_lat
    dev = lat.device
    res, first, count = {
        # a partial x-plane: linear tiles, far fewer than the SMs
        'fewer_tiles_than_sms': (64, 12345, 20 * 128 - 7),
        # 132 k + 1 linear tiles (k = 3 on an H100)
        'sms_k_plus_1': (128, 5000, (3 * n_sms(dev)) * 128 + 1),
        # an x-slab of 32 planes with a ghost plane on each side (compact tiles)
        'slab_ghost_planes': (128, 47 * 128 ** 2, 34 * 128 ** 2),
        'full_grid': (64, 0, 64 ** 3),
    }[case]
    got = grid_nan(eng, lat[0], res, first, count)
    assert_all_written(got)
    ref = shuffled_query(eng, grid_xyz(res, first, count, dev), lat[:1]).reshape(-1)
    assert torch.equal(got, ref)


@pytest.mark.gpu
def test_xyz_two_queries(eng_lat):
    eng, lat = eng_lat
    dev = lat.device
    g = torch.Generator().manual_seed(11)
    n = (n_sms(dev) + 1) * 128 + 5
    xyz = (torch.randn(2, n, 3, generator=g) * 0.4).to(dev)
    got = xyz_nan(eng, xyz, lat[:2])
    assert_all_written(got)
    for b in range(2):                       # each query alone
        assert torch.equal(got[b], xyz_nan(eng, xyz[b:b + 1], lat[b:b + 1])[0])


@pytest.mark.gpu
def test_pruned_every_point_once(eng_lat):
    eng, lat = eng_lat
    dev = lat.device
    res, first, count = 64, 0, 64 ** 3
    pruned = grid_nan(eng, lat[1], res, first, count, impl='tc_pruned')
    assert_all_written(pruned)
    assert torch.equal(pruned, grid_nan(eng, lat[1], res, first, count, impl='tc_pruned'))
    dense = grid_nan(eng, lat[1], res, first, count)
    assert float((pruned - dense).abs().max()) < 1e-4
    xyz = grid_xyz(res, 1000, 3 * 128 + 1, dev)
    p_xyz = xyz_nan(eng, xyz, lat[1:2], impl='tc_pruned')
    assert_all_written(p_xyz)


@pytest.mark.gpu
def test_back_to_back_launches_reset_the_counter(eng_lat):
    eng, lat = eng_lat
    dev = lat.device
    g = torch.Generator().manual_seed(4)
    xyz_a = (torch.randn(1, 700, 3, generator=g) * 0.4).to(dev)
    xyz_b = (torch.randn(2, 50 * 128 + 3, 3, generator=g) * 0.4).to(dev)
    calls = [
        lambda: grid_nan(eng, lat[0], 64, 0, 64 ** 3),
        lambda: xyz_nan(eng, xyz_a, lat[:1]),
        lambda: grid_nan(eng, lat[2], 128, 47 * 128 ** 2, 34 * 128 ** 2),
        lambda: xyz_nan(eng, xyz_b, lat[1:3]),
        lambda: grid_nan(eng, lat[1], 64, 777, 5 * 128, impl='tc_pruned'),
        lambda: grid_nan(eng, lat[0], 64, 0, 64 ** 3),
    ]
    torch.cuda.synchronize(dev)
    together = [c() for c in calls]          # one stream, no synchronisation in between
    torch.cuda.synchronize(dev)
    for c, t in zip(calls, together):
        alone = c()
        torch.cuda.synchronize(dev)
        assert_all_written(t)
        assert torch.equal(t, alone)


def pre_pass_masks(eng):
    from nphm_b200 import _native
    L = _native.lib()
    n = ctypes.c_longlong(0)
    _native.check(L.nphm_debug_ens_tile_masks(eng.handle, None, ctypes.c_longlong(0), ctypes.byref(n)), 'masks')
    buf = np.zeros(n.value, dtype=np.uint64)
    _native.check(L.nphm_debug_ens_tile_masks(eng.handle, buf.ctypes.data_as(ctypes.c_void_p), ctypes.c_longlong(n.value),
                                              ctypes.byref(n)), 'masks')
    return buf


@pytest.mark.gpu
@pytest.mark.parametrize('res', [64, 128])
def test_pre_pass_masks_match_the_cpu_count(cuda_device, res):
    from conftest import MAXI, MINI, make_ensemble, sample_latent
    from nphm_b200 import _native
    import zero_member_tiles as Z
    dec = make_ensemble(0, device=cuda_device).eval()
    eng = _native.EnsembleEngine(dec)
    eng.refresh(dec)
    eng.query_grid(sample_latent(1).to(cuda_device), MINI, MAXI, res, 0, res ** 3, CHUNK, impl='tc')
    masks = pre_pass_masks(eng)
    r = Z.zero_member_tiles(Z.anchors_of(1), MINI, MAXI, res)
    assert masks.size == r['tiles']
    assert np.all(masks >> np.uint64(39) == 1), 'the global member is in every tile, members >= 40 in none'
    evaluated = int(sum(bin(int(m)).count('1') for m in masks))
    assert evaluated == r['evaluated_member_tiles']
