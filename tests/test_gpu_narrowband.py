"""Narrow-band mesh extraction (csrc/narrowband.cu, utils/reconstruction.extract_mesh_narrowband) against the dense path
``mesh_from_logits(get_logits(...))``: the same vertex ids, float64 positions and triangles, bit for bit."""
import math

import numpy as np
import pytest
import torch

from conftest import MAXI, MINI, make_ensemble, sample_latent
from narrowband_common import make_npm_head, tilted_plate
from oracle import band_oracle as BO

pytestmark = pytest.mark.gpu


def _grid(res, dev):
    from nphm_b200.utils.reconstruction import create_grid_points_from_bounds
    return torch.from_numpy(create_grid_points_from_bounds(MINI, MAXI, res)).to(dev, dtype=torch.float32)[None]


def _dense(dec, lat, res, nbatch, dev):
    """(dense volume (res^3,) float32, dense mesh)."""
    from nphm_b200.models.reconstruction import get_logits
    from nphm_b200.utils.reconstruction import mesh_from_logits
    logits = get_logits(dec, lat, _grid(res, dev), nbatch_points=nbatch)
    vol = logits.copy()
    return vol, mesh_from_logits(logits, MINI, MAXI, res)


def _assert_same_mesh(a, b):
    va, vb = np.asarray(a.vertices), np.asarray(b.vertices)
    fa, fb = np.asarray(a.faces), np.asarray(b.faces)
    assert va.shape == vb.shape and fa.shape == fb.shape
    assert np.array_equal(fa, fb)
    assert np.array_equal(va, vb)                       # float64 positions bit for bit


def _evaluated_mask(states, res, block):
    """voxels of the active blocks (the block corners and quirk voxels lie in them or are corners)."""
    nb = states.shape[0]
    m = np.zeros((res,) * 3, bool)
    for bx, by, bz in zip(*np.nonzero(states)):
        lo = np.array([bx, by, bz]) * block
        hi = np.minimum(lo + block, res - 1)
        m[lo[0]:hi[0] + 1, lo[1]:hi[1] + 1, lo[2]:hi[2] + 1] = True
    ci = np.minimum(np.arange(nb + 1) * block, res - 1)
    m[np.ix_(ci, ci, ci)] = True
    return m


@pytest.fixture(scope='module')
def head(cuda_device):
    return make_ensemble(0, device=cuda_device).eval(), sample_latent(1).to(cuda_device)


@pytest.mark.parametrize('res,train,nbatch', [(64, False, 25000), (64, True, 25000), (128, False, 20000), (128, True, 20000),
                                              (256, False, 25000), (64, False, 97), (128, False, 1000)])
def test_ensemble_mesh_equals_dense(cuda_device, head, res, train, nbatch):
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband
    dec, lat = head
    dec.train(train)
    try:
        _, ref = _dense(dec, lat, res, nbatch, cuda_device)
        mesh, stats = extract_mesh_narrowband(dec, lat, MINI, MAXI, res, nbatch_points=nbatch, return_stats=True)
    finally:
        dec.eval()
    assert len(ref.vertices) > 0
    _assert_same_mesh(mesh, ref)
    # at 64^3 the default margin (4 grid steps) covers this shallow random head; a small period activates the blocks around
    # thousands of quirk voxels
    if res >= 128 and nbatch >= 20000:
        assert stats['voxels_evaluated'] < res ** 3 and 0 < stats['blocks_active'] < stats['blocks_total']
    cached = getattr(mesh, '_nphm_device_vertices', None)
    if cached is not None:
        assert torch.equal(cached, ref._nphm_device_vertices)


@pytest.mark.parametrize('train', [False, True])
def test_evaluated_voxels_equal_dense_volume(cuda_device, head, train):
    """Batch invariance: every voxel the band evaluates, in whatever call and tile, has the dense value bit for bit; the
    rest hold their block's corner 0."""
    from nphm_b200.utils.reconstruction import _band_evaluators, narrowband_volume
    dec, lat = head
    res, nbatch, block = 96, 5000, 4
    dec.train(train)
    try:
        dense, _ = _dense(dec, lat, res, nbatch, cuda_device)
        ev, evq = _band_evaluators(dec, lat, cuda_device)
        vol, stats, band = narrowband_volume(ev, MINI, MAXI, res, cuda_device, block=block, quirk_period=0 if train else nbatch,
                                             evaluate_quirk=evq)
    finally:
        dec.eval()
    dense = dense.reshape((res,) * 3)
    vol = vol.cpu().numpy()
    m = _evaluated_mask(band.block_states().cpu().numpy(), res, block)
    assert int(m.sum()) == stats['voxels_evaluated']
    assert np.array_equal(vol[m], dense[m])
    nb = band.blocks_per_axis
    fi = np.minimum(np.arange(res) // block, nb - 1) * block
    assert np.array_equal(vol[~m], dense[np.ix_(fi, fi, fi)][~m])


def test_block_states_equal_oracle(cuda_device, head):
    from nphm_b200.utils.reconstruction import _band_evaluators, default_margin, narrowband_volume
    dec, lat = head
    res, nbatch, block = 48, 997, 4
    dense, _ = _dense(dec, lat, res, nbatch, cuda_device)
    ev, evq = _band_evaluators(dec, lat, cuda_device)
    vol, stats, band = narrowband_volume(ev, MINI, MAXI, res, cuda_device, block=block, quirk_period=nbatch, evaluate_quirk=evq)
    r = BO.band_volume(dense.reshape((res,) * 3), block=block, tau=default_margin(MINI, MAXI, res, block), quirk_period=nbatch)
    assert np.array_equal(band.block_states().cpu().numpy(), r['active'])
    assert np.array_equal(vol.cpu().numpy(), r['volume'])
    assert stats['voxels_evaluated'] == r['voxels_evaluated'] and stats['growth_rounds'] == r['growth_rounds']


def test_thin_plate_grows(cuda_device):
    """An analytic SDF through the internal form: the band grows along a plate that leaves it, as the oracle does."""
    from nphm_b200 import _native
    from nphm_b200.utils.reconstruction import _device_mesh, narrowband_volume
    res, block = 65, 4
    lo, hi = [-1.0] * 3, [1.0] * 3
    h = 2.0 / (res - 1)
    plate = lambda p: tilted_plate(p, h, xp=torch).float()                    # noqa: E731  (elementwise: batch invariant)
    from nphm_b200.utils.reconstruction import create_grid_points_from_bounds
    pts = torch.from_numpy(create_grid_points_from_bounds(lo, hi, res)).to(cuda_device, dtype=torch.float32)
    dense = plate(pts).reshape((res,) * 3)
    vol, stats, band = narrowband_volume(plate, lo, hi, res, cuda_device, block=block, margin=4 * math.sqrt(3) * h)
    r = BO.band_volume(dense.cpu().numpy(), block=block, tau=4 * math.sqrt(3) * h)
    assert stats['growth_rounds'] == r['growth_rounds'] >= 2
    assert np.array_equal(band.block_states().cpu().numpy(), r['active'])
    v_b, t_b = _native.marching_cubes_device(vol, 0.0, negate=True)
    v_d, t_d = _native.marching_cubes_device(-dense, 0.0)
    assert len(v_d) > 0 and torch.equal(v_b, v_d) and torch.equal(t_b, t_d)
    mesh = _device_mesh(v_b, t_b, lo, hi, res)
    assert len(mesh.faces) == len(t_d)


def test_npm_deepsdf_mesh_equals_dense(cuda_device):
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband
    dec, lat = make_npm_head(cuda_device)
    for res in (64, 128):
        _, ref = _dense(dec, lat, res, 25000, cuda_device)
        mesh, stats = extract_mesh_narrowband(dec, lat, MINI, MAXI, res, nbatch_points=25000, return_stats=True)
        assert len(ref.vertices) > 0
        _assert_same_mesh(mesh, ref)
        assert stats['voxels_evaluated'] < res ** 3


def test_infinite_margin_evaluates_every_voxel(cuda_device, head):
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband
    dec, lat = head
    res = 64
    _, ref = _dense(dec, lat, res, 25000, cuda_device)
    mesh, stats = extract_mesh_narrowband(dec, lat, MINI, MAXI, res, nbatch_points=25000, margin=math.inf, return_stats=True)
    assert stats['voxels_evaluated'] == res ** 3 and stats['blocks_active'] == stats['blocks_total']
    _assert_same_mesh(mesh, ref)


def test_two_runs_bitwise_equal(cuda_device, head):
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband
    dec, lat = head
    a, sa = extract_mesh_narrowband(dec, lat, MINI, MAXI, 128, nbatch_points=25000, return_stats=True)
    b, sb = extract_mesh_narrowband(dec, lat, MINI, MAXI, 128, nbatch_points=25000, return_stats=True)
    _assert_same_mesh(a, b)
    assert sa == sb


def test_cpu_decoder_takes_the_dense_path(cuda_device):
    from nphm_b200.models.reconstruction import get_logits
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband, mesh_from_logits
    dec, lat, res = make_ensemble(0).eval(), sample_latent(1), 20
    ref = mesh_from_logits(get_logits(dec, lat, _grid(res, 'cpu'), nbatch_points=3000), MINI, MAXI, res)
    mesh, stats = extract_mesh_narrowband(dec, lat, MINI, MAXI, res, nbatch_points=3000, return_stats=True)
    _assert_same_mesh(mesh, ref)
    assert stats['voxels_evaluated'] == res ** 3


def test_error_paths(cuda_device, head):
    from ctypes import c_longlong
    from nphm_b200 import _native
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband, narrowband_volume
    dec, lat = head
    L = _native.lib()
    assert L.nphm_band_slab_workspace_bytes(1, 4, 0, 1) == -1 and L.nphm_band_slab_workspace_bytes(64, 0, 0, 16) == -1
    assert L.nphm_band_slab_workspace_bytes(1025, 4, 0, 256) == -1 and L.nphm_band_slab_workspace_bytes(64, 65, 0, 1) == -1
    with pytest.raises(_native.NativeError):
        extract_mesh_narrowband(dec, lat, MINI, MAXI, 32, margin=-1.0)
    with pytest.raises(_native.NativeError):
        extract_mesh_narrowband(dec, lat, MINI, MAXI, 32, margin=float('nan'))
    with pytest.raises(_native.NativeError):
        extract_mesh_narrowband(dec, lat, MINI, MAXI, 32, block=0)
    with pytest.raises(ValueError):
        narrowband_volume(lambda p: p[:, 0], MINI, MAXI, 32, cuda_device, quirk_period=10)
    need = L.nphm_band_slab_workspace_bytes(32, 4, 0, 8)
    ws = torch.empty(need - 1, device=cuda_device, dtype=torch.uint8)
    counts = (c_longlong * 2)()
    stream = torch.cuda.current_stream(cuda_device).cuda_stream
    assert L.nphm_band_slab_begin(32, 4, 0, 8, 0, ws.data_ptr(), ws.numel(), counts, stream) == -4     # NPHM_ERR_CAPACITY
    assert L.nphm_band_slab_begin(32, 4, 0, 8, -1, ws.data_ptr(), need, counts, stream) == -1          # negative quirk period
    assert L.nphm_band_slab_begin(32, 4, 0, 8, 0, None, need, counts, stream) == -1                    # no workspace
