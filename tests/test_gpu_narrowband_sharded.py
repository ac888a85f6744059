"""The narrow band sharded in x-slabs (nphm_band_slab_*, nphm_b200.distributed.extract_mesh_narrowband_sharded) on one H100:
every slab of the grid driven by one process through the in-process exchange, and two gloo ranks sharing the GPU.  Rank 0's
mesh is bit for bit extract_mesh_narrowband's and the dense mesh_from_logits(get_logits(...))'s."""
import math
import os
import socket

import numpy as np
import pytest
import torch

from conftest import MAXI, MINI, make_ensemble, sample_latent
from narrowband_common import make_npm_head, tilted_plate

pytestmark = pytest.mark.gpu

WORLDS = [1, 2, 3, 8]


def _same_mesh(a, b):
    va, vb = np.asarray(a.vertices), np.asarray(b.vertices)
    fa, fb = np.asarray(a.faces), np.asarray(b.faces)
    return va.shape == vb.shape and fa.shape == fb.shape and np.array_equal(fa, fb) and np.array_equal(va, vb)


def _dense(dec, lat, res, nbatch, dev):
    from nphm_b200.models.reconstruction import get_logits
    from nphm_b200.utils.reconstruction import create_grid_points_from_bounds, mesh_from_logits
    grid = torch.from_numpy(create_grid_points_from_bounds(MINI, MAXI, res)).to(dev, dtype=torch.float32)[None]
    logits = get_logits(dec, lat, grid, nbatch_points=nbatch)
    vol = logits.copy()
    return vol.reshape((res,) * 3), mesh_from_logits(logits, MINI, MAXI, res)


@pytest.fixture(scope='module')
def head(cuda_device):
    return make_ensemble(0, device=cuda_device).eval(), sample_latent(1).to(cuda_device)


_REFS = {}


def _refs(key, dec, lat, res, nbatch, dev):
    """(dense mesh, extract_mesh_narrowband mesh, its stats), once per decoder and setting."""
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband
    if key not in _REFS:
        _, dense = _dense(dec, lat, res, nbatch, dev)
        band, stats = extract_mesh_narrowband(dec, lat, MINI, MAXI, res, nbatch_points=nbatch, return_stats=True)
        assert len(dense.vertices) > 0 and _same_mesh(band, dense)
        _REFS[key] = dense, band, stats
    return _REFS[key]


def _check_stats(stats, single, world):
    assert len(stats['blocks_active']) == world and sum(stats['blocks_active']) == single['blocks_active']
    # a voxel is evaluated twice at most, and only on one of the world - 1 shared planes
    extra = sum(stats['voxels_evaluated']) - single['voxels_evaluated']
    assert 0 <= extra <= (world - 1) * stats['voxels_total'] ** (2 / 3) + 1
    assert stats['blocks_total'] == single['blocks_total'] and stats['margin'] == single['margin']


@pytest.mark.parametrize('world', WORLDS)
@pytest.mark.parametrize('res,train,nbatch', [(64, False, 25000), (64, True, 25000), (128, False, 20000), (128, True, 20000)])
def test_ensemble_slabs_equal_single_gpu_band(cuda_device, head, res, train, nbatch, world):
    from nphm_b200.distributed import extract_mesh_narrowband_slabs
    dec, lat = head
    dec.train(train)
    try:
        dense, band, single = _refs(('nphm', res, train, nbatch), dec, lat, res, nbatch, cuda_device)
        mesh, stats = extract_mesh_narrowband_slabs(dec, lat, MINI, MAXI, res, world, nbatch_points=nbatch, return_stats=True)
    finally:
        dec.eval()
    assert _same_mesh(mesh, band) and _same_mesh(mesh, dense)
    assert torch.equal(mesh._nphm_device_vertices, band._nphm_device_vertices)
    _check_stats(stats, single, world)


@pytest.mark.parametrize('world', WORLDS)
def test_npm_deepsdf_slabs_equal_single_gpu_band(cuda_device, world):
    from nphm_b200.distributed import extract_mesh_narrowband_slabs
    dec, lat = make_npm_head(cuda_device)
    dense, band, single = _refs(('npm', 64), dec, lat, 64, 25000, cuda_device)
    mesh, stats = extract_mesh_narrowband_slabs(dec, lat, MINI, MAXI, 64, world, nbatch_points=25000, return_stats=True)
    assert _same_mesh(mesh, band) and _same_mesh(mesh, dense)
    _check_stats(stats, single, world)


def _slab_run(evaluate, res, block, tau, world, dev, quirk_period=0, evaluate_quirk=None, lo=MINI, hi=MAXI):
    from nphm_b200 import _native
    from nphm_b200.utils.reconstruction import LocalExchange, narrowband_slab_volumes, plan_block_slabs
    slabs = [None if l1 <= l0 else _native.NarrowBandSlab(res, block, l0, l1, dev) for l0, l1 in plan_block_slabs(res, block, world)]
    vols, stats = narrowband_slab_volumes(slabs, evaluate, lo, hi, tau, LocalExchange(world), quirk_period, evaluate_quirk)
    return slabs, vols, stats


@pytest.mark.parametrize('world', WORLDS)
def test_thin_plate_across_slabs(cuda_device, world):
    """The analytic plate spanning the x axis: the band grows along it through the slab boundaries, and every slab's filled
    volume (ghost plane included) and block states are the single-grid band's."""
    from nphm_b200 import _native
    from nphm_b200.utils.reconstruction import (LocalExchange, create_grid_points_from_bounds, narrowband_slabs_mesh,
                                                narrowband_volume, plan_block_slabs)
    res, block = 65, 4
    lo, hi = [-1.0] * 3, [1.0] * 3
    h = 2.0 / (res - 1)
    plate = lambda p: tilted_plate(p[:, [2, 1, 0]], h, xp=torch).float()     # noqa: E731  (normal mostly along z)
    pts = torch.from_numpy(create_grid_points_from_bounds(lo, hi, res)).to(cuda_device, dtype=torch.float32)
    dense = plate(pts).reshape((res,) * 3)
    tau = 4 * math.sqrt(3) * h
    vol, single, band = narrowband_volume(plate, lo, hi, res, cuda_device, block=block, margin=tau)
    assert single['growth_rounds'] >= 2
    slabs, vols, stats = _slab_run(plate, res, block, tau, world, cuda_device, lo=lo, hi=hi)
    live = [(s, v) for s, v in zip(slabs, vols) if s is not None]
    assert torch.equal(torch.cat([s.block_states() for s, _ in live]), band.block_states())
    for s, v in live:
        assert torch.equal(v, vol[s.first_plane:s.x1 + 1])
    slabs = [None if l1 <= l0 else _native.NarrowBandSlab(res, block, l0, l1, cuda_device) for l0, l1 in plan_block_slabs(res, block, world)]
    verts, tris, _ = narrowband_slabs_mesh(slabs, plate, lo, hi, res, block, tau, LocalExchange(world), device=cuda_device)
    v_d, t_d = _native.marching_cubes_device(-dense, 0.0)
    assert len(v_d) > 0 and torch.equal(verts, v_d) and torch.equal(tris, t_d)


@pytest.mark.parametrize('train', [False, True])
def test_evaluated_voxels_are_the_single_band_and_dense(cuda_device, head, train):
    """Every slab's own planes hold the single-GPU band's filled volume bit for bit (so its evaluated voxels are the dense
    values), and the slabs' active blocks are the single band's: the union of the evaluated voxels is the single band's, apart
    from the duplicates on the shared planes."""
    from nphm_b200.utils.reconstruction import _band_evaluators, default_margin, narrowband_volume
    dec, lat = head
    res, nbatch, block = 96, 5000, 4
    dec.train(train)
    try:
        dense, _ = _dense(dec, lat, res, nbatch, cuda_device)
        ev, evq = _band_evaluators(dec, lat, cuda_device)
        period = 0 if train else nbatch
        vol, single, band = narrowband_volume(ev, MINI, MAXI, res, cuda_device, block=block, quirk_period=period, evaluate_quirk=evq)
        tau = default_margin(MINI, MAXI, res, block)
        for world in (3, 8):
            slabs, vols, stats = _slab_run(ev, res, block, tau, world, cuda_device, period, evq)
            for s, v in zip(slabs, vols):
                assert torch.equal(v, vol[s.first_plane:s.x1 + 1])
            assert torch.equal(torch.cat([s.block_states() for s in slabs]), band.block_states())
    finally:
        dec.eval()
    states = band.block_states().cpu().numpy()
    m = np.zeros((res,) * 3, bool)
    for bx, by, bz in zip(*np.nonzero(states)):
        a = np.array([bx, by, bz]) * block
        b = np.minimum(a + block, res - 1)
        m[a[0]:b[0] + 1, a[1]:b[1] + 1, a[2]:b[2] + 1] = True
    assert np.array_equal(vol.cpu().numpy()[m], dense[m])


def test_two_runs_bitwise_equal_and_no_host_sync(cuda_device, head):
    """Two runs give the same mesh and stats; the round loop makes no synchronising torch call (the per-round count read-back
    is the native listing step's)."""
    from nphm_b200.distributed import extract_mesh_narrowband_slabs
    from nphm_b200.utils.reconstruction import _band_evaluators, default_margin
    dec, lat = head
    a, sa = extract_mesh_narrowband_slabs(dec, lat, MINI, MAXI, 128, 3, nbatch_points=25000, return_stats=True)
    b, sb = extract_mesh_narrowband_slabs(dec, lat, MINI, MAXI, 128, 3, nbatch_points=25000, return_stats=True)
    assert _same_mesh(a, b) and sa == sb
    ev, evq = _band_evaluators(dec, lat, cuda_device)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        _slab_run(ev, 128, 4, default_margin(MINI, MAXI, 128, 4), 3, cuda_device, 25000, evq)
    finally:
        torch.cuda.set_sync_debug_mode(0)


def test_error_paths(cuda_device):
    from ctypes import c_longlong
    from nphm_b200 import _native
    L = _native.lib()
    for l0, l1 in ((3, 3), (5, 4), (-1, 2), (0, 17)):
        assert L.nphm_band_slab_workspace_bytes(65, 4, l0, l1) == -1
        with pytest.raises(_native.NativeError):
            _native.NarrowBandSlab(65, 4, l0, l1, cuda_device)
    need = L.nphm_band_slab_workspace_bytes(65, 4, 4, 8)
    assert 0 < need < L.nphm_band_slab_workspace_bytes(65, 4, 0, 16)
    ws = torch.empty(need, device=cuda_device, dtype=torch.uint8)
    counts = (c_longlong * 2)()
    stream = torch.cuda.current_stream(cuda_device).cuda_stream
    assert L.nphm_band_slab_begin(65, 4, 4, 8, 0, ws.data_ptr(), need - 1, counts, stream) == -4       # NPHM_ERR_CAPACITY
    assert L.nphm_band_slab_begin(65, 4, 4, 9, 0, ws.data_ptr(), need, counts, stream) == -4           # a larger slab's
    assert L.nphm_band_slab_begin(65, 4, 4, 8, -1, ws.data_ptr(), need, counts, stream) == -1
    mid = _native.NarrowBandSlab(65, 4, 4, 8, cuda_device)                  # planes 16 .. 32, shared both ways
    first = _native.NarrowBandSlab(65, 4, 0, 4, cuda_device)                # planes 0 .. 16, no lower neighbour
    mid.begin()
    first.begin()
    vm, vf = mid.volume(), first.volume()
    buf = mid.export(16, vm)
    assert buf.numel() == 5 * 65 * 65
    for plane in (17, 31, 14, 33):                                         # not shared, and not the ghost plane 15
        with pytest.raises(_native.NativeError):
            mid.import_(plane, buf, vm)
    for plane in (15, 33):
        with pytest.raises(_native.NativeError):
            mid.export(plane, vm)
    with pytest.raises(_native.NativeError):
        first.import_(0, buf, vf)                                           # plane 0 is nobody's to share
    with pytest.raises(_native.NativeError):
        first.import_(-1, buf, vf)                                          # the first slab has no ghost plane
    with pytest.raises(ValueError):
        mid.import_(16, buf[:-1], vm)
    mid.import_(16, first.export(16, vf), vm)
    mid.import_(15, first.export(15, vf), vm)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- torch.distributed
def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _dist_worker(rank, world, port, backend, q):
    import torch.distributed as dist
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dev = torch.device('cuda', rank if backend == 'nccl' else 0)
    torch.cuda.set_device(dev)
    kw = {'device_id': dev} if backend == 'nccl' else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    try:
        from nphm_b200.distributed import extract_mesh_narrowband_sharded
        dec, lat = make_ensemble(0, device=dev).eval(), sample_latent(1).to(dev)
        mesh, stats = extract_mesh_narrowband_sharded(dec, lat, MINI, MAXI, 96, nbatch_points=20000, return_stats=True)
        if rank == 0:
            q.put((np.asarray(mesh.vertices).copy(), np.asarray(mesh.faces).copy(), stats))
        else:
            assert mesh is None and stats is None
    finally:
        dist.destroy_process_group()


def _run_ranks(world, backend):
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.SimpleQueue()
    port = _free_port()
    procs = [ctx.Process(target=_dist_worker, args=(r, world, port, backend, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        out = q.get()
        for p in procs:
            p.join(300)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()
    return out


def _check_rank0(out, cuda_device, world):
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband
    verts, faces, stats = out
    dec, lat = make_ensemble(0, device=cuda_device).eval(), sample_latent(1).to(cuda_device)
    ref, single = extract_mesh_narrowband(dec, lat, MINI, MAXI, 96, nbatch_points=20000, return_stats=True)
    assert len(ref.vertices) > 0
    assert np.array_equal(verts, np.asarray(ref.vertices)) and np.array_equal(faces, np.asarray(ref.faces))
    _check_stats(stats, single, world)
    assert stats['slabs'] == [(0, 12), (12, 24)]
    assert all(b == [5 * 96 * 96] * (stats['growth_rounds'] + 1) + [b[-1]] for b in stats['bytes_exchanged'])


def test_gloo_two_processes_share_the_gpu(cuda_device):
    """Two ranks on one GPU through gloo (planes and mesh staged through host tensors): rank 0's mesh is the single-GPU band's."""
    _check_rank0(_run_ranks(2, 'gloo'), cuda_device, 2)


def test_nccl_two_gpus(cuda_device):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    _check_rank0(_run_ranks(2, 'nccl'), cuda_device, 2)
