"""Narrow band in block-sparse storage (csrc/narrowband_sparse.cu, ``sparse=True``, DESIGN §4.17) against the dense-storage band
and the dense path: the same mesh bit for bit, the same block states and counts, on one slab, on several slabs in one process and
on two gloo ranks, at 1024^3 against the dense-storage band, and at 2048^3 against a dense mesh built slab by slab."""
import math
import os
import socket

import numpy as np
import pytest
import torch

from conftest import MAXI, MINI, make_ensemble, sample_latent
from narrowband_common import make_npm_head, tilted_plate

pytestmark = pytest.mark.gpu

STAT_KEYS = ('blocks_active', 'voxels_evaluated', 'growth_rounds', 'blocks_total', 'voxels_total')


def _same_mesh(a, b):
    return (np.array_equal(np.asarray(a.faces), np.asarray(b.faces)) and np.array_equal(np.asarray(a.vertices), np.asarray(b.vertices))
            and len(a.vertices) > 0)


def _grid(res, dev, lo=MINI, hi=MAXI):
    from nphm_b200.utils.reconstruction import create_grid_points_from_bounds
    return torch.from_numpy(create_grid_points_from_bounds(lo, hi, res)).to(dev, dtype=torch.float32)


@pytest.fixture(scope='module')
def head(cuda_device):
    return make_ensemble(0, device=cuda_device).eval(), sample_latent(1).to(cuda_device)


@pytest.mark.parametrize('res,train,nbatch', [(64, False, 25000), (64, True, 25000), (128, False, 20000), (128, True, 20000),
                                              (256, False, 25000), (256, True, 25000), (64, False, 97)])
def test_ensemble_sparse_equals_dense_band_and_dense_path(cuda_device, head, res, train, nbatch):
    from nphm_b200.models.reconstruction import get_logits
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband, mesh_from_logits
    dec, lat = head
    dec.train(train)
    try:
        ref = mesh_from_logits(get_logits(dec, lat, _grid(res, cuda_device)[None], nbatch_points=nbatch), MINI, MAXI, res)
        band, sb = extract_mesh_narrowband(dec, lat, MINI, MAXI, res, nbatch_points=nbatch, return_stats=True)
        mesh, ss = extract_mesh_narrowband(dec, lat, MINI, MAXI, res, nbatch_points=nbatch, return_stats=True, sparse=True)
    finally:
        dec.eval()
    assert _same_mesh(mesh, ref) and _same_mesh(band, ref)
    assert all(ss[k] == sb[k] for k in STAT_KEYS), (ss, sb)
    assert ss['device_bytes']['band'] > 0 and 'device_bytes' not in sb


def test_npm_deepsdf_sparse_equals_dense(cuda_device):
    from nphm_b200.models.reconstruction import get_logits
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband, mesh_from_logits
    dec, lat = make_npm_head(cuda_device)
    for res in (64, 128):
        ref = mesh_from_logits(get_logits(dec, lat, _grid(res, cuda_device)[None], nbatch_points=25000), MINI, MAXI, res)
        _, sb = extract_mesh_narrowband(dec, lat, MINI, MAXI, res, nbatch_points=25000, return_stats=True)
        mesh, ss = extract_mesh_narrowband(dec, lat, MINI, MAXI, res, nbatch_points=25000, return_stats=True, sparse=True)
        assert _same_mesh(mesh, ref)
        assert all(ss[k] == sb[k] for k in STAT_KEYS)


def _mesh_of(band, vol, dev, sparse):
    from nphm_b200.utils.reconstruction import LocalExchange, _mc_pair, _slab_mesh
    return _slab_mesh([band], [vol], LocalExchange(1), *_mc_pair(sparse), dev)


def test_thin_plate_grows_and_fills_as_the_dense_band(cuda_device):
    from nphm_b200.utils.reconstruction import narrowband_volume
    res, block = 65, 4
    lo, hi = [-1.0] * 3, [1.0] * 3
    h = 2.0 / (res - 1)
    plate = lambda p: tilted_plate(p, h, xp=torch).float()                    # noqa: E731
    tau = 4 * math.sqrt(3) * h
    vd, sd, bd = narrowband_volume(plate, lo, hi, res, cuda_device, block=block, margin=tau)
    vs, ss, bs = narrowband_volume(plate, lo, hi, res, cuda_device, block=block, margin=tau, sparse=True)
    assert ss == sd and sd['growth_rounds'] >= 2
    assert torch.equal(bs.block_states(), bd.block_states())
    assert torch.equal(bs.dense_volume(), vd)
    v_d, t_d = _mesh_of(bd, vd, cuda_device, False)
    v_s, t_s = _mesh_of(bs, vs, cuda_device, True)
    assert len(v_d) > 0 and torch.equal(v_s, v_d) and torch.equal(t_s, t_d)


@pytest.mark.parametrize('train', [False, True])
def test_dense_volume_equals_filled_volume(cuda_device, head, train):
    from nphm_b200.utils.reconstruction import _band_evaluators, narrowband_volume
    dec, lat = head
    res, nbatch = 96, 5000
    dec.train(train)
    try:
        ev, evq = _band_evaluators(dec, lat, cuda_device)
        q = 0 if train else nbatch
        vd, sd, bd = narrowband_volume(ev, MINI, MAXI, res, cuda_device, quirk_period=q, evaluate_quirk=evq)
        vs, ss, bs = narrowband_volume(ev, MINI, MAXI, res, cuda_device, quirk_period=q, evaluate_quirk=evq, sparse=True)
    finally:
        dec.eval()
    assert ss == sd
    assert torch.equal(bs.block_states(), bd.block_states())
    assert torch.equal(bs.dense_volume(), vd)


@pytest.mark.parametrize('world', [2, 3, 8])
def test_slabs_equal_one_slab(cuda_device, head, world):
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband, extract_mesh_narrowband_slabs
    dec, lat = head
    ref, single = extract_mesh_narrowband(dec, lat, MINI, MAXI, 128, nbatch_points=20000, return_stats=True)
    mesh, st = extract_mesh_narrowband_slabs(dec, lat, MINI, MAXI, 128, world, nbatch_points=20000, return_stats=True, sparse=True)
    assert _same_mesh(mesh, ref)
    assert sum(st['blocks_active']) == single['blocks_active'] and st['growth_rounds'] == single['growth_rounds']
    dense_mesh, dst = extract_mesh_narrowband_slabs(dec, lat, MINI, MAXI, 128, world, nbatch_points=20000, return_stats=True)
    assert st['voxels_evaluated'] == dst['voxels_evaluated'] and st['bytes_exchanged'] == dst['bytes_exchanged']
    assert len(st['device_bytes']) == world


# ---------------------------------------------------------------------------------------------- analytic SDFs at 1024^3 and 2048^3
def _sdf(name, res):
    """Elementwise float32 SDF on [-1, 1]^3 (every path gets the same bits), evaluated in chunks to bound its temporaries."""
    h = 2.0 / (res - 1)
    c = torch.tensor(0.3 + 2 * h, dtype=torch.float32)

    def one(p):
        x, y, z = p[:, 0], p[:, 1], p[:, 2]
        if name == 'sphere':
            return torch.sqrt(x * x + y * y + z * z) - 0.5
        a = torch.sqrt((x - c) * (x - c) + y * y + z * z) - 0.3
        b = torch.sqrt((x + c) * (x + c) + y * y + z * z) - 0.3
        return torch.minimum(a, b)

    def f(p):
        out = torch.empty(p.shape[0], device=p.device, dtype=torch.float32)
        for i in range(0, p.shape[0], 1 << 24):
            out[i:i + (1 << 24)] = one(p[i:i + (1 << 24)])
        return out
    return f


def _band_run(name, res, dev, sparse):
    from nphm_b200.utils.reconstruction import narrowband_volume
    lo, hi = [-1.0] * 3, [1.0] * 3
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    vol, st, band = narrowband_volume(_sdf(name, res), lo, hi, res, dev, sparse=sparse)
    v, t = _mesh_of(band, vol, dev, sparse)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(dev) - base
    del vol, band
    return v, t, st, peak


@pytest.mark.parametrize('name', ['sphere', 'two_spheres'])
def test_1024_sparse_equals_dense_band_in_a_fraction_of_the_memory(cuda_device, name):
    vs, ts, ss, ps = _band_run(name, 1024, cuda_device, True)
    vd, td, sd, pd = _band_run(name, 1024, cuda_device, False)
    print('%s 1024^3: peak device memory sparse %.2f GB, dense storage %.2f GB' % (name, ps / 1e9, pd / 1e9))
    assert ss == sd
    assert len(vd) > 0 and torch.equal(vs, vd) and torch.equal(ts, td)
    assert ps < 0.25 * pd                                  # 1/4 of the dense-storage band's peak, evaluation included


def test_2048_sphere_equals_the_dense_mesh_built_slab_by_slab(cuda_device):
    from nphm_b200 import _native
    res = 2048
    vs, ts, ss, ps = _band_run('sphere', res, cuda_device, True)
    print('sphere 2048^3: peak device memory sparse %.2f GB, %d vertices' % (ps / 1e9, len(vs)))
    assert ps < 8e9                                        # the dense-storage band would need ~88 GB
    assert ss['voxels_evaluated'] < res ** 3 // 20
    f = _sdf('sphere', res)
    ax = torch.from_numpy(np.linspace(-1.0, 1.0, res).astype(np.float32))          # the band's float32(linspace_f64) axes
    yz = torch.stack(torch.meshgrid(ax, ax, indexing='ij'), -1).reshape(-1, 2).to(cuda_device)
    off_v = off_t = 0
    for a in range(0, res - 1, 64):                        # cell layers [a, b) from the planes [a - 1, b]
        b = min(a + 64, res - 1)
        first = max(a - 1, 0)
        xs = ax[first:b + 1].to(cuda_device)
        pts = torch.cat([xs.repeat_interleave(res * res)[:, None], yz.repeat(len(xs), 1)], 1)
        vol = (-f(pts)).reshape(len(xs), res, res)
        del pts
        nv, nt, p, ws = _native.marching_cubes_count(vol, 0.0, False, x_global0=first, ghost_lo=a > 0)
        v, t = _native.marching_cubes_emit(vol, p, ws, nv, nt, off_v)
        assert torch.equal(v, vs[off_v:off_v + nv]) and torch.equal(t, ts[off_t:off_t + nt]), 'cell layers [%d, %d)' % (a, b)
        off_v, off_t = off_v + nv, off_t + nt
    assert (off_v, off_t) == (len(vs), len(ts)) and off_v > 0


# ---------------------------------------------------------------------------------------------- syncs, determinism, errors
def test_two_runs_equal_and_no_torch_sync(cuda_device, head):
    from nphm_b200.utils.reconstruction import (LocalExchange, _band_evaluators, _mc_pair, default_margin, narrowband_slabs_mesh,
                                                plan_block_slabs)
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband
    from nphm_b200 import _native
    dec, lat = head
    a, sa = extract_mesh_narrowband(dec, lat, MINI, MAXI, 128, nbatch_points=25000, return_stats=True, sparse=True)
    b, sb = extract_mesh_narrowband(dec, lat, MINI, MAXI, 128, nbatch_points=25000, return_stats=True, sparse=True)
    assert _same_mesh(a, b) and sa == sb
    ev, evq = _band_evaluators(dec, lat, cuda_device)
    # pools large enough that no step has to grow one: then every slab synchronises once per listing step (begin, corners,
    # classify, one grow per round and the closing grow) and once for its marching-cubes counts, and torch not at all
    slabs = [_native.SparseNarrowBand(128, 4, cuda_device, l0, l1, slots=(l1 - l0) * 32 * 32) for l0, l1 in plan_block_slabs(128, 4, 2)]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        _, _, st = narrowband_slabs_mesh(slabs, ev, MINI, MAXI, 128, 4, default_margin(MINI, MAXI, 128, 4), LocalExchange(2), 25000,
                                         evq, *_mc_pair(True), device=cuda_device)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert [s.native_syncs for s in slabs] == [3 + st['growth_rounds'] + 1 + 1] * 2


def test_pool_grows_between_rounds(cuda_device, head):
    """A band that starts with one brick grows its pool as the band needs and gives the same mesh."""
    from nphm_b200 import _native
    from nphm_b200.utils.reconstruction import (LocalExchange, _band_evaluators, _mc_pair, default_margin, narrowband_slabs_mesh)
    dec, lat = head
    ev, evq = _band_evaluators(dec, lat, cuda_device)
    tau = default_margin(MINI, MAXI, 96, 4)
    outs = []
    for slots in (1, None):
        band = _native.SparseNarrowBand(96, 4, cuda_device, slots=slots)
        outs.append(narrowband_slabs_mesh([band], ev, MINI, MAXI, 96, 4, tau, LocalExchange(1), 20000, evq, *_mc_pair(True),
                                          device=cuda_device))
        assert band.slots >= band.slots_used > 1
    (v1, t1, s1), (v2, t2, s2) = outs
    assert torch.equal(v1, v2) and torch.equal(t1, t2) and s1 == s2


def test_error_paths(cuda_device):
    from ctypes import byref, c_longlong
    from nphm_b200 import _native
    L = _native.lib()
    assert L.nphm_band_sparse_workspace_bytes(8193, 4, 0, 2048) == -1          # res above the cap
    assert L.nphm_band_sparse_workspace_bytes(2048, 1, 0, 2047) == -1          # 2048^3 corners: u32 corner indices
    assert L.nphm_band_sparse_workspace_bytes(2048, 4, 0, 512) > 0
    assert L.nphm_band_sparse_workspace_bytes(64, 0, 0, 16) == -1 and L.nphm_band_sparse_workspace_bytes(64, 4, 3, 3) == -1
    with pytest.raises(_native.NativeError):
        _native.SparseNarrowBand(8193, 4, cuda_device)
    band = _native.SparseNarrowBand(64, 4, cuda_device, slots=1)
    counts = (c_longlong * 4)()
    stream = torch.cuda.current_stream(cuda_device).cuda_stream
    ws, n = band.ws.data_ptr(), band.ws.numel()
    assert L.nphm_band_sparse_begin(64, 4, 0, 16, 0, ws, n - 1, byref(band.pool), counts, stream) == -4       # short workspace
    assert L.nphm_band_sparse_begin(64, 4, 0, 16, -1, ws, n, byref(band.pool), counts, stream) == -1
    short = _native.BandPool.from_buffer_copy(band.pool)
    short.list_len = 0
    assert L.nphm_band_sparse_begin(64, 4, 0, 16, 0, ws, n, byref(short), counts, stream) == -4              # short pool buffers
    # a pool of one brick: the quirk blocks do not fit, nothing is written, and the bricks needed come back
    assert L.nphm_band_sparse_begin(64, 4, 0, 16, 5000, ws, n, byref(band.pool), counts, stream) == -4
    assert counts[3] > 1 and counts[2] == 0 and counts[0] == 0
    assert band.begin(5000) > 0 and band.slots >= band.slots_used > 1                                        # the binding grows it
    with pytest.raises(ValueError):
        band.classify(1.0, torch.zeros(1, device=cuda_device))
    # list entries are u32: at 2048^3 with 4^3-cell blocks a pool holds at most (2^32 - 1) // 5^3 of the 512^3 blocks' bricks
    big = _native.SparseNarrowBand(2048, 4, cuda_device, slots=1)
    assert big.max_slots == (2 ** 32 - 1) // 125 < big.n_blocks
    del big
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- torch.distributed (gloo)
def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _dist_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        from nphm_b200.distributed import extract_mesh_narrowband_sharded
        dec, lat = make_ensemble(0, device=dev).eval(), sample_latent(1).to(dev)
        mesh, stats = extract_mesh_narrowband_sharded(dec, lat, MINI, MAXI, 96, nbatch_points=20000, return_stats=True, sparse=True)
        if rank == 0:
            q.put((np.asarray(mesh.vertices).copy(), np.asarray(mesh.faces).copy(), stats))
        else:
            assert mesh is None and stats is None
    finally:
        dist.destroy_process_group()


def test_gloo_two_processes_sparse(cuda_device):
    import torch.multiprocessing as mp
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband
    ctx = mp.get_context('spawn')
    q = ctx.SimpleQueue()
    port = _free_port()
    procs = [ctx.Process(target=_dist_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        verts, faces, stats = q.get()
        for p in procs:
            p.join(300)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()
    dec, lat = make_ensemble(0, device=cuda_device).eval(), sample_latent(1).to(cuda_device)
    ref, single = extract_mesh_narrowband(dec, lat, MINI, MAXI, 96, nbatch_points=20000, return_stats=True)
    assert np.array_equal(verts, np.asarray(ref.vertices)) and np.array_equal(faces, np.asarray(ref.faces))
    assert sum(stats['blocks_active']) == single['blocks_active'] and stats['growth_rounds'] == single['growth_rounds']
