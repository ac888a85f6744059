"""The narrow band on x-slabs (nphm_b200.utils.reconstruction.narrowband_slabs_mesh) with the numpy restatement of the slab steps
(narrowband_slab_common.OracleSlab): for every world size, the mesh, the block states, the evaluated voxels and the filled
volume are the single-grid oracle's (oracle/band_oracle.py), in process and through gloo."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from narrowband_common import analytic_volume, tilted_plate
from narrowband_slab_common import DONE, oracle_slab_mc, oracle_slabs, OracleSlab
from oracle import band_oracle as BO
from oracle import nphm_oracle as O


def _tau(h, block=4):
    return block * np.sqrt(3) * h


def _run(dense, block, tau, world, quirk_period=0, exchange=None, slabs=None):
    from nphm_b200.utils.reconstruction import LocalExchange, narrowband_slabs_mesh
    res = dense.shape[0]
    flat = dense.reshape(-1)
    ref = BO.band_volume(dense, block=block, tau=tau, quirk_period=quirk_period)
    evaluate = lambda idx: torch.from_numpy(flat[idx.numpy()])         # noqa: E731
    slabs = oracle_slabs(res, block, world) if slabs is None else slabs
    count, emit = oracle_slab_mc(ref['volume'])
    verts, tris, stats = narrowband_slabs_mesh(slabs, evaluate, None, None, res, block, tau, exchange or LocalExchange(world),
                                               quirk_period, evaluate if quirk_period else None, count, emit)
    return ref, slabs, verts, tris, stats


def _check_against_oracle(dense, ref, slabs, verts, tris, stats):
    res = dense.shape[0]
    live = [s for s in slabs if s is not None]
    # block states: the slabs' layers concatenated along x are the single grid's
    assert np.array_equal(np.concatenate([s.block_states().numpy() for s in live]), ref['active'])
    assert sum(stats['blocks_active']) == int(ref['active'].sum())
    # evaluated voxels: the union is the single grid's; a voxel may be evaluated twice only on a shared plane
    ev = np.zeros((res,) * 3, bool)
    for s in live:
        mine = s.marks == DONE
        twice = ev[s.x0:s.x1 + 1] & mine
        assert not twice[1:].any()
        ev[s.x0:s.x1 + 1] |= mine
    assert np.array_equal(ev, ref['evaluated'])
    assert sum(stats['voxels_evaluated']) >= ref['voxels_evaluated']
    # the mesh: the single-grid band's, and the dense one's
    rv, rt = O.marching_cubes(ref['volume'], 0.0, True)
    dv, dt = O.marching_cubes(dense, 0.0, True)
    assert len(rv) > 0 and np.array_equal(rv, dv) and np.array_equal(rt, dt)
    assert np.array_equal(verts.numpy(), rv) and np.array_equal(tris.numpy().astype(np.uint64), rt)


@pytest.mark.parametrize('world', [1, 2, 3, 5])
@pytest.mark.parametrize('name,res', [('sphere', 33), ('torus', 49), ('two_spheres', 65), ('thin_plate', 65)])
def test_slabs_equal_single_grid(name, res, world):
    dense, h = analytic_volume(name, res)
    ref, slabs, verts, tris, stats = _run(dense, 4, _tau(h), world)
    _check_against_oracle(dense, ref, slabs, verts, tris, stats)
    assert len(stats['blocks_active']) == world and len(stats['bytes_exchanged']) == world
    assert all(len(b) == stats['growth_rounds'] + 2 for b in stats['bytes_exchanged'])
    if world == 1:
        assert stats['growth_rounds'] == ref['growth_rounds'] and stats['bytes_exchanged'] == [[0] * (ref['growth_rounds'] + 2)]


class _NoBoundaryExchange:
    """The in-process exchange with the shared planes dropped (the ghost planes still move): growth no longer sees what the
    neighbour evaluated."""

    def __init__(self, world):
        from nphm_b200.utils.reconstruction import LocalExchange
        self.inner = LocalExchange(world)
        self.ranks = self.inner.ranks

    def swap(self, sends, expects, nbytes):
        got = self.inner.swap(sends, expects, nbytes)
        ghost = all(s[0] is None for s in sends)
        return got if ghost else [(None, None)] * len(got)

    def __getattr__(self, name):
        return getattr(self.inner, name)


def _plate_along_x(res):
    """tilted_plate with its normal mostly along z: the plate spans the x axis, so the band grows along it through the slab
    boundaries."""
    ax = np.linspace(-1.0, 1.0, res)
    X, Y, Z = np.meshgrid(ax, ax, ax, indexing='ij')
    h = 2.0 / (res - 1)
    return tilted_plate(np.stack([Z, Y, X], -1), h).astype(np.float32), h


def test_growth_crosses_slab_boundaries():
    dense, h = _plate_along_x(65)
    ref, slabs, verts, tris, stats = _run(dense, 4, _tau(h), 5)
    assert ref['growth_rounds'] >= 2
    _check_against_oracle(dense, ref, slabs, verts, tris, stats)
    # without the boundary exchange the slabs miss blocks the single grid activates: growth did cross a boundary
    slabs2 = oracle_slabs(65, 4, 5)
    from nphm_b200.utils.reconstruction import narrowband_slab_volumes
    flat = dense.reshape(-1)
    ev = lambda idx: torch.from_numpy(flat[idx.numpy()])               # noqa: E731
    narrowband_slab_volumes(slabs2, ev, None, None, _tau(h), _NoBoundaryExchange(5))
    cut = np.concatenate([s.block_states().numpy() for s in slabs2])
    assert cut.sum() < ref['active'].sum() and not (cut & ~ref['active']).any()


def test_surface_inside_one_slab():
    res = 65
    ax = np.linspace(-1.0, 1.0, res)
    X, Y, Z = np.meshgrid(ax, ax, ax, indexing='ij')
    h = 2.0 / (res - 1)
    c = -1.0 + 34 * h                                    # slab 2 of 5 holds the planes 28 .. 40
    dense = (np.sqrt((X - c) ** 2 + Y ** 2 + Z ** 2) - 4.5 * h).astype(np.float32)
    ref, slabs, verts, tris, stats = _run(dense, 4, 1.0 * h, 5)
    _check_against_oracle(dense, ref, slabs, verts, tris, stats)
    assert [a > 0 for a in stats['blocks_active']] == [False, False, True, False, False]


def test_world_larger_than_block_layers():
    dense, h = analytic_volume('sphere', 17)             # 4 block layers over 6 ranks: the last two own nothing
    ref, slabs, verts, tris, stats = _run(dense, 4, _tau(h), 6)
    assert slabs[4] is None and slabs[5] is None
    _check_against_oracle(dense, ref, slabs, verts, tris, stats)
    assert stats['blocks_active'][4:] == [0, 0] and stats['voxels_evaluated'][4:] == [0, 0]


@pytest.mark.parametrize('period', [33 * 33, 8 * 33 * 33 + 1, 97])
@pytest.mark.parametrize('world', [1, 2, 3, 5])
def test_quirk_voxels_on_boundary_planes(period, world):
    """period res^2: the quirk voxels are the last voxel of every plane, so every shared plane holds one; period 8 res^2 + 1: the
    k-th lies on plane 8k, a block face; both ranks around a boundary list it and activate their blocks around it."""
    dense, h = analytic_volume('torus', 33)
    g = np.union1d(np.arange(period - 1, 33 ** 3, period), [33 ** 3 - 1])
    dense.reshape(-1)[g] = 1.0                           # the spurious values of get_logits' last point of every chunk
    ref, slabs, verts, tris, stats = _run(dense, 4, _tau(h), world, quirk_period=period)
    assert ref['evaluated'].reshape(-1)[g].all()
    _check_against_oracle(dense, ref, slabs, verts, tris, stats)


def test_slab_restatement_rejects_planes_it_does_not_share():
    s = OracleSlab(33, 4, 2, 5)
    s.begin()
    vol = s.volume()
    with pytest.raises(AssertionError):
        s.import_(s.x0 + 1, s.export(s.x0, vol), vol)


# ---------------------------------------------------------------------------------------------- gloo: the real GroupExchange
def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _gloo_worker(rank, world, port, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        from nphm_b200.distributed import GroupExchange
        from nphm_b200.utils.reconstruction import narrowband_slabs_mesh, plan_block_slabs
        dense, h = _plate_along_x(49)
        period = 49 * 49
        g = np.union1d(np.arange(period - 1, 49 ** 3, period), [49 ** 3 - 1])
        dense.reshape(-1)[g] = 1.0
        ref = BO.band_volume(dense, block=4, tau=_tau(h), quirk_period=period)
        l0, l1 = plan_block_slabs(49, 4, world)[rank]
        slab = OracleSlab(49, 4, l0, l1)
        flat = dense.reshape(-1)
        ev = lambda idx: torch.from_numpy(flat[idx.numpy()])           # noqa: E731
        count, emit = oracle_slab_mc(ref['volume'])
        verts, tris, stats = narrowband_slabs_mesh([slab], ev, None, None, 49, 4, _tau(h), GroupExchange('cpu'), period, ev,
                                                   count, emit)
        states = slab.block_states().numpy()
        assert np.array_equal(states, ref['active'][l0:l1])
        assert sum(stats['blocks_active']) == int(ref['active'].sum())
        if rank == 0:
            rv, rt = O.marching_cubes(ref['volume'], 0.0, True)
            q.put(bool(len(rv) > 0 and np.array_equal(verts.numpy(), rv) and np.array_equal(tris.numpy().astype(np.uint64), rt)
                       and stats['growth_rounds'] >= 1 and len(stats['bytes_exchanged']) == world))
        else:
            assert verts is None and tris is None
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('world', [2, 3])
def test_group_exchange_gloo(world):
    """The host driver on gloo ranks, one oracle slab each; at world 3 the middle rank has two neighbours."""
    ctx = mp.get_context('spawn')
    q = ctx.SimpleQueue()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        for p in procs:
            p.join(300)
            assert p.exitcode == 0
        assert q.get() is True
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()
