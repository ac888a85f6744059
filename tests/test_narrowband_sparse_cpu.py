"""The block-sparse narrow band (narrowband_sparse_common.OracleSparseSlab, the numpy restatement of csrc/narrowband_sparse.cu)
driven by the real host driver (nphm_b200.utils.reconstruction.narrowband_slabs_mesh): for every world size, the block states,
the evaluated voxels, the filled volume, the stats and the mesh are those of the dense-storage slabs and of the single-grid oracle
(oracle/band_oracle.py), and the marching cubes over x-chunks materialised from the bricks gives the ids of mc_oracle."""
import numpy as np
import pytest
import torch

from narrowband_common import analytic_volume
from narrowband_slab_common import oracle_slab_mc, oracle_slabs
from narrowband_sparse_common import oracle_sparse_mc, oracle_sparse_slabs
from oracle import band_oracle as BO
from oracle import nphm_oracle as O


def _tau(h, block=4):
    return block * np.sqrt(3) * h


def _run(dense, block, tau, world, quirk_period=0, sparse=True):
    from nphm_b200.utils.reconstruction import LocalExchange, narrowband_slabs_mesh
    res = dense.shape[0]
    flat = dense.reshape(-1)
    ref = BO.band_volume(dense, block=block, tau=tau, quirk_period=quirk_period)
    evaluate = lambda idx: torch.from_numpy(flat[idx.numpy()])         # noqa: E731
    slabs = (oracle_sparse_slabs if sparse else oracle_slabs)(res, block, world)
    count, emit = oracle_sparse_mc() if sparse else oracle_slab_mc(ref['volume'])
    verts, tris, stats = narrowband_slabs_mesh(slabs, evaluate, None, None, res, block, tau, LocalExchange(world), quirk_period,
                                               evaluate if quirk_period else None, count, emit)
    return ref, slabs, verts, tris, stats


def _check(dense, block, tau, world, quirk_period=0):
    res = dense.shape[0]
    ref, slabs, verts, tris, stats = _run(dense, block, tau, world, quirk_period)
    _, _, dverts, dtris, dstats = _run(dense, block, tau, world, quirk_period, sparse=False)
    live = [s for s in slabs if s is not None]
    assert stats == dstats                                               # blocks, voxels evaluated, rounds, bytes exchanged
    assert np.array_equal(np.concatenate([s.block_states().numpy() for s in live]), ref['active'])
    ev = np.zeros((res,) * 3, bool)
    for s in live:
        vol = s.dense_volume().numpy()
        assert np.array_equal(vol, ref['volume'][s.first_plane:s.x1 + 1])                  # the filled volume, ghost plane included
        ev[s.x0:s.x1 + 1] |= np.array([[[s.lookup(x, y, z)[1] for z in range(res)] for y in range(res)]
                                       for x in range(s.x0, s.x1 + 1)])
    assert np.array_equal(ev, ref['evaluated'])
    if world == 1:
        assert stats['voxels_evaluated'] == [ref['voxels_evaluated']] and stats['growth_rounds'] == ref['growth_rounds']
    rv, rt = O.marching_cubes(ref['volume'], 0.0, True)
    dv, dt = O.marching_cubes(dense, 0.0, True)
    assert len(rv) > 0 and np.array_equal(rv, dv) and np.array_equal(rt, dt)
    assert np.array_equal(verts.numpy(), rv) and np.array_equal(tris.numpy().astype(np.uint64), rt)
    assert torch.equal(verts, dverts) and torch.equal(tris, dtris)
    return ref, stats


@pytest.mark.parametrize('world', [1, 2, 3, 5])
@pytest.mark.parametrize('name,res', [('sphere', 33), ('torus', 41), ('two_spheres', 49), ('thin_plate', 49)])
def test_sparse_slabs_equal_dense_slabs_and_oracle(name, res, world):
    dense, h = analytic_volume(name, res)
    _check(dense, 4, _tau(h), world)


def test_thin_plate_grows():
    dense, h = analytic_volume('thin_plate', 65)
    ref, stats = _check(dense, 4, _tau(h), 1)
    assert ref['growth_rounds'] >= 2


@pytest.mark.parametrize('world', [1, 2, 3])
def test_quirk_voxels_on_shared_planes(world):
    """Quirk period 33^2 * 8 + 1: quirk voxels lie on the planes 8, 16, 24 the slabs share, and their blocks are forced on both sides."""
    dense, h = analytic_volume('sphere', 33)
    ref, stats = _check(dense, 4, _tau(h), world, quirk_period=33 * 33 * 8 + 1)
    assert ref['voxels_evaluated'] > 0


@pytest.mark.parametrize('world', [1, 3])
def test_brick_ids_equal_mc_oracle_on_the_materialised_volume(world):
    """The restated brick marching cubes of every slab, on its bricks alone, gives mc_oracle's ids, positions and triangles on the
    slab's filled volume (the one-volume ids of the slab's own cells, shifted by the ghost layer's vertices)."""
    from narrowband_sparse_common import brick_marching_cubes
    dense, h = analytic_volume('torus', 41)
    ref, slabs, verts, tris, _ = _run(dense, 4, _tau(h), world)
    vol = ref['volume']
    for s in (s for s in slabs if s is not None):
        v, t = brick_marching_cubes(s)
        first_own = s.x0                                 # vertices created by cells before layer x0 come before the slab's
        n_before = len(O.marching_cubes(vol[:first_own + 1], 0.0, True)[0]) if first_own > 0 else 0
        rv, rt = O.marching_cubes(vol[:s.x1 + 1], 0.0, True)
        _, pt = O.marching_cubes(vol[:first_own + 1], 0.0, True) if first_own > 0 else (None, np.zeros((0, 3)))
        assert len(v) > 0 and np.array_equal(v, rv[n_before:])
        assert np.array_equal((t + n_before).astype(np.uint64), rt[len(pt):])
