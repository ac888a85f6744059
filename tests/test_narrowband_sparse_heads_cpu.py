"""The block-sparse band of S heads without a GPU: a numpy restatement of nphm_band_sparse_heads_* (S OracleSparseSlabs of the
whole grid behind the interface of _native.SparseNarrowBandHeads, with its pool policy) driven by the real host driver
(utils/reconstruction.narrowband_heads_volumes).  For every head, the block states, evaluated voxels, filled volume, stats and
brick marching cubes equal the single-grid oracle's (oracle/band_oracle.py) and mc_oracle's ids, whatever the pool's first size."""
import copy

import numpy as np
import pytest
import torch

from narrowband_common import analytic_volume, tilted_plate
from narrowband_sparse_common import OracleSparseSlab, brick_marching_cubes
from oracle import band_oracle as BO
from oracle import nphm_oracle as O


class OracleSparseHeads:
    """S :class:`OracleSparseSlab` of the whole grid in lockstep, with the pool policy of the native band: S pools of one size.  A
    listing step that needs more bricks in some head than a pool holds changes no head; the pools grow (to at least twice their
    size) and the same step repeats, as ``SparseNarrowBandHeads._call_listing`` does.  ``gather`` yields S x n_pad global flat
    indices, each head's listed voxels first, then the padding rows the kernels write (its last listed voxel, voxel 0 when it listed
    nothing)."""

    def __init__(self, res, block, n_heads, slots):
        self.res, self.block, self.n_heads = int(res), int(block), int(n_heads)
        self.blocks_per_axis = -(-(self.res - 1) // self.block)
        self.heads = [OracleSparseSlab(res, block, 0, self.blocks_per_axis) for _ in range(n_heads)]
        self.slots = int(slots)
        self.retries = 0
        self.readbacks = 0
        self.active_blocks = [0] * n_heads

    def _step(self, fn):
        while True:
            trial = [copy.deepcopy(h) for h in self.heads]
            ns = [fn(h) for h in trial]
            self.readbacks += 1
            need = max(len(h.sblock) for h in trial)
            if need <= self.slots:
                break
            self.retries += 1
            self.slots = max(need, 2 * self.slots)
        self.heads = trial
        self.active_blocks = [h.active_blocks for h in self.heads]
        return ns

    def _own(self, vols):
        assert vols is self

    def volumes(self):
        return self

    def begin(self, quirk_period=0):
        return self._step(lambda h: h.begin(quirk_period))

    def corners(self):
        return self._step(lambda h: h.corners())

    def classify(self, tau, vols):
        self._own(vols)
        return self._step(lambda h: h.classify(tau, h))

    def grow(self, vols):
        self._own(vols)
        return self._step(lambda h: h.grow(h))

    def gather(self, n_pad, mini, maxi):
        out = torch.zeros(self.n_heads, n_pad, dtype=torch.int64)
        for i, h in enumerate(self.heads):
            idx = h.gather(len(h.list), mini, maxi)
            out[i, :len(idx)] = idx
            if len(idx):
                out[i, len(idx):] = idx[-1]
        return out

    def scatter(self, values, vols):
        self._own(vols)
        for h, v in zip(self.heads, values):
            h.scatter(v[:len(h.list)], h)

    def fill(self, vols):
        self._own(vols)

    def block_states(self):
        return torch.stack([h.block_states() for h in self.heads])

    def marching_cubes(self, vols):
        self._own(vols)
        parts = [brick_marching_cubes(h) for h in self.heads]
        return (np.concatenate([v for v, _ in parts]), np.concatenate([t for _, t in parts]),
                [(len(v), len(t)) for v, t in parts])


def _tau(h, block=4):
    return block * np.sqrt(3) * h


def _heads_volumes(res):
    """Heads that close at different rounds: spheres of three radii, a field without a surface, and the thin plate (growth)."""
    ax = np.linspace(-1.0, 1.0, res)
    X, Y, Z = np.meshgrid(ax, ax, ax, indexing='ij')
    h = 2.0 / (res - 1)
    r = np.sqrt(X ** 2 + Y ** 2 + Z ** 2)
    return [(r - 0.5).astype(np.float32), (r + 5.0).astype(np.float32),
            tilted_plate(np.stack([X, Y, Z], -1), h).astype(np.float32), (r - 0.27).astype(np.float32),
            analytic_volume('torus', res)[0]], h


def _run(vols, block, tau, slots, quirk_period=0):
    from nphm_b200.utils.reconstruction import narrowband_heads_volumes
    flats = [v.reshape(-1) for v in vols]
    S = len(vols)

    def evaluate(idx):                  # S x n_pad global indices -> S x n_pad values
        assert idx.shape[0] == S and idx.shape[1] % 128 == 0
        return torch.stack([torch.from_numpy(f[i.numpy()]) for f, i in zip(flats, idx)])

    bands = OracleSparseHeads(vols[0].shape[0], block, S, slots)
    out, stats = narrowband_heads_volumes(bands, evaluate, None, None, tau, quirk_period, evaluate if quirk_period else None)
    assert out is bands
    return bands, stats


def _check(vols, block, tau, slots, quirk_period=0):
    res = vols[0].shape[0]
    bands, stats = _run(vols, block, tau, slots, quirk_period)
    states = bands.block_states().numpy()
    verts, tris, counts = bands.marching_cubes(bands)
    v_off = t_off = 0
    for i, (dense, head) in enumerate(zip(vols, bands.heads)):
        ref = BO.band_volume(dense, block=block, tau=tau, quirk_period=quirk_period)
        assert np.array_equal(states[i], ref['active']), 'head %d' % i
        assert np.array_equal(head.dense_volume().numpy(), ref['volume']), 'head %d' % i
        ev = np.array([[[head.lookup(x, y, z)[1] for z in range(res)] for y in range(res)] for x in range(res)])
        assert np.array_equal(ev, ref['evaluated']), 'head %d' % i
        assert stats[i]['voxels_evaluated'] == ref['voxels_evaluated'] and stats[i]['growth_rounds'] == ref['growth_rounds']
        assert stats[i]['blocks_active'] == int(ref['active'].sum())
        rv, rt = O.marching_cubes(ref['volume'], 0.0, True)
        nv, nt = counts[i]
        assert (nv, nt) == (len(rv), len(rt))
        assert np.array_equal(verts[v_off:v_off + nv], rv) and np.array_equal(tris[t_off:t_off + nt].astype(np.uint64), rt)
        v_off, t_off = v_off + nv, t_off + nt
    # one read-back per listing step whatever S is, plus one per capacity retry
    assert bands.readbacks == 3 + max(s['growth_rounds'] for s in stats) + 1 + bands.retries
    return bands, stats


@pytest.mark.parametrize('quirk', [False, True])
def test_heads_equal_single_grid_oracle(quirk):
    """Five heads of a 33^3 grid (res - 1 a multiple of the block), the thin plate needing growth rounds, one head without a
    surface; with the quirk, period 33^2 * 8 + 1 puts quirk voxels on block faces."""
    vols, h = _heads_volumes(33)
    bands, stats = _check(vols, 4, _tau(h), slots=4096, quirk_period=33 * 33 * 8 + 1 if quirk else 0)
    rounds = [s['growth_rounds'] for s in stats]
    assert rounds[2] >= 2 and rounds[0] < rounds[2] and rounds[1] == 0
    assert bands.retries == 0


def test_small_pool_forces_retries_and_changes_nothing():
    """A pool of one brick per head: the allocating steps have to grow it, and every head's result is the same."""
    vols, h = _heads_volumes(35)                       # (res - 1) % block != 0: partial blocks at the far faces
    big, st_big = _check(vols, 4, _tau(h), slots=1 << 20, quirk_period=35 ** 3 // 7)
    small, st_small = _check(vols, 4, _tau(h), slots=1, quirk_period=35 ** 3 // 7)
    assert small.retries >= 2 and big.retries == 0
    assert st_small == st_big
    assert small.slots >= max(len(hd.sblock) for hd in small.heads)


def test_one_head_equals_the_single_sparse_band():
    """S = 1 of the heads oracle against OracleSparseSlab driven by the single-band driver: the same states, values and mesh."""
    from nphm_b200.utils.reconstruction import LocalExchange, narrowband_slab_volumes
    vols, h = _heads_volumes(29)
    dense = vols[2]
    tau = _tau(h)
    bands, stats = _run([dense], 4, tau, slots=8)
    single = OracleSparseSlab(29, 4, 0, bands.blocks_per_axis)
    flat = dense.reshape(-1)
    ev = lambda idx: torch.from_numpy(flat[idx.numpy()])            # noqa: E731
    _, st = narrowband_slab_volumes([single], ev, None, None, tau, LocalExchange(1))
    assert np.array_equal(single.block_states().numpy(), bands.block_states()[0].numpy())
    assert np.array_equal(single.dense_volume().numpy(), bands.heads[0].dense_volume().numpy())
    assert st['voxels_evaluated'] == [stats[0]['voxels_evaluated']] and st['growth_rounds'] == stats[0]['growth_rounds']
    v1, t1 = brick_marching_cubes(single)
    v2, t2, _ = bands.marching_cubes(bands)
    assert np.array_equal(v1, v2) and np.array_equal(t1, t2)
