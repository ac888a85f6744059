"""Numpy restatement of the narrow-band extraction (``csrc/narrowband.cu``, ``utils/reconstruction.py:narrowband_volume``,
DESIGN §4.13) on a volume whose values are all known: "evaluating" a voxel copies its dense value.

The marching-cubes test runs on -sdf at 0, so a voxel is inside when ``v >= 0`` (NaN: outside).  Blocks of ``block^3`` cells;
block b covers the voxels [b*block, min(b*block + block, res - 1)] of every axis.
"""
from __future__ import annotations

import numpy as np


def _side(v):
    return v >= 0


def band_volume(dense: np.ndarray, block: int = 4, tau: float = 0.0, quirk_period: int = 0):
    """-> dict(volume: the filled float32 volume, evaluated: bool mask, active: bool block states, growth_rounds, voxels_evaluated).
    ``dense``: (res, res, res) float32."""
    dense = np.asarray(dense, dtype=np.float32)
    res = dense.shape[0]
    C, B = res - 1, int(block)
    nb = -(-C // B)
    tau = np.float32(tau)
    lo = np.arange(nb) * B
    hi = np.minimum(lo + B, C)
    ev = np.zeros(dense.shape, bool)
    active = np.zeros((nb, nb, nb), bool)
    if quirk_period:
        g = np.union1d(np.arange(quirk_period - 1, res ** 3, quirk_period), [res ** 3 - 1])
        ev.reshape(-1)[g] = True
        for x, y, z in zip(*np.unravel_index(g, dense.shape)):
            rng = [range(max(c - 1, 0) // B, min(c, C - 1) // B + 1) for c in (x, y, z)]
            for bx in rng[0]:
                for by in rng[1]:
                    for bz in rng[2]:
                        active[bx, by, bz] = True
    # coarse pass: block corners
    ci = np.minimum(np.arange(nb + 1) * B, C)
    ev[np.ix_(ci, ci, ci)] = True
    cv = dense[np.ix_(ci, ci, ci)]
    corners = [cv[dx:dx + nb, dy:dy + nb, dz:dz + nb] for dx in (0, 1) for dy in (0, 1) for dz in (0, 1)]
    near = np.any([~(np.abs(c) > tau) for c in corners], axis=0)
    n_in = np.sum([_side(c) for c in corners], axis=0)
    active |= near | ((n_in != 0) & (n_in != 8))

    def mark(blocks):
        for bx, by, bz in zip(*np.nonzero(blocks)):
            ev[lo[bx]:hi[bx] + 1, lo[by]:hi[by] + 1, lo[bz]:hi[bz] + 1] = True

    mark(active)
    rounds = 0
    while True:
        grown = np.zeros_like(active)
        for bx, by, bz in zip(*np.nonzero(~active)):
            box = (slice(lo[bx], hi[bx] + 1), slice(lo[by], hi[by] + 1), slice(lo[bz], hi[bz] + 1))
            s0 = _side(dense[lo[bx], lo[by], lo[bz]])
            if np.any(ev[box] & (_side(dense[box]) != s0)):
                grown[bx, by, bz] = True
        before = int(ev.sum())
        active |= grown
        mark(grown)
        if int(ev.sum()) == before:
            break
        rounds += 1
    fi = np.minimum(np.arange(res) // B, nb - 1) * B
    volume = np.where(ev, dense, dense[np.ix_(fi, fi, fi)]).astype(np.float32)
    return {'volume': volume, 'evaluated': ev, 'active': active, 'growth_rounds': rounds, 'voxels_evaluated': int(ev.sum())}
