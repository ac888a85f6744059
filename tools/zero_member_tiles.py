#!/usr/bin/env python
"""How many member-tiles of a dense grid query the ensemble kernel skips, predicted on the CPU.

The dense ensemble kernel skips member k on a tile of 128 grid points when its blend weight exp(-(|x - a_k| + 1e-5)^2 / 0.01)
is exactly +0 in fp32 at every valid point of the tile (DESIGN 4.1).  This tool evaluates that formula in numpy float32 for
the anchors of the seeded head of bench.py and counts, over the tiles of a grid query, the (tile, member) pairs whose weights
are all zero.  The weight is monotone in each coordinate distance, so a tile's largest weight is the one at its smallest
squared distance.  fp32 rounding (fused multiply-adds, expf) can differ from the GPU's at the underflow edge, so the count is
a prediction: the -DNPHM_ENS_TRACE build (tools/ens_trace.py) measures the member-tiles the kernel evaluated.

    python tools/zero_member_tiles.py [--latent 1] [--res 256] [--tile auto|linear|XxYxZ] [--first F --count N]
                                      [--mini X Y Z --maxi X Y Z]

--tile auto picks the tiles the kernel picks for the dense path: 1 x 16 x 8 blocks, or 128 consecutive points where blocks
would add more than 3 % tiles."""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

DENSE_BLOCK = (1, 16, 8)


def parse_args(argv=None):
    from conftest import MAXI, MINI
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--latent', type=int, default=1, help='seed of sample_latent (bench.py uses 1)')
    ap.add_argument('--res', type=int, default=256)
    ap.add_argument('--tile', default='auto', help="auto, linear or a block shape XxYxZ with X*Y*Z = 128")
    ap.add_argument('--first', type=int, default=0)
    ap.add_argument('--count', type=int, default=-1, help='points of the query (default: the rest of the grid)')
    ap.add_argument('--mini', type=float, nargs=3, default=MINI)
    ap.add_argument('--maxi', type=float, nargs=3, default=MAXI)
    return ap.parse_args(argv)


def anchors_of(latent_seed):
    """(39, 3) float32 anchors of the seeded head (make_ensemble(0)) for sample_latent(latent_seed)."""
    import torch
    from conftest import make_ensemble, sample_latent
    dec = make_ensemble(0).eval()
    with torch.no_grad():
        a = dec.predict_anchors(sample_latent(latent_seed).reshape(1, 1, -1))
    return a[0].numpy().astype(np.float32)


def tile_layout(res, first, count, tile):
    """(kind, block) as the kernel chooses it: ('linear', None) or ('blocked', (tbx, tby, tbz))."""
    if tile == 'linear':
        return 'linear', None
    if tile == 'auto':
        block = DENSE_BLOCK
    else:
        block = tuple(int(v) for v in tile.split('x'))
        assert len(block) == 3 and np.prod(block) == 128, 'a block has 128 points'
    tbx, tby, tbz = block
    rr = res * res
    px0, px1 = first // rr, (first + count - 1) // rr
    blocked = ((px1 - px0 + tbx) // tbx) * ((res + tby - 1) // tby) * ((res + tbz - 1) // tbz)
    if tile == 'auto' and blocked * 100 > -(-count // 128) * 103:
        return 'linear', None
    return 'blocked', block


def tile_points(res, first, count, kind, block):
    """(ix, iy, iz, valid), each (tiles, 128): the grid point of every row of every tile, in the kernel's order."""
    rows = np.arange(128, dtype=np.int64)
    if kind == 'linear':
        n_tiles = -(-count // 128)
        idx = np.arange(n_tiles, dtype=np.int64)[:, None] * 128 + rows[None]
        valid = idx < count
        g = first + np.where(valid, idx, 0)
        return g // (res * res), (g // res) % res, g % res, valid
    tbx, tby, tbz = block
    rr = res * res
    px0, px1 = first // rr, (first + count - 1) // rr
    by, bz = (res + tby - 1) // tby, (res + tbz - 1) // tbz
    n_tiles = ((px1 - px0 + tbx) // tbx) * by * bz
    t = np.arange(n_tiles, dtype=np.int64)[:, None]
    tz, txy = t % bz, t // bz
    ty, tx = txy % by, txy // by
    ix = px0 + tx * tbx + rows[None] // (tby * tbz)
    iy = ty * tby + (rows[None] // tbz) % tby
    iz = tz * tbz + rows[None] % tbz
    g = (ix * res + iy) * res + iz
    valid = (ix <= px1) & (iy < res) & (iz < res) & (g >= first) & (g < first + count)
    return np.minimum(ix, res - 1), np.minimum(iy, res - 1), np.minimum(iz, res - 1), valid


def zero_member_tiles(anchors, mini, maxi, res, first=0, count=-1, tile='auto'):
    """dict: layout, tiles, member-tiles (40 per tile), zero member-tiles, evaluated member-tiles."""
    if count < 0:
        count = res ** 3 - first
    kind, block = tile_layout(res, first, count, tile)
    ix, iy, iz, valid = tile_points(res, first, count, kind, block)
    axes = [np.linspace(mini[a], maxi[a], res).astype(np.float32) for a in range(3)]
    n_tiles, n_members = ix.shape[0], anchors.shape[0] + 1
    zero = 0
    with np.errstate(under='ignore'):
        for a in anchors:
            sq = [np.square(a[d] - axes[d]) for d in range(3)]            # float32 (a - x)^2 per axis
            d2 = sq[0][ix] + sq[1][iy] + sq[2][iz]
            d2 = np.where(valid, d2, np.float32(np.inf)).min(axis=1)     # the tile's nearest valid point
            nrm = np.sqrt(d2) + np.float32(10e-6)
            w = np.exp(-(nrm * nrm) / np.float32(0.01))
            zero += int(np.count_nonzero(w == 0))
    total = n_tiles * n_members
    return {'layout': kind if kind == 'linear' else 'x'.join(map(str, block)), 'tiles': int(n_tiles),
            'member_tiles': int(total), 'zero_member_tiles': zero, 'evaluated_member_tiles': int(total - zero),
            'zero_share': zero / total}


def main():
    args = parse_args()
    r = zero_member_tiles(anchors_of(args.latent), args.mini, args.maxi, args.res, args.first, args.count, args.tile)
    print('latent %d, %d^3 grid, points [%d, +%s), %s tiles: %d tiles, %d member-tiles, %d with all weights zero (%.1f %%), '
          '%d evaluated' % (args.latent, args.res, args.first, args.count if args.count >= 0 else 'rest', r['layout'],
                            r['tiles'], r['member_tiles'], r['zero_member_tiles'], 100 * r['zero_share'],
                            r['evaluated_member_tiles']))


if __name__ == '__main__':
    main()
