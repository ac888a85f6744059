#!/usr/bin/env python
"""Timeline of one CTA of the dense ensemble kernel (build with -DNPHM_ENS_TRACE: tools/build_variant.sh): runs one grid query
of the seeded head of bench.py and prints, for four consecutive members of CTA 0, when each consumer warpgroup waited for its
weights, issued and retired its MMAs and finished its epilogues, when the producer issued each weight unit, and per member:
cycles waiting for weights, cycles in which neither warpgroup had MMAs in flight, epilogue cycles.  Then, per tile of CTA 0,
when warpgroup 0 took it from the producer's queue, when the producer knew its member mask (before that, when negative) and
when the first member's layer-1 weights were ready; over all CTAs the member-tiles the kernel evaluated (to set against
tools/zero_member_tiles.py and tools/absorbed_member_tiles.py), the cycles per evaluated member-tile, the spread of
member-tiles and cycles per CTA, and the producer's cycles per tile from an absorption candidate's first wait to its decision.

    bash tools/build_variant.sh /tmp/ens -DNPHM_ENS_TRACE && NPHM_B200_LIB=/tmp/ens/libnphm_b200.so python tools/ens_trace.py [res]"""
import ctypes, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np
import torch

# layout of g_ens_trace, g_ens_tiles and g_ens_ctas (csrc/tc_ensemble_wgmma.cu)
MEMBERS, WG, STRIDE = 4, 32, 2 * 32 + 16
TILES, MAX_CTAS, CTA_WORDS = 4, 1024, 5
PHASES = ['L1', 'L2', 'L3a', 'L3b']
EVENTS = ['wait', 'ready', 'turn', 'issued', 'retired', 'epi']


def union_length(intervals):
    total, end = 0, None
    for a, b in sorted(intervals):
        if end is None or a > end:
            total += b - a
            end = b
        elif b > end:
            total += b - end
            end = b
    return total


def main():
    from conftest import MAXI, MINI, make_ensemble, sample_latent
    from nphm_b200 import _native
    res = int(sys.argv[1]) if len(sys.argv) > 1 else 64
    dev = torch.device('cuda', 0)
    dec = make_ensemble(0, device=dev).eval()
    eng = _native.EnsembleEngine(dec)
    eng.refresh(dec)
    lat = sample_latent(1).to(dev)
    n = res ** 3
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    eng.query_grid(lat, MINI, MAXI, res, 0, n, 25000, impl='tc')
    ev0.record()
    eng.query_grid(lat, MINI, MAXI, res, 0, n, 25000, impl='tc')
    ev1.record(); torch.cuda.synchronize()
    print('grid query %d^3: %.2f ms' % (res, ev0.elapsed_time(ev1)))
    lib = _native.lib()
    if not hasattr(lib, 'nphm_debug_ens_trace'):
        print('not a -DNPHM_ENS_TRACE build: no timeline')
        return
    buf = (ctypes.c_longlong * (1 + MEMBERS * STRIDE))()
    _native.check(lib.nphm_debug_ens_trace(buf, len(buf)), 'nphm_debug_ens_trace')
    t = np.array(buf[:], dtype=np.int64)
    t0 = t[0]
    rec = t[1:].reshape(MEMBERS, STRIDE)
    print('cycles from CTA start; consumer events per phase: ' + ' / '.join(EVENTS))
    totals = []
    for mi in range(MEMBERS):
        r = rec[mi] - t0
        print('member %d' % mi)
        prod = r[2 * WG:2 * WG + 16]
        print('  producer  unit issued: ' + ' '.join('%8d' % prod[u] for u in range(8) if rec[mi, 2 * WG + u]))
        print('            slot wait:   ' + ' '.join('%8d' % prod[8 + u] for u in range(8) if rec[mi, 2 * WG + 8 + u]))
        mma, wait, epi = [], 0, 0
        for w in range(2):
            c = r[w * WG:(w + 1) * WG]
            print('  wg%d start %8d  layer 0 done %8d' % (w, c[24], c[25]))
            epi += c[25] - c[24]
            for p, name in enumerate(PHASES):
                e = c[6 * p:6 * p + 6]
                print('    %-4s ' % name + ' '.join('%8d' % v for v in e))
                wait += e[1] - e[0]
                mma.append((e[2], e[4]))
                epi += e[5] - e[4]
        span = max(r[w * WG + 23] for w in range(2)) - min(r[w * WG + 24] for w in range(2))
        idle = span - union_length(mma)
        totals.append((span, wait, idle, epi))
        print('  span %d cycles: weight waits %d (both warpgroups), no MMA in flight %d, epilogues %d (both warpgroups)'
              % (span, wait, idle, epi))
    tt = np.array(totals, dtype=np.float64).mean(axis=0)
    print('mean per member: span %.0f, weight waits %.0f, no MMA in flight %.0f, epilogues %.0f' % tuple(tt))
    if not hasattr(lib, 'nphm_debug_ens_work'):
        return
    buf = (ctypes.c_longlong * (3 * TILES + 1 + CTA_WORDS * MAX_CTAS))()
    _native.check(lib.nphm_debug_ens_work(buf, len(buf)), 'nphm_debug_ens_work')
    w = np.array(buf[:], dtype=np.int64)
    tiles = w[:3 * TILES].reshape(TILES, 3) - t0
    for i in range(TILES):
        length = ' (%d cycles to the next tile)' % (tiles[i + 1, 0] - tiles[i, 0]) if i + 1 < TILES else ''
        print('tile %d of CTA 0: taken from the queue at %d, mask known to the producer %+d, first member\'s layer-1 '
              'weights ready %+d%s' % (i, tiles[i, 0], tiles[i, 1] - tiles[i, 0], tiles[i, 2] - tiles[i, 0], length))
    n_ctas = int(w[3 * TILES])
    ctas = w[3 * TILES + 1:3 * TILES + 1 + CTA_WORDS * n_ctas].reshape(n_ctas, CTA_WORDS)
    mt, cyc = int(ctas[:, 0].sum()), int(ctas[:, 1].sum())
    print('all %d CTAs: %d member-tiles evaluated, %.0f cycles per evaluated member-tile (CTA cycles summed / member-tiles)'
          % (n_ctas, mt, cyc / max(mt, 1)))
    for col, name in ((0, 'member-tiles'), (1, 'cycles')):
        v = ctas[:, col].astype(np.float64)
        print('per CTA %s: min %.0f, mean %.0f, max %.0f, max / mean %.4f' % (name, v.min(), v.mean(), v.max(), v.max() / v.mean()))
    # the producer's absorption decisions: from a candidate's first wait for the consumers' |num| to the warp's vote
    tiles, decide, wait = int(ctas[:, 2].sum()), int(ctas[:, 3].sum()), int(ctas[:, 4].sum())
    print('producer absorption decisions: %.0f cycles per tile (%.0f of them waiting for |num|), %.2f %% of the CTA cycles'
          % (decide / max(tiles, 1), wait / max(tiles, 1), 100.0 * decide / max(cyc, 1)))


if __name__ == '__main__':
    main()
