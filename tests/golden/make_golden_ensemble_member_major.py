"""Writes tests/golden/ensemble_member_major.npz: per member, the (point, member) pairs a dense grid query evaluates member by
member, as tools/absorbed_member_tiles.py predicts them on the CPU (key compact_pairs): the benchmark's head and latent,
quirk period 25 000, the 64^3 and 128^3 grids over the benchmark bounds.  tests/test_gpu_ensemble_member_major.py checks
that the member passes list exactly these counts.

    python tests/golden/make_golden_ensemble_member_major.py [--check]

About 6 CPU-minutes.  --check compares a fresh prediction with the stored file instead of writing it."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
OUT = os.path.join(HERE, 'ensemble_member_major.npz')
RESES = (64, 128)
QUIRK_PERIOD = 25000


def main():
    import absorbed_member_tiles as A
    got = {'pairs_%d' % res: A.predict(1, res, quirk_period=QUIRK_PERIOD)['compact_pairs'] for res in RESES}
    if '--check' in sys.argv:
        ref = np.load(OUT)
        for k, v in got.items():
            assert np.array_equal(ref[k], v), k
        print('ok')
        return
    np.savez(OUT, quirk_period=QUIRK_PERIOD, **got)
    for k, v in got.items():
        print('%s: %d pairs, %d compact tiles' % (k, v.sum(), ((v + 127) // 128).sum()))


if __name__ == '__main__':
    main()
