"""Writes tests/golden/ensemble_zero_skip.npz: sha256 of the outputs of the dense tensor-core ensemble kernel on queries where
many members have exactly zero blend weight on whole tiles, the bit-identity contract of tests/test_gpu_ensemble_zero_skip.py.
Skipping those members, and the compact grid tiles that find them, must not change a single bit.

    NPHM_B200_LIB=<build>/libnphm_b200.so python tests/golden/make_golden_ensemble_zero_skip.py [--check]

Cases: the 64^3 and 128^3 grids over the benchmark bounds for three latents, a 64^3 grid over [-1.5, 1.5]^3 (most
member-tiles skipped, some tiles keep only the global member), a range that starts and ends inside x-planes (linear tiles),
an x-slab of 32 planes with a ghost plane on each side, and a three-query xyz call with far points.  Every case runs twice
and must be identical between the two runs.  --check compares the build against the stored file instead of writing it.
The stored file was written by the build of commit cc20eb4 (the kernel before the zero-weight skip) on an H100."""
import hashlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
OUT = os.path.join(HERE, 'ensemble_zero_skip.npz')
WIDE_MIN, WIDE_MAX = [-1.5, -1.5, -1.5], [1.5, 1.5, 1.5]
CHUNK = 25000


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def engine(dev):
    from conftest import make_ensemble, sample_latent
    from nphm_b200 import _native
    dec = make_ensemble(0, device=dev).eval()
    eng = _native.EnsembleEngine(dec)
    eng.refresh(dec)
    lat = torch.stack([sample_latent(s).reshape(-1) for s in (1, 2, 3)]).to(dev)
    return eng, lat


def run_cases(dev):
    """name -> numpy array, for every case."""
    from conftest import MAXI, MINI
    eng, lat = engine(dev)
    out = {}

    def grid(i, mini, maxi, res, first, count):
        return eng.query_grid(lat[i], mini, maxi, res, first, count, CHUNK, impl='tc')[0].cpu().numpy()

    for res in (64, 128):
        for i in range(3):
            out['grid%d_latent%d' % (res, i + 1)] = grid(i, MINI, MAXI, res, 0, res ** 3)
    out['wide64'] = grid(0, WIDE_MIN, WIDE_MAX, 64, 0, 64 ** 3)
    out['unaligned64'] = grid(1, MINI, MAXI, 64, 12345, 25000)
    out['slab128'] = grid(2, MINI, MAXI, 128, 47 * 128 ** 2, 34 * 128 ** 2)
    g = torch.Generator().manual_seed(17)
    xyz = (torch.randn(3, 3000, 3, generator=g) * 0.6).to(dev)
    out['xyz_far'] = eng.query(xyz, lat, eval_quirk=False, impl='tc')[0].cpu().numpy()
    return out


def main():
    dev = torch.device('cuda', 0)
    a = run_cases(dev)
    b = run_cases(dev)
    varying = sorted(k for k in a if not np.array_equal(a[k], b[k]))
    assert not varying, 'outputs differ between two runs of the same build: %s' % varying
    if '--check' in sys.argv:
        ref = np.load(OUT)
        bad = [k for k in a if not matches(ref, k, a[k])]
        print('mismatch: %s' % bad if bad else 'all %d outputs match %s' % (len(a), OUT))
        sys.exit(1 if bad else 0)
    store = {}
    for k, v in a.items():
        store[k + '.sha256'] = np.array(sha(v))
        store[k + '.shape'] = np.array(v.shape, dtype=np.int64)
    np.savez_compressed(OUT, **store)
    print('wrote %s (%d bytes)' % (OUT, os.path.getsize(OUT)))


def matches(ref, k, v):
    return tuple(ref[k + '.shape']) == v.shape and str(ref[k + '.sha256']) == sha(v)


if __name__ == '__main__':
    main()
