"""Writes tests/golden/ensemble_pipeline.npz: outputs of the tensor-core ensemble kernel on a fixed set of cases, the
bit-identity contract of tests/test_gpu_ensemble_pipeline.py (a rescheduled kernel must reproduce every bit).

    NPHM_B200_LIB=<build>/libnphm_b200.so python tests/golden/make_golden_ensemble_pipeline.py [--check]

Small arrays are stored as they are, large ones as sha256 of their bytes.  The loss terms and gradients of the fitting call
are sums the fitting backward forms with atomics, so their last bits vary from run to run: they are listed in
`nondeterministic`, stored as values and compared with a tolerance.  Every case runs twice, and every other output must be
identical between the two runs.  --check compares the build against the stored file instead of writing it.
The stored file was written by the build of commit 310dbb2 (the kernel before the 4-slot weight ring) on an H100."""
import hashlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
OUT = os.path.join(HERE, 'ensemble_pipeline.npz')
EXACT_MAX = 4096          # arrays with more elements are stored as sha256
PRUNE_TAU = 1e-8
ATOMIC_SUMS = ('fit_loss_terms', 'fit_grad_latent', 'fit_grad_points')


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def run_cases(dev):
    """name -> numpy array, for every case."""
    from conftest import MAXI, MINI, make_ensemble, sample_latent
    from nphm_b200 import _native
    dec = make_ensemble(0, device=dev).eval()
    eng = _native.EnsembleEngine(dec)
    eng.refresh(dec)
    lat = torch.stack([sample_latent(s) for s in (1, 2, 3)]).to(dev)
    g = torch.Generator().manual_seed(11)
    out = {}

    def pts(n, b=1):
        return (torch.randn(b, n, 3, generator=g) * 0.25).to(dev)

    for name, n in (('one_tile', 128), ('three_tiles', 384), ('ragged', 300)):
        out[name] = eng.query(pts(n), lat[:1], eval_quirk=False, impl='tc')[0].cpu().numpy()
    out['three_latents'] = eng.query(pts(200, 3), lat, eval_quirk=False, impl='tc')[0].cpu().numpy()
    res, first = 64, 12345
    out['grid64_quirk'] = eng.query_grid(lat[0], MINI, MAXI, res, first, res ** 3 - first - 1000, 25000,
                                         impl='tc')[0].cpu().numpy()
    eng.set_prune_threshold(PRUNE_TAU)
    out['grid64_pruned'] = eng.query_grid(lat[1], MINI, MAXI, res, 0, res ** 3, 0, impl='tc_pruned')[0].cpu().numpy()

    # fitting surface gradient: the activation-dump variant, members split over CTAs, per-member outputs (members_out)
    lib = _native.lib()
    dec_t = make_ensemble(0, device=dev).train()
    eng_t = dec_t.engine()
    n = 1000
    p = pts(n)[0].contiguous()
    mask = (torch.rand(n, generator=g) > 0.2).to(torch.uint8).to(dev)
    z = lat[2].contiguous()
    ws = torch.zeros(lib.nphm_fit_batch_workspace_bytes(eng_t.handle, 1, n), dtype=torch.uint8, device=dev)
    terms = torch.zeros(8, device=dev)
    gl = torch.empty(dec_t.lat_dim, device=dev)
    gp = torch.empty_like(p)
    stream = torch.cuda.current_stream(dev).cuda_stream
    _native.check(lib.nphm_fit_surface_grad(eng_t.handle, p.data_ptr(), n, z.data_ptr(), mask.data_ptr(), 0.1,
                                            terms.data_ptr(), gl.data_ptr(), gp.data_ptr(), ws.data_ptr(), stream))
    torch.cuda.synchronize()
    members = 40
    w = ws.view(torch.float32)
    out['fit_member_s'] = w[:n * members].cpu().numpy()        # members_out: first block of the fitting workspace
    out['fit_loss_terms'] = terms[:6].cpu().numpy()            # the call writes entries 0-5 (loss .. kept count) only
    out['fit_grad_latent'] = gl.cpu().numpy()
    out['fit_grad_points'] = gp.cpu().numpy()
    return out


def main():
    dev = torch.device('cuda', 0)
    a = run_cases(dev)
    b = run_cases(dev)
    varying = sorted(k for k in a if k not in ATOMIC_SUMS and not np.array_equal(a[k], b[k]))
    assert not varying, 'outputs differ between two runs of the same build: %s' % varying
    nondet = list(ATOMIC_SUMS)
    if '--check' in sys.argv:
        ref = np.load(OUT)
        bad = [k for k in a if not matches(ref, k, a[k])]
        print('mismatch: %s' % bad if bad else 'all %d outputs match %s' % (len(a), OUT))
        sys.exit(1 if bad else 0)
    store = {'nondeterministic': np.array(nondet, dtype='U32')}
    for k, v in a.items():
        if v.size > EXACT_MAX and k not in nondet:
            store[k + '.sha256'] = np.array(sha(v))
            store[k + '.shape'] = np.array(v.shape, dtype=np.int64)
        else:
            store[k] = v
    np.savez_compressed(OUT, **store)
    print('wrote %s (%d bytes); nondeterministic: %s' % (OUT, os.path.getsize(OUT), nondet))


def matches(ref, k, v):
    if k + '.sha256' in ref.files:
        return tuple(ref[k + '.shape']) == v.shape and str(ref[k + '.sha256']) == sha(v)
    if k in set(ref['nondeterministic'].tolist()):
        return np.allclose(v, ref[k], rtol=1e-5, atol=1e-7 * max(1.0, float(np.abs(ref[k]).max())))
    return np.array_equal(v, ref[k])


if __name__ == '__main__':
    main()
