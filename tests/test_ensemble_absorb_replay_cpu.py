"""The replay of the dense ensemble kernel's per-point absorption decisions (tools/absorbed_member_tiles.py replay, DESIGN
4.1) and the inputs the GPU replay test gives it, checked against exact rational arithmetic: the emulated fmaf and the
latent fold of the layer constants, the replay's verdicts point by point, that every member it skips changes no bit of the
fp32 blend, the borderline classification around the rule's threshold, and that the kernel's decisions drive its state."""
import os
import sys
from fractions import Fraction

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import absorbed_member_tiles as A  # noqa: E402
from test_ensemble_absorb_cpu import exact_fma_unchanged, round_f32  # noqa: E402

f32 = np.float32
F = lambda v: Fraction(float(v))        # noqa: E731


def exact_fma(a, b, c):
    return f32(float(round_f32(F(a) * F(b) + F(c))))


def test_fmaf32_is_correctly_rounded():
    rng = np.random.default_rng(5)
    a = (rng.standard_normal(4000) * 10.0 ** rng.integers(-8, 8, 4000)).astype(f32)
    b = (rng.standard_normal(4000) * 10.0 ** rng.integers(-8, 8, 4000)).astype(f32)
    c = (rng.standard_normal(4000) * 10.0 ** rng.integers(-8, 8, 4000)).astype(f32)
    # halfway cases of the float64 sum: c = -a b rounded, plus products whose low half is a tie
    c[:500] = (-(a[:500].astype(np.float64) * b[:500])).astype(f32)
    a[500:600], b[500:600], c[500:600] = f32(1 + 2 ** -12), f32(1 + 2 ** -12), f32(2 ** -48)
    got = A.fmaf32(a, b, c)
    for i in range(a.size):
        assert got[i] == exact_fma(a[i], b[i], c[i]), (a[i], b[i], c[i])


def test_fold_consts_matches_the_warp_order():
    """fold_consts against a scalar restatement of cvec_kernel with exactly rounded fmaf and fp32 adds."""
    from conftest import make_ensemble, sample_latent
    from ensemble_f64_common import Params
    P = Params(make_ensemble(0).eval(), torch.float32)
    z = sample_latent(2).reshape(-1)
    for m in (0, 1, 39):
        got = A.fold_consts(P, z, m)
        s_ = P.weight_set(m)
        zz = z.numpy()
        u = np.concatenate([zz[:P.G], zz[P.G + m * P.L:P.G + (m + 1) * P.L]]).astype(f32)
        for l in (0, 2):
            W, b = P.layers[l][0][s_].numpy(), P.layers[l][1][s_].numpy()
            Wc = W[:, W.shape[1] - u.size:]
            for n in (0, 7, W.shape[0] - 1):
                lanes = [f32(0.0)] * 32
                for j in range(u.size):
                    lanes[j % 32] = exact_fma(Wc[n, j], u[j], lanes[j % 32])
                for o in (16, 8, 4, 2, 1):
                    lanes = [f32(lanes[i] + lanes[i ^ o]) for i in range(32)]
                scale = f32(1.0) if l == 0 else f32(1.0 / np.sqrt(2.0))
                assert got[l][n] == exact_fma(lanes[0], scale, b[n]), (m, l, n)
        assert np.array_equal(got[1], P.layers[1][1][s_].numpy())


def scalar_pass(w, B, pub, lag):
    """The rule at one valid point in exact arithmetic: L = round_down(pub - lag), w B rounded up < ulp(L) / 4."""
    if w == 0:
        return True
    d = F(pub) - F(lag)
    L = round_f32(d)
    if L > d:
        L = F(np.nextafter(f32(float(L)), f32(-np.inf)))
    if L < Fraction(2) ** -100:
        return False
    wb = round_f32(F(w) * F(B))
    if wb < F(w) * F(B):
        wb = F(np.nextafter(f32(float(wb)), f32(np.inf)))
    e = int(np.floor(np.log2(float(L))))
    return wb < Fraction(2) ** (e - 25)


def tiles(seed, T=8, M=7):
    """Random tiles whose weights span the absorption threshold: members 0 and 1 (never candidates) weigh 0.5, every later
    member's weights span three decades somewhere between 1e-16 and 1e-6 per tile, s within +-B."""
    rng = np.random.default_rng(seed)
    lo = rng.uniform(-16, -9, (T, 1, M))
    W = (10.0 ** (lo + rng.uniform(0, 3, (T, 128, M)))).astype(f32)
    W[:, :, :2] = f32(0.5)
    W[rng.random((T, 128, M)) < 0.1] = f32(0.0)
    B = f32(10.0 ** rng.uniform(0, 0.5, M))
    S = (B[None, None, :] * rng.uniform(-1, 1, (T, 128, M))).astype(f32)
    V = rng.random((T, 128)) < 0.95
    mask = np.ones((T, M), bool)
    mask[:, 3] = rng.random(T) < 0.5
    amask = mask & (rng.random((T, M)) < 0.9)
    return W, S, V, mask, amask, B


def torch_args(W, S, V, mask, amask, B):
    return [torch.from_numpy(np.ascontiguousarray(a)) for a in (W, S, V, mask, amask, B)]


def test_replay_matches_the_exact_rule_and_skips_only_absorbed_members():
    n_skip = 0
    for seed in range(4):
        W, S, V, mask, amask, B = tiles(seed)
        r = A.replay(*torch_args(W, S, V, mask, amask, B))
        skip = r['skip'].numpy()
        T, _, M = W.shape
        for t in range(T):
            num = [f32(0.0)] * 128
            pp = [[f32(0.0)] * 128, [f32(0.0)] * 128]
            lag = [f32(0.0)] * 128
            npos = 0
            for k in range(M):
                if not mask[t, k]:
                    continue
                cand = amask[t, k] and npos >= 2
                verdict = cand and all(not V[t, i] or scalar_pass(W[t, i, k], B[k], pp[0][i], lag[i]) for i in range(128))
                assert verdict == skip[t, k], (seed, t, k)
                if verdict:
                    n_skip += 1
                    assert all(not V[t, i] or exact_fma_unchanged(W[t, i, k], S[t, i, k], num[i]) for i in range(128))
                    continue
                num = [exact_fma(W[t, i, k], S[t, i, k], num[i]) for i in range(128)]
                pp = [pp[1], [abs(v) for v in num]]
                lag = [A.fmul_ru(W[t, i, k], B[k]) for i in range(128)]
                npos += 1
    assert n_skip > 10                  # not vacuous


def test_borderline_classification():
    """One point per tile decides: w B at, just under and far under ulp(L) / 4 of |num| = 1.  With num known to within its
    rounding (no s error), a margin of 2^-10 relative is sure, 2^-30 is borderline; far over the threshold is a sure keep."""
    T, M = 4, 3
    W = np.zeros((T, 128, M), f32)
    S = np.zeros((T, 128, M), f32)
    W[:, 0, 0], S[:, 0, 0] = f32(1.0), f32(1.0)            # num = 1 after member 0
    W[:, 0, 1], S[:, 0, 1] = f32(2.0 ** -40), f32(0.0)     # member 1 adds 0: num stays 1, lag = 2^-40
    thr = 2.0 ** -26                                       # ulp(L) / 4 for L = 1 - 2^-24 (1 minus the lag, rounded down)
    for t, w in enumerate((thr * (1 - 2 ** -10), thr * (1 - 2 ** -23), thr * 8, thr * 2 ** -20)):
        W[t, 0, 2] = f32(w)
    V = np.zeros((T, 128), bool)
    V[:, 0] = True
    mask = np.ones((T, M), bool)
    B = np.ones(M, f32)
    r = A.replay(*torch_args(W, S, V, mask, mask, B))
    skip, sure_skip, sure_keep = (r[k][:, 2].tolist() for k in ('skip', 'sure_skip', 'sure_keep'))
    assert skip == [True, True, False, True]
    assert sure_skip == [True, False, False, True]
    assert sure_keep == [False, False, True, False]
    assert r['margin'][1, 2] < 2 ** -20 < r['margin'][0, 2]


def test_follow_drives_the_state():
    """With follow, the kernel's skips (not the replay's verdicts) decide which members enter num and the lag."""
    W, S, V, mask, amask, B = tiles(11)
    args = torch_args(W, S, V, mask, amask, B)
    own = A.replay(*args)
    same = A.replay(*args, follow=own['skip'])
    for k in ('skip', 'sure_skip', 'sure_keep'):
        assert torch.equal(own[k], same[k])
    none = A.replay(*args, follow=torch.zeros_like(own['skip']))    # a kernel that skips nothing
    assert torch.equal(none['cand'], args[3] & args[4] & (torch.cumsum(args[3].long(), 1) - args[3].long() >= 2))
