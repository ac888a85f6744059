"""The fp32 absorption certificate of tools/absorbed_member_tiles.py (DESIGN 4.1, 8): skipping member k is exact when
den + w == den in fp32 and w * B < ulp(L) / 4 with L <= |num| and B >= |s|, so that fmaf(w, s, num) returns num.  The
predicate is checked against exact rational arithmetic, the member-output bound B_k against the float64 reference, and the
predictor's counts against each other on a small grid."""
import os
import sys
from fractions import Fraction

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import absorbed_member_tiles as A  # noqa: E402


def round_f32(v):
    """Fraction -> the float32 round-to-nearest-even of it (as a Fraction), denormals included, no overflow."""
    if v == 0:
        return Fraction(0)
    sign, a = (1, v) if v > 0 else (-1, -v)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    q = Fraction(2) ** (max(e, -126) - 23)
    m = a / q
    lo = m.numerator // m.denominator
    rem = m - lo
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and lo % 2 == 1):
        lo += 1
    return sign * lo * q


def exact_fma_unchanged(w, s, num):
    return round_f32(Fraction(float(w)) * Fraction(float(s)) + Fraction(float(num))) == Fraction(float(num))


def exact_add_unchanged(den, w):
    return round_f32(Fraction(float(den)) + Fraction(float(w))) == Fraction(float(den))


def check(den, w, num, s):
    """The certificate with the exact |num| and |s| as bounds: if it passes, the exact fp32 updates change nothing."""
    den, w, num, s = (np.float32(v) for v in (den, w, num, s))
    ok = bool(A.absorbable(den, w, np.float64(abs(num)), np.float64(w), np.float64(abs(s))))
    if ok:
        assert exact_add_unchanged(den, w), (den, w)
        assert exact_fma_unchanged(w, s, num), (w, s, num)
        assert np.float32(den + w) == den
    return ok


def test_round_f32_matches_numpy():
    rng = np.random.default_rng(0)
    for _ in range(2000):
        x = rng.standard_normal() * 10.0 ** rng.integers(-45, 30)
        assert round_f32(Fraction(x)) == Fraction(float(np.float32(x)))


def test_certificate_random():
    rng = np.random.default_rng(1)
    passed = 0
    for _ in range(4000):
        den = np.float32(10.0 ** rng.uniform(-10, 1))
        num = np.float32(rng.standard_normal() * den * 10.0 ** rng.uniform(-3, 1))
        w = np.float32(den * 10.0 ** rng.uniform(-16, -5))
        s = np.float32(rng.standard_normal() * 10.0 ** rng.uniform(-2, 1))
        passed += check(den, w, num, s)
    assert passed > 400                 # not vacuous


def test_certificate_adversarial():
    f32 = np.float32
    cases = []
    for e in (-126, -100, -30, -1, 0, 1, 20):
        p = f32(2.0 ** e)
        u = float(np.spacing(p))                      # ulp(p): the spacing above a power of two
        for sgn_num in (1, -1):
            for sgn_s in (1, -1):
                # w * |s| just below, at and just above ulp / 4, toward and away from zero
                for ws in (u / 4 * (1 - 2 ** -20), u / 4, u / 4 * (1 + 2 ** -20), u / 2, u / 8):
                    w = f32(ws / 3.0)
                    if w == 0:
                        continue
                    s = f32(sgn_s * ws / float(w))
                    cases.append((f32(1.0), w, f32(sgn_num * p), s))
        # ties of round-to-nearest-even: num with an odd mantissa and w * s at exactly half the spacing
        q = f32(p * f32(1 + 2 ** -23))
        cases.append((f32(1.0), f32(2.0 ** -20), q, f32(u * 2 ** 19)))
    # den at powers of two and ties: den + w == den decided by the fp32 add
    for e in (-20, 0, 5):
        d = f32(2.0 ** e)
        for w in (np.spacing(d) / 2, np.spacing(d) / 4, np.spacing(d), np.spacing(d) * 0.49):
            cases.append((d, f32(w), f32(1.0), f32(1e-30)))
    # denormal weights and num, num = 0, den = 0
    tiny = np.float32(np.finfo(np.float32).tiny)
    for w in (f32(1e-45), f32(1e-40), tiny):
        cases += [(f32(1.0), w, f32(0.0), f32(1.0)), (f32(0.0), w, f32(1.0), f32(1.0)),
                  (f32(1.0), w, f32(1e-39), f32(1.0)), (f32(1.0), w, tiny, f32(1.0))]
    passed = [check(*c) for c in cases]
    assert any(passed) and not all(passed)
    # the strict inequality: w * |s| == ulp(|num|) / 4 is never certified
    assert not A.absorbable(f32(1.0), f32(2.0 ** -25), 1.0, 2.0 ** -25, 1.0)        # ulp(1) / 4 = 2^-25
    assert A.absorbable(f32(1.0), f32(2.0 ** -26), 1.0, 2.0 ** -26, 1.0)
    # num = 0 and a lower bound that is not positive: never certified
    assert not A.absorbable(f32(1.0), f32(1e-30), 0.0, 1e-30, 1.0)
    assert not A.absorbable(f32(1.0), f32(1e-30), -1.0, 1e-30, 1.0)
    # a bound that is not finite: never certified
    assert not A.absorbable(f32(1.0), f32(1e-30), 1.0, 1e-30, np.inf)


@pytest.mark.parametrize('scale', [1.0, 2.0])
@pytest.mark.parametrize('seed', [1, 2, 3])
def test_member_bound_covers_reference(seed, scale):
    from conftest import MAXI, MINI
    from ensemble_f64_common import members
    P32, P64, z, anc32 = A.grid_setup(seed, scale)
    anc = anc32.double()
    lo, hi = np.array(MINI, np.float64), np.array(MAXI, np.float64)
    rng = np.random.default_rng(seed)
    corners = np.array([[(hi if (c >> a) & 1 else lo)[a] for a in range(3)] for c in range(8)])
    pts = np.concatenate([corners, lo + (hi - lo) * rng.random((1500, 3))])
    # points near every anchor inside the box, where the member is sampled most densely by the blend
    near = anc.numpy()[rng.integers(0, anc.shape[0], 500)] + 0.05 * rng.standard_normal((500, 3))
    pts = np.concatenate([pts, np.clip(near, lo, hi)])
    with torch.no_grad():
        S = members(P64, torch.from_numpy(pts), z.double(), anc).numpy()
    for m in range(P64.M):
        B = A.member_bound(P64, m, z, anc.numpy(), lo, hi)
        assert np.isfinite(B) and B >= 1.0
        assert np.abs(S[:, m]).max() <= B, (m, np.abs(S[:, m]).max(), B)
    # a sub-box bound covers the outputs in it and is no looser than the whole box's
    sub_lo, sub_hi = lo + 0.3 * (hi - lo), lo + 0.4 * (hi - lo)
    sub = sub_lo + (sub_hi - sub_lo) * rng.random((300, 3))
    with torch.no_grad():
        Ssub = members(P64, torch.from_numpy(sub), z.double(), anc).numpy()
    for m in (0, 1, P64.M - 1):
        Bs = A.member_bound(P64, m, z, anc.numpy(), sub_lo, sub_hi)
        assert np.abs(Ssub[:, m]).max() <= Bs <= A.member_bound(P64, m, z, anc.numpy(), lo, hi)


def test_predictor_counts_are_consistent():
    r = A.predict(latent_seed=1, res=24)
    # every certified member changes no bit (asserted per tile inside predict); the weaker certificates skip less
    assert 0 < r['absorbed'] <= r['absorbed_no_lag'] <= r['absorbed_tile_max'] <= r['unchanged'] <= r['den_absorbed']
    assert r['evaluated_absorb'] + r['absorbed'] + r['zero'] == r['member_tiles']
