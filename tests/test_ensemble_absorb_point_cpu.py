"""The per-point absorption rule of the dense ensemble kernel (tools/absorbed_member_tiles.py point_pass, DESIGN 4.1): at a
valid point with w_m != +0, skipping member m is exact when w_m * B_m < ulp(L) / 4, L = |num| two evaluated positions back
minus w * B of the member in between, with the kernel's directed roundings.  Checked against exact rational arithmetic: the
member in between runs its fp32 fmaf, and then member m's fmaf must return num unchanged.  Also the predictor's counts."""
import os
import sys
from fractions import Fraction

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import absorbed_member_tiles as A  # noqa: E402
from test_ensemble_absorb_cpu import exact_fma_unchanged, round_f32  # noqa: E402

f32 = np.float32


def fma32(w, s, num):
    """fp32 fmaf(w, s, num), exactly rounded."""
    return f32(float(round_f32(Fraction(float(w)) * Fraction(float(s)) + Fraction(float(num)))))


def check(num2, w1, s1, B1, w, s, B):
    """The rule with |s1| <= B1 and |s| <= B: if it passes, member m leaves num = fmaf(w1, s1, num2) unchanged."""
    num2, w1, s1, B1, w, s, B = (f32(v) for v in (num2, w1, s1, B1, w, s, B))
    assert abs(s1) <= B1 and abs(s) <= B
    ok = bool(A.point_pass(w, B, abs(num2), A.fmul_ru(w1, B1), True))
    if ok:
        num1 = fma32(w1, s1, num2)
        assert exact_fma_unchanged(w, s, num1), (num2, w1, s1, B1, w, s, B)
    return ok


def test_directed_roundings_are_exact():
    rng = np.random.default_rng(3)
    for _ in range(3000):
        a = f32(rng.standard_normal() * 10.0 ** rng.integers(-23, 18))
        b = f32(rng.standard_normal() * 10.0 ** rng.integers(-23, 18))
        d = Fraction(float(a)) - Fraction(float(b))
        r = A.fsub_rd(a, b)
        assert Fraction(float(r)) <= d and Fraction(float(np.nextafter(r, f32(np.inf)))) > d, (a, b, r)
        p = Fraction(float(a)) * Fraction(float(b))
        q = A.fmul_ru(a, b)
        if np.isfinite(q):
            assert Fraction(float(q)) >= p and Fraction(float(np.nextafter(q, f32(-np.inf)))) < p, (a, b, q)


def test_point_rule_random():
    rng = np.random.default_rng(4)
    passed = 0
    for _ in range(3000):
        num2 = f32(rng.standard_normal() * 10.0 ** rng.uniform(-6, 1))
        B1, B = f32(10.0 ** rng.uniform(0, 1)), f32(10.0 ** rng.uniform(0, 1))
        s1, s = f32(B1 * rng.uniform(-1, 1)), f32(B * rng.uniform(-1, 1))
        w1 = f32(10.0 ** rng.uniform(-12, 0))
        w = f32(abs(num2) * 10.0 ** rng.uniform(-12, -5))
        passed += check(num2, w1, s1, B1, w, s, B)
    assert passed > 300                 # not vacuous


def test_point_rule_adversarial():
    cases = []
    for e in (-100, -99, -30, -1, 0, 1, 20):
        p = f32(2.0 ** e)
        u = float(np.spacing(p))
        for sgn in (1, -1):
            for lag_frac in (0.0, 0.5, 1.0, 1.5):
                # the member in between moves |num| down by up to its bound: to or across the power of two below
                w1 = f32(u * lag_frac) if lag_frac else f32(0.0)
                for ws in (u / 8 * (1 - 2 ** -20), u / 8, u / 4 * (1 - 2 ** -20), u / 4, u / 4 * (1 + 2 ** -20), u / 2):
                    w = f32(ws)
                    if w == 0:
                        continue
                    for s in (f32(1.0), f32(-1.0), f32(1 - 2 ** -24)):
                        cases.append((f32(sgn * p), w1, f32(-sgn), f32(1.0), w, s, f32(1.0)))
        # ties: num with an odd mantissa
        q = f32(p * f32(1 + 2 ** -23))
        cases.append((q, f32(0.0), f32(1.0), f32(1.0), f32(u / 2), f32(1.0), f32(1.0)))
    tiny = f32(np.finfo(np.float32).tiny)
    for w in (f32(1e-45), f32(1e-40), tiny):
        cases += [(f32(0.0), f32(0.0), f32(1.0), f32(1.0), w, f32(1.0), f32(1.0)),
                  (f32(1e-39), f32(0.0), f32(1.0), f32(1.0), w, f32(1.0), f32(1.0)),
                  (f32(1.0), w, f32(1.0), f32(1.0), w, f32(-1.0), f32(1.0))]
    passed = [check(*c) for c in cases]
    assert any(passed) and not all(passed)
    # w = +0 passes whatever num is; invalid points pass; L below 2^-100 or NaN never certifies a non-zero weight
    assert A.point_pass(f32(0.0), f32(1.0), f32(0.0), f32(0.0), True)
    assert A.point_pass(f32(1.0), f32(1.0), f32(0.0), f32(0.0), False)
    assert not A.point_pass(f32(1e-45), f32(1.0), f32(2.0 ** -101), f32(0.0), True)
    assert not A.point_pass(f32(1e-45), f32(1.0), f32(np.inf), f32(np.inf), True)
    assert not A.point_pass(f32(1e-45), f32(1.0), f32(np.nan), f32(0.0), True)
    # the strict inequality at ulp(1) / 4 = 2^-25, and the lag: L = 1 - 2^-30 rounds down into [1/2, 1)
    assert not A.point_pass(f32(2.0 ** -25), f32(1.0), f32(1.0), f32(0.0), True)
    assert A.point_pass(f32(2.0 ** -26), f32(1.0), f32(1.0), f32(0.0), True)
    assert not A.point_pass(f32(2.0 ** -26), f32(1.0), f32(1.0), f32(2.0 ** -30), True)
    assert A.point_pass(f32(2.0 ** -27), f32(1.0), f32(1.0), f32(2.0 ** -30), True)


def test_predictor_point_counts():
    r = A.predict(latent_seed=1, res=24)
    # every member the per-point rule certifies changes no bit (asserted per tile inside predict)
    assert 0 < r['absorbed_point'] <= r['absorbed_point_no_lag'] <= r['unchanged'] <= r['den_absorbed']
    assert r['evaluated_point'] + r['absorbed_point'] + r['zero'] == r['member_tiles']
    assert r['evaluated_point'] < r['evaluated_absorb']
