"""The oracle of exact caches (no GPU): the C restatement of embeddingDotProduct under both sum rules, and the bound eps
(csrc/cache_scan.cu exact_eps, restated as cache_exact_oracle.exact_eps) on adversarial rows."""
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle import cache_exact_oracle as co


def _rn32(x: Fraction) -> float:
    """x rounded to the nearest float32, ties to even (subnormals included)."""
    if x == 0:
        return 0.0
    a = abs(x)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    ulp = Fraction(2) ** (max(e, -126) - 23)
    m = a / ulp
    f = math.floor(m)
    r = m - f
    f = f + 1 if r > Fraction(1, 2) or (r == Fraction(1, 2) and f % 2) else f
    return math.copysign(float(f * ulp), x)


def _families(rng, d, n=6):
    """rows and a query: random, cancelling (row = -query plus a small part), wide dynamic range, subnormal fp16
    components, non-unit norms."""
    q = rng.standard_normal(d).astype(np.float32)
    r = rng.standard_normal((n, d)).astype(np.float32)
    yield "random", q, r
    yield "cancel", q, (-q[None] + 1e-3 * rng.standard_normal((n, d))).astype(np.float32)
    wide = lambda *s: (rng.standard_normal(s) * 2.0 ** rng.integers(-24, 12, s)).astype(np.float32)
    yield "wide", wide(d), wide(n, d)
    sub = lambda *s: (rng.standard_normal(s) * 2.0 ** -16).astype(np.float32)      # fp16 subnormals (< 2^-14)
    yield "subnormal", sub(d), np.concatenate([sub(n // 2, d), rng.standard_normal((n - n // 2, d))]).astype(np.float32)
    yield "norms", (q * 300).astype(np.float32), (r * 2.0 ** rng.integers(-10, 8, (n, 1))).astype(np.float32)


@pytest.mark.parametrize("d", [8, 64, 768])
def test_unfused_equals_float32_in_order(d):
    rng = np.random.default_rng(d)
    for name, q, r in _families(rng, d):
        acc = np.zeros(len(r), np.float32)
        for i in range(d):
            acc = acc + (q[i] * r[:, i])                      # float32 product rounded, then float32 sum
        got = co.scores_go(q[None], r, 0)[0]
        assert np.array_equal(got.view(np.uint32), acc.view(np.uint32)), name


@pytest.mark.parametrize("d", [8, 64, 200])
def test_fused_equals_exact_rational(d):
    rng = np.random.default_rng(100 + d)
    for name, q, r in _families(rng, d, n=3):
        got = co.scores_go(q[None], r, 1)[0]
        for j in range(len(r)):
            dot = 0.0
            for i in range(d):
                dot = _rn32(Fraction(float(q[i])) * Fraction(float(r[j, i])) + Fraction(dot))
            assert got[j] == np.float32(dot), (name, j)
    # the two rules differ somewhere on random data
    q, r = rng.standard_normal((1, 64)).astype(np.float32), rng.standard_normal((200, 64)).astype(np.float32)
    assert not np.array_equal(co.scores_go(q, r, 0), co.scores_go(q, r, 1))


@pytest.mark.parametrize("d", [8, 16, 64, 256, 768, 1024])
def test_eps_bounds_fp16_score_against_go(d):
    """|s16 - s_go| <= eps for the exact fp16-operand score and for fp32 sums of its products in index order, reversed
    order and numpy's pairwise order, under both rules."""
    rng = np.random.default_rng(200 + d)
    worst = 0.0
    for rep in range(4):
        for name, q, r in _families(rng, d, n=8):
            q16, r16 = q.astype(np.float16).astype(np.float64), r.astype(np.float16).astype(np.float64)
            prods = q16[None] * r16                            # exact: 11 x 11 significant bits
            sums = [np.array([math.fsum(p) for p in prods])]
            p32 = prods.astype(np.float32)                     # exact as well
            for order in (slice(None), slice(None, None, -1)):
                acc = np.zeros(len(r), np.float32)
                for col in p32[:, order].T:
                    acc = acc + col
                sums.append(acc.astype(np.float64))
            sums.append(p32.sum(axis=1, dtype=np.float32).astype(np.float64))
            eps = co.exact_eps(float(np.linalg.norm(q.astype(np.float64))),
                               float(np.linalg.norm(r.astype(np.float64), axis=1).max()), d)
            for rule in (0, 1):
                go = co.scores_go(q[None], r, rule)[0].astype(np.float64)
                for s16 in sums:
                    err = np.abs(s16 - go).max()
                    assert err <= eps, (name, rule, err, eps)
                    worst = max(worst, err / eps)
    assert worst > 1e-3                                       # the families come near enough to the bound to test it
