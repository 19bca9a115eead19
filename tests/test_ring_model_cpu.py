"""The stated arithmetic of the ring GEMV (oracle.fma32 / ring_stated / ring_norm_row, DESIGN.md section 4) checked on its own:
fma32 against exact rational arithmetic, including operands built to land on fp32 midpoints; ring_stated against the fp64
block-sum model imma_stated to the error bound of its fp32 chains; ring_norm_row against an fp64 RMSNorm, and bit-exact on
constructions where every fp32 step is exact.  tests/test_gpu_ring.py holds the kernel to these functions bit for bit."""
from fractions import Fraction

import numpy as np
import pytest

import oracle


def f32_of(q: Fraction) -> np.float32:
    """a rational rounded to the nearest fp32 (ties to even); normal range only"""
    if q == 0:
        return np.float32(0)
    sign, q = (-1 if q < 0 else 1), abs(q)
    e = q.numerator.bit_length() - q.denominator.bit_length()
    while Fraction(2) ** e > q:
        e -= 1
    while Fraction(2) ** (e + 1) <= q:
        e += 1
    assert -126 <= e <= 127
    mant = q / Fraction(2) ** (e - 23)  # in [2^23, 2^24)
    fl = mant.numerator // mant.denominator
    rem = mant - fl
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and fl % 2 == 1):
        fl += 1
    return np.float32(sign * float(fl) * 2.0 ** (e - 23))


def exact_fma(x, y, z):
    return f32_of(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z)))


def test_fma32_matches_exact_rounding_on_random_operands():
    rng = np.random.default_rng(1)
    n = 4000
    x = (rng.normal(0, 1, n) * 2.0 ** rng.integers(-20, 20, n)).astype(np.float32)
    y = (rng.normal(0, 1, n) * 2.0 ** rng.integers(-20, 20, n)).astype(np.float32)
    z = (rng.normal(0, 1, n) * 2.0 ** rng.integers(-30, 30, n)).astype(np.float32)
    xi = rng.integers(-2 ** 17, 2 ** 17, n)
    got, goti = oracle.fma32(x, y, z), oracle.fma32(xi, y, z)
    for i in range(n):
        assert got[i] == exact_fma(x[i], y[i], z[i]), i
        assert goti[i] == exact_fma(xi[i], y[i], z[i]), i
    # cancellation to zero gives +0 (round to nearest), as fmaf does
    zero = oracle.fma32(np.array([3], np.int64), np.float32([0.5]), np.float32([-1.5]))
    assert zero[0] == 0 and not np.signbit(zero[0])


def integer_midpoint_operands(count=6):
    """(x, y) with x an integer below 2^17 and y fp32 such that x * y = 2^-24 (1 +- t 2^-40), 0 < t < 2^11: added to z in [1, 2)
    the fp64 sum lands exactly on the fp32 midpoint z + 2^-24 and the lost tail decides the rounding"""
    out = []
    for sign in (1, -1):
        found = 0
        for x in range(2 ** 16 + 1, 2 ** 17):
            t = (-sign * 2 ** 40) % x  # x divides 2^40 + sign t
            if 0 < t < 2 ** 11 and (2 ** 40 + sign * t) // x < 2 ** 24:
                out.append((x, np.float32((2 ** 40 + sign * t) // x * 2.0 ** -64)))
                found += 1
                if found == count:
                    break
    return out


def test_fma32_on_fp32_midpoints():
    """the fp64 sum sits exactly on an fp32 midpoint and only the fp64 rounding error tells which way the exact value lies"""
    # fp32 operands: x y = 1 - 2^-40 against z of ulp 2 (midpoints at odd integers)
    a, b = np.float32(1 + 2.0 ** -20), np.float32(1 - 2.0 ** -20)
    fcases = [(np.float32(sx * a), b, np.float32(sz * z)) for z in (2.0 ** 24 + 2, 2.0 ** 24 + 6, 2.0 ** 24 + 4, 3 * 2.0 ** 23 + 2)
              for sx in (1, -1) for sz in (1, -1)]
    # an integer x (the ring's isum) times an fp32 scale
    pairs = integer_midpoint_operands()
    assert len(pairs) == 12
    icases = [(s * x, y, np.float32(s * z)) for x, y in pairs for z in (1.0, 1.0 + 2.0 ** -23, 1.5, 1.5 + 2.0 ** -23) for s in (1, -1)]
    differ = 0
    for cases, xt in ((fcases, np.float32), (icases, np.int64)):
        xs, ys, zs = (np.array([c[i] for c in cases], dt) for i, dt in enumerate((xt, np.float32, np.float32)))
        got = oracle.fma32(xs, ys, zs)
        want = np.array([exact_fma(*c) for c in cases], np.float32)
        assert np.array_equal(got, want)
        naive = (xs.astype(np.float64) * ys.astype(np.float64) + zs.astype(np.float64)).astype(np.float32)
        differ += int((naive != want).sum())
    assert differ >= (len(fcases) + len(icases)) // 4  # the constructions do hit the double-rounding cases


def test_fma32_rejects_subnormals():
    with pytest.raises(AssertionError):
        oracle.fma32(np.float32([1e-40]), np.float32([1]), np.float32([0]))


def random_weights(rng, k, n, g, asym):
    nb = -(-k // g)
    q = rng.integers(-8, 8, (k, n)).astype(np.int8)
    zp = rng.integers(-8, 8, (nb, n)).astype(np.int8) if asym else None
    sc = (rng.uniform(0.5, 1.5, (nb, n)) / 16).astype(np.float32)
    return q, sc, zp


@pytest.mark.parametrize("comp,g,asym,k", [("q8_0", 32, False, 4096), ("int8", 128, True, 11008), ("int8_s8", 32, False, 1056),
                                           ("int8", 32, False, 2048), ("q8_0", 128, True, 4000), ("int8_s8", 256, True, 1024)])
def test_ring_stated_within_the_bound_of_imma_stated(comp, g, asym, k):
    """the per-lane fp32 chains plus the butterfly stay within gamma_n sum |t_b| of the exact sum, n = chain length + 5"""
    rng = np.random.default_rng(k + g)
    m, n = 2, 96
    q, sc, zp = random_weights(rng, k, n, g, asym)
    a = rng.normal(0, 1, (m, k)).astype(np.float32)
    codes, asc, ab = oracle.imma_act(a, comp, g)
    got = oracle.ring_stated(codes, asc, ab, q, sc, zp, g)
    tot, mag, _ = oracle.imma_stated(codes, asc, ab, q, sc, zp, g)
    chain = -(-k // 1024)  # chunks per lane
    assert oracle.imma_bound_ratio(got, tot, mag, chain, splits=5) <= 1.0


def test_ring_stated_exact_on_exact_data():
    """power-of-two scales and small codes: every fp32 step is exact, so the chains equal the fp64 sum"""
    rng = np.random.default_rng(3)
    k, n, g = 2048, 40, 64
    q = rng.integers(-8, 8, (k, n)).astype(np.int8)
    zp = rng.integers(-8, 8, (k // g, n)).astype(np.int8)
    sc = (2.0 ** -rng.integers(0, 3, (k // g, n))).astype(np.float32)
    codes = rng.integers(-5, 6, (3, k)).astype(np.int64)
    asc = (2.0 ** -rng.integers(0, 3, (3, k // g))).astype(np.float32)
    got, lanes = oracle.ring_stated(codes, asc, g, q, sc, zp, g, lanes=True)
    tot, _, _ = oracle.imma_stated(codes, asc, g, q, sc, zp, g)
    assert np.array_equal(got, tot.astype(np.float32))
    # lane L holds exactly the chunks c = L mod 32
    isum = (codes[:, None, :].reshape(3, 1, k // 32, 32) *
            (q.astype(np.int64) - np.repeat(zp, g, 0)).T.reshape(1, n, k // 32, 32)).sum(-1)          # [M, N, chunks]
    t = asc[:, None, (np.arange(k // 32) * 32) // g] * sc[(np.arange(k // 32) * 32) // g].T[None]  # [M, N, chunks]
    per_lane = (isum * t.astype(np.float64)).reshape(3, n, -1, 32).sum(2)
    assert np.array_equal(lanes.transpose(1, 2, 0), per_lane.astype(np.float32))


def test_ring_stated_partial_chunk_and_group_equal_to_k():
    """K = 1000 with one group of K (the prepared path): 32 chunks, the last one partial, all under scale 0"""
    rng = np.random.default_rng(4)
    k, n = 1000, 24
    q, sc, zp = random_weights(rng, k, n, k, True)
    a = rng.normal(0, 1, (1, k)).astype(np.float32)
    codes, asc, ab = oracle.imma_act(a, "int8", k)
    got = oracle.ring_stated(codes, asc, ab, q, sc, zp, k)
    tot, mag, _ = oracle.imma_stated(codes, asc, ab, q, sc, zp, k)
    assert oracle.imma_bound_ratio(got, tot, mag, 1, splits=5) <= 1.0


@pytest.mark.parametrize("nt", [224, 448])
@pytest.mark.parametrize("k", [4096, 5376, 5408, 10752, 10784, 1000])
def test_ring_norm_row_against_fp64(nt, k):
    rng = np.random.default_rng(k + nt)
    x = rng.normal(0, 1, k).astype(np.float32)
    w = rng.uniform(0.5, 1.5, k).astype(np.float32)
    got = oracle.ring_norm_row(x, w, 1e-5, nt)
    xd = x.astype(np.float64)
    want = xd / np.sqrt((xd * xd).mean() + np.float64(np.float32(1e-5))) * w
    assert np.abs(got - want).max() <= 1e-6 * np.abs(want).max()


@pytest.mark.parametrize("nt", [224, 448])
def test_ring_norm_row_exact_construction(nt):
    """eps = 0, |x| = 2^e everywhere, norm weights powers of two: tot = k 4^e, inv = 2^-e exactly, row = sign(x) w"""
    rng = np.random.default_rng(nt)
    for k in (5376, 5408, 10752, 10784):
        e = int(rng.integers(-6, 6))
        x = (rng.choice([-1.0, 1.0], k) * 2.0 ** e).astype(np.float32)
        w = (2.0 ** rng.integers(-3, 4, k)).astype(np.float32)
        assert np.array_equal(oracle.ring_norm_row(x, w, 0.0, nt), np.sign(x) * w)


def test_ring_norm_row_order_matters():
    """the two CTA widths sum the squares in different orders: on random rows the rows differ in the last bits somewhere"""
    rng = np.random.default_rng(9)
    diffs = 0
    for _ in range(20):
        x = rng.normal(0, 1, 4096).astype(np.float32) * np.float32(3.7)
        w = np.ones(4096, np.float32)
        diffs += not np.array_equal(oracle.ring_norm_row(x, w, 1e-6, 224), oracle.ring_norm_row(x, w, 1e-6, 448))
    assert diffs > 0
