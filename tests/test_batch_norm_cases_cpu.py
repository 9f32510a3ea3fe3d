"""CPU: the cases and restatements of tests/_batch_norm_cases.py, rehearsed before tests/test_batch_norm_envelope_gpu.py spends GPU time
on them -- exact cases that are what they claim (one integer mean per piece, a variance that is a power of four with eps, every
intermediate exact against Fraction, the ReLU's equality case present), the correctly rounded fma against Fraction on random triples
and midpoint ties, the pieces' order model against fp64 and on values whose sum shows the order, and the shape list against the C
ABI's checks and workspace size."""
import math
from fractions import Fraction

import numpy as np
import pytest

from fiery_b200 import _lib
from tests import _batch_norm_cases as BC


def _f32_of(fr):
    """a Fraction rounded once to the nearest fp32, ties to even (normal and subnormal range)"""
    if fr == 0:
        return np.float32(0.0)
    sign, a = (-1, -fr) if fr < 0 else (1, fr)
    e = math.floor(math.log2(a.numerator) - math.log2(a.denominator))
    while Fraction(2) ** e > a:
        e -= 1
    while Fraction(2) ** (e + 1) <= a:
        e += 1
    ulp = Fraction(2) ** (max(e, -126) - 23)
    q = a / ulp
    n = q.numerator // q.denominator
    rem = q - n
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and n % 2):
        n += 1
    return np.float32(sign * float(n * ulp))


# ------------------------------------------------------------------------------------------------------------------------------
# fmaf_exact
# ------------------------------------------------------------------------------------------------------------------------------
def test_fmaf_exact_against_fraction_on_random_triples():
    rng = np.random.default_rng(0)
    n = 4000
    a = (rng.standard_normal(n) * np.exp2(rng.integers(-20, 20, n))).astype(np.float32)
    b = (rng.standard_normal(n) * np.exp2(rng.integers(-20, 20, n))).astype(np.float32)
    c = (-(a.astype(np.float64) * b) * (1 + rng.standard_normal(n) * np.exp2(rng.integers(-30, 0, n)))).astype(np.float32)
    c[::3] = (rng.standard_normal(n)[::3] * 1e3).astype(np.float32)                 # and unrelated addends
    got = BC.fmaf_exact(a, b, c)
    want = np.array([_f32_of(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in zip(a, b, c)], np.float32)
    assert got.dtype == np.float32 and np.array_equal(got.view(np.int32), want.view(np.int32))


def test_fmaf_exact_at_midpoint_ties():
    """(1 + 2^-12)^2 = 1 + 2^-11 + 2^-24 is exactly half an fp32 ulp above 1 + 2^-11; a tiny addend decides the side, and without one
    the tie goes to even"""
    a = np.float32(1 + 2.0 ** -12)
    base = 1 + 2.0 ** -11
    up, even = np.float32(base + 2.0 ** -23), np.float32(base)
    assert BC.fmaf_exact(a, a, np.float32(0.0)) == even                               # tie, to the even mantissa
    assert BC.fmaf_exact(a, a, np.float32(2.0 ** -60)) == up                          # just above the tie
    assert BC.fmaf_exact(a, a, np.float32(-2.0 ** -60)) == even                       # just below
    assert BC.fmaf_exact(-a, a, np.float32(-2.0 ** -60)) == -up
    # an odd-mantissa neighbour: ties go up
    b = np.float32(1 + 2.0 ** -12 + 2.0 ** -22)
    exact = Fraction(float(a)) * Fraction(float(b))
    for c in (0.0, 2.0 ** -70, -2.0 ** -70):
        want = _f32_of(exact + Fraction(c))
        assert BC.fmaf_exact(a, b, np.float32(c)) == want, c
    # the plain fp64 route rounds twice and misses the side
    assert np.float32(float(a) * float(a) + 2.0 ** -60) == even
    # exact zeros and non-finite values pass through
    assert BC.fmaf_exact(np.float32(0.25), np.float32(4.0), np.float32(-1.0)) == 0.0
    assert np.isnan(BC.fmaf_exact(np.float32(np.nan), np.float32(1.0), np.float32(0.0)))
    assert BC.fmaf_exact(np.float32(np.inf), np.float32(2.0), np.float32(-1.0)) == np.inf


def test_fma64_is_rounded_once():
    a = 1 + 2.0 ** -30
    assert BC.fma64(a, a, -(1 + 2.0 ** -29))[()] == 2.0 ** -60                        # the product's low bits survive
    assert a * a - (1 + 2.0 ** -29) == 0.0


# ------------------------------------------------------------------------------------------------------------------------------
# the pieces' order model
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pixels", [1, 3, 5, 1023, 4092, 4095, 4096, 4097, 8193, 12289])
def test_piece_sums_model_on_exactly_summable_data_and_mixed_magnitudes(pixels):
    rng = np.random.default_rng(pixels)
    ints = rng.integers(-50, 51, (3, pixels)).astype(np.float32)
    got = BC.bn_piece_sums_model(ints, pixels)
    sizes = BC.piece_sizes(pixels)
    assert got.shape == (3, len(sizes)) and got.dtype == np.float32
    edges = np.cumsum([0] + sizes)
    want = np.stack([ints[:, a:b].astype(np.float64).sum(1) for a, b in zip(edges, edges[1:])], 1)
    assert np.array_equal(got.astype(np.float64), want)
    if pixels < 64:
        return
    mixed = (rng.standard_normal((64, pixels)) * np.exp2(rng.integers(-12, 13, (64, pixels)))).astype(np.float32)
    model = BC.bn_piece_sums_model(mixed, pixels)[:, 0]
    seq = np.add.accumulate(mixed[:, :sizes[0]], axis=1, dtype=np.float32)[:, -1]
    ref = mixed[:, :sizes[0]].astype(np.float64).sum(1)
    assert not np.array_equal(model, seq)                                          # the order shows in the bits
    bound = 4 * math.sqrt(sizes[0]) * np.spacing(np.abs(mixed).max(1)).astype(np.float64)
    assert np.all(np.abs(model.astype(np.float64) - ref) <= bound)


def _one(pixels, values):
    x = np.zeros(pixels, np.float32)
    for i, v in values.items():
        x[i] = v
    return float(BC.bn_piece_sums_model(x, pixels)[0])


def test_piece_sums_model_order_on_chosen_values():
    """2^24 and two 1.0s: 2^24 + 1 rounds back to 2^24 (ties to even) but 2^24 + 2 is exact, so where the two 1.0s meet each other
    before meeting 2^24 shows the order.  Thread 0 holds pixels 0-3, 1024-1027, 2048-2051, 3072-3075."""
    big, pixels = 2.0 ** 24, 4096
    assert _one(pixels, {0: big, 2: 1.0, 3: 1.0}) == big + 2              # (p0 + p1) + (p2 + p3)
    assert _one(pixels, {0: big, 1: 1.0, 2: 1.0}) == big                  # p1 meets p0 first
    assert _one(pixels, {0: big, 1024: 1.0, 2048: 1.0}) == big            # the chunks one after the other
    assert _one(pixels, {1024: big, 0: 1.0, 1: 1.0}) == big + 2           # chunk 0 first: the two 1.0s meet before 2^24
    assert _one(pixels, {0: big, 4: 1.0, 68: 1.0}) == big + 2             # threads 1 and 17 meet at butterfly offset 16
    assert _one(pixels, {0: big, 4: 1.0, 8: 1.0}) == big                  # threads 1 and 2 meet thread 0 first
    assert _one(pixels, {0: big, 128: 1.0, 256: 1.0}) == big              # warps 0, 1, 2 one after the other
    assert _one(pixels, {0: big, 512: 1.0, 768: 1.0}) == big              # warps 4 and 6
    assert _one(4097, {4096: 3.0}) == 0.0 and float(BC.bn_piece_sums_model(np.full(4097, 3.0, np.float32), 4097)[-1]) == 3.0


def test_chan_merge_roundings():
    """The two roundings of the merge agree with an exact Fraction merge to within fp64 rounding, and differ on some data"""
    rng = np.random.default_rng(3)
    means = (rng.standard_normal((64, 30)) * 3 + 100).astype(np.float32)
    m2s = (rng.random((64, 30)) * 4096).astype(np.float32)
    counts = np.array([4096] * 9 + [3136], np.float64)
    counts = np.tile(counts, 3)
    mu, vu = BC.chan_merge(means, m2s, counts, False)
    mc, vc = BC.chan_merge(means, m2s, counts, True)
    n = Fraction(int(counts.sum()))
    for c in range(4):
        m = sum(Fraction(float(v)) * int(k) for v, k in zip(means[c], counts)) / n
        assert abs(float(mu[c]) - float(m)) <= 2 * np.spacing(mu[c]) and abs(float(mc[c]) - float(m)) <= 2 * np.spacing(mc[c])
    assert np.allclose(vu, vc, rtol=1e-6)


# ------------------------------------------------------------------------------------------------------------------------------
# exact cases
# ------------------------------------------------------------------------------------------------------------------------------
def _exact_checks(shape, eps, affine=True):
    case = BC.exact_case(shape, seed=sum(shape), eps=eps, affine=affine)
    b, c, s, X, Y = shape
    pixels = X * Y
    x = case["x"]
    assert x.shape == (b, c, s, pixels) and np.all(x == np.round(x)) and np.abs(x).max() < 64
    sizes = BC.piece_sizes(pixels)
    edges = np.cumsum([0] + sizes)
    d = x.astype(np.int64) - case["mu"].reshape(1, c, 1, 1)
    for a, e in zip(edges, edges[1:]):                                        # every piece: the channel's integer mean
        assert np.all(d[..., a:e].sum(-1) == 0)
        if e - a == 1:
            assert np.all(d[..., a] == 0)
    v = case["var"]
    n = b * s * pixels
    assert np.all((d ** 2).sum((0, 2, 3)) == v * n)
    ve = Fraction(v) + Fraction(case["eps"])
    k = round(math.log(float(ve), 4))
    assert ve == Fraction(4) ** k, "var + eps is a power of four"
    for training in (True, False):
        for relu in (True, False):
            u = BC.restate(x, case["w"], case["b"], case["rm"], case["rv"], case["r"], case["dy"], training, relu, case["eps"], False)
            if relu:                                                        # the contraction touches the statistics and shift only
                k_ = BC.restate(x, case["w"], case["b"], case["rm"], case["rv"], case["r"], case["dy"], training, relu, case["eps"],
                                True)
                for name in ("mean", "var", "scale", "shift", "y", "dx", "dw", "db"):
                    assert np.array_equal(u[name].view(np.int32), k_[name].view(np.int32)), (name, training, relu)
            assert np.array_equal(u["mean"], case["mu"].astype(np.float32)) and np.all(u["var"] == v)
            w = np.ones(c) if case["w"] is None else case["w"].astype(np.float64)
            bias = np.zeros(c) if case["b"] is None else case["b"].astype(np.float64)
            for ch in range(0, c, max(1, c // 7)):                           # against Fraction, a handful of channels
                sc = Fraction(float(w[ch])) / Fraction(2) ** k
                sh = Fraction(float(bias[ch])) - Fraction(int(case["mu"][ch])) * sc
                assert Fraction(float(u["scale"][ch])) == sc and Fraction(float(u["shift"][ch])) == sh
                xs = x[:, ch].ravel()[:64]
                pre = [sc * Fraction(float(t)) + sh for t in xs]
                yv = [max(p, Fraction(0)) if relu else p for p in pre]
                yv = [p + Fraction(float(r)) for p, r in zip(yv, case["r"][:, ch].ravel()[:64])]
                assert [Fraction(float(t)) for t in u["y"][:, ch].ravel()[:64]] == yv
                g = case["dy"][:, ch].astype(np.float64)
                if relu:
                    pre_all = float(sc) * x[:, ch].astype(np.float64) + float(sh)
                    g = np.where(pre_all <= 0, 0.0, g)
                s1 = int(g.sum())
                s2 = int((g * d[:, ch]).sum())
                assert float(u["db"][ch]) == s1 and Fraction(float(u["dw"][ch])) == Fraction(s2) / Fraction(2) ** k
    return case


@pytest.mark.parametrize("shape", BC.SHAPE_LIST, ids=lambda s: "x".join(map(str, s)))
def test_exact_cases_are_exact(shape):
    case = _exact_checks(shape, 0.0)
    if case["w"] is not None and np.prod(shape[3:]) > 1:
        u = BC.restate(case["x"], case["w"], case["b"], None, None, None, None, True, True, case["eps"])
        pre = BC.fmaf_exact(u["scale"].reshape(1, -1, 1, 1), case["x"], u["shift"].reshape(1, -1, 1, 1))
        assert np.any(pre == 0) and np.any(pre > 0) and np.any(pre < 0)      # the ReLU's equality case is there


@pytest.mark.parametrize("shape,eps", [((2, 3, 1, 1, 4097), 8.0), ((2, 129, 1, 1, 2), 8.0), ((2, 4, 3, 200, 200), 8.0),
                                       ((1, 2, 1, 1, 7), 12.0)], ids=str)
def test_exact_cases_with_eps(shape, eps):
    _exact_checks(shape, eps)


def test_exact_cases_without_affine():
    _exact_checks((2, 3, 1, 1, 4097), 0.0, affine=False)


# ------------------------------------------------------------------------------------------------------------------------------
# the shape list
# ------------------------------------------------------------------------------------------------------------------------------
def test_shape_list_covers_the_envelope():
    pixels = {X * Y for _, _, _, X, Y in BC.SHAPE_LIST}
    assert set(BC.PIXELS) <= pixels
    assert set(BC.CHANNELS) <= {c for _, c, _, _, _ in BC.SHAPE_LIST}
    bs = {b * s for b, _, s, _, _ in BC.SHAPE_LIST}
    assert {1, 2, 3, 6, 64} <= bs
    assert any(b * s * len(BC.piece_sizes(X * Y)) >= 10 ** 4 for b, _, s, X, Y in BC.SHAPE_LIST)
    assert any(c >= 1000 and X * Y == 1 for _, c, _, X, Y in BC.SHAPE_LIST)
    assert {n for p in pixels for n in BC.piece_sizes(p)} >= {1, 2, 3, 4, 4096}


def _desc(shape, training, relu, eps=1e-5):
    b, c, s, X, Y = shape
    d = _lib.BatchNormDesc()
    d.batch, d.channels, d.frames, d.pixels = b, c, s, X * Y
    d.stride_b, d.stride_c, d.stride_t = c * s * X * Y, s * X * Y, X * Y
    d.training, d.relu, d.eps = training, relu, eps
    return d


@pytest.mark.parametrize("shape", BC.SHAPE_LIST, ids=lambda s: "x".join(map(str, s)))
def test_shapes_pass_the_checks_with_the_workspace_rule(shape):
    lib = _lib.load()
    b, c, s, X, Y = shape
    want = BC.workspace_bytes(c, b, s, X * Y)
    for training in (1, 0):
        for relu in (1, 0):
            assert lib.fiery_batch_norm_workspace_bytes(_desc(shape, training, relu)) == want
            assert lib.fiery_batch_norm_workspace_bytes(_desc(shape, training, relu, eps=0.0)) == want
