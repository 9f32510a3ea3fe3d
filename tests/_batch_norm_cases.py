"""Cases and host-side restatements shared by tests/test_batch_norm_cases_cpu.py and tests/test_batch_norm_envelope_gpu.py: the shapes
that walk the fused BatchNorm3d's (csrc/batch_norm.cu) accepted range, the piece reduction's summation order in fp32, a correctly
rounded fp32 fma, the finalize's fp64 steps with and without the multiply-adds nvcc contracts, and exact cases whose every
intermediate is exact, so that any order and any contraction give the same bits.  Importable without a GPU: everything here is numpy.

The header (include/fiery_b200.h, fiery_batch_norm_*) fixes: pieces of 4096 pixels per (b, c, t) plane, the last one shorter; within
a piece thread i of 256 adds its 4-pixel chunks i, i + 256, i + 512, i + 768 in ascending order, each as (p0 + p1) + (p2 + p3), then
an xor butterfly 16 .. 1 and the 8 warp sums in ascending order; the piece mean is that sum over the count (an IEEE division: the
build has no fast math); per channel the pieces merge in ascending (b, t, piece) order in fp64; scale and shift are computed in fp64
from the fp32 statistics and rounded once; the apply is fmaf(scale, x, shift)."""
import math
from fractions import Fraction

import numpy as np

BN_THREADS = 256
BN_PIECE = 4096


def piece_sizes(pixels):
    """the pixel counts of one plane's pieces"""
    full, tail = divmod(pixels, BN_PIECE)
    return [BN_PIECE] * full + ([tail] if tail else [])


def workspace_bytes(channels, batch, frames, pixels):
    """fiery_batch_norm_workspace_bytes: 20-byte coefficients per channel in a 256-byte-rounded block, then one float2 per piece"""
    return (20 * channels + 255) // 256 * 256 + 8 * channels * batch * frames * len(piece_sizes(pixels))


# ------------------------------------------------------------------------------------------------------------------------------
# the piece reduction's order
# ------------------------------------------------------------------------------------------------------------------------------
def bn_piece_sums_model(planes, pixels):
    """The fp32 sum of every piece of every plane in the kernels' order: planes (..., pixels) -> (..., pieces per plane) np.float32.
    Pixels past a piece's end are zeros, as the kernels read them."""
    x = np.asarray(planes, dtype=np.float32)
    lead = x.shape[:-1]
    per_plane = len(piece_sizes(pixels))
    rows = int(np.prod(lead, dtype=np.int64)) * per_plane
    # threads holding a chunk: all 256 over 4 rounds, or the first ceil(n / 4) of one round; the others' totals are +0 (0.f plus
    # zeros) and change no sum, so a plane of a few pixels is modelled without its 4096-pixel padding
    rounds = 4 if pixels > BN_PIECE else -(-pixels // (4 * BN_THREADS))
    threads = BN_THREADS if rounds > 1 else -(-pixels // 4)
    pad = np.zeros((rows // per_plane, per_plane * rounds * threads * 4), np.float32)
    pad[:, :pixels] = x.reshape(-1, pixels)
    v = pad.reshape(rows, rounds, threads, 4)               # [piece, u, thread, lane]: chunk thread + 256 u holds pixels 4 chunk ..
    chunk = (v[..., 0] + v[..., 1]) + (v[..., 2] + v[..., 3])
    t = np.zeros((rows, threads), np.float32)
    for u in range(rounds):
        t = t + chunk[:, u]
    a = np.zeros((rows, BN_THREADS), np.float32)
    a[:, :threads] = t
    a = a.reshape(-1, BN_THREADS // 32, 32)
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        a = a + a[..., lane ^ o]
    total = a[:, 0, 0]
    for w in range(1, BN_THREADS // 32):
        total = total + a[:, w, 0]
    return total.reshape(*lead, per_plane)


def piece_counts(pixels):
    return np.array(piece_sizes(pixels), np.float32)


def channel_pieces(t, pixels):
    """(b, C, s, pixels) per-piece values (b, C, s, pieces) -> (C, b * s * pieces) in the finalize's ascending (b, t, piece) order"""
    b, c, s, p = t.shape
    return np.ascontiguousarray(np.transpose(t, (1, 0, 2, 3))).reshape(c, b * s * p)


def seq_sum64(v):
    """the fp64 sum of the last axis in ascending order, one addition after the other (the backward finalize's)"""
    return np.add.accumulate(np.asarray(v, np.float64), axis=-1)[..., -1]


# ------------------------------------------------------------------------------------------------------------------------------
# correctly rounded fp32 fma and fp64 multiply-adds
# ------------------------------------------------------------------------------------------------------------------------------
def fmaf_exact(a, b, c):
    """fmaf(a, b, c) on fp32 arrays, rounded once to nearest even: a * b is exact in fp64; p + c is resolved into s + e by TwoSum, and s
    rounded to fp32 unless it lies exactly on a midpoint between two fp32 values while e != 0, in which case e picks the side."""
    a, b, c = (np.asarray(t, np.float32) for t in (a, b, c))
    a, b, c = np.broadcast_arrays(a, b, c)
    with np.errstate(invalid="ignore", over="ignore"):
        p = a.astype(np.float64) * b.astype(np.float64)
        c64 = c.astype(np.float64)
        s = p + c64
        bb = s - p
        e = (p - (s - bb)) + (c64 - bb)
        r = s.astype(np.float32)
        toward = np.where(r.astype(np.float64) < s, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32)
        o = np.nextafter(r, toward)
        mid = (r.astype(np.float64) + o.astype(np.float64)) * 0.5
        tie = np.isfinite(s) & np.isfinite(o) & (r.astype(np.float64) != s) & (s == mid) & (e != 0)
        up = np.where(r > o, r, o)
        down = np.where(r > o, o, r)
        out = np.where(tie, np.where(e > 0, up, down), r)
    return out.astype(np.float32)


def fma64(a, b, c):
    """a * b + c rounded once to fp64 (what a contracted fp64 multiply-add gives), element by element through Fraction.  An exact
    zero takes IEEE's sign: a * b = -c is then exact in fp64, so the plain expression gives it."""
    a, b, c = np.broadcast_arrays(np.asarray(a, np.float64), np.asarray(b, np.float64), np.asarray(c, np.float64))
    out = np.empty(a.shape, np.float64)
    for i, (x, y, z) in enumerate(zip(a.flat, b.flat, c.flat)):
        plain = x * y + z
        exact = Fraction(x) * Fraction(y) + Fraction(z) if math.isfinite(plain) else None
        out.flat[i] = plain if exact is None or exact == 0 else float(exact)
    return out


# ------------------------------------------------------------------------------------------------------------------------------
# the finalize's fp64 steps
# ------------------------------------------------------------------------------------------------------------------------------
def chan_step(n, m, m2, nb, mb, m2b, contracted):
    """bn_chan_step: (n, m, m2) fp64 merged with a part of nb values, mean mb and M2 m2b.  contracted: m += delta * (nb / nn) and
    m2 += M2 + delta^2 * (n nb / nn) as fp64 fmas (nvcc's default), else each product rounded before its add."""
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        delta = np.asarray(mb, np.float64) - m
        nn = n + nb
        if contracted:
            m = fma64(delta, nb / nn, m)
            m2 = m2 + fma64(delta * delta, n * nb / nn, np.asarray(m2b, np.float64))
        else:
            m = m + delta * (nb / nn)
            m2 = m2 + (np.asarray(m2b, np.float64) + delta * delta * (n * nb / nn))
    return nn, m, m2


def chan_merge64(means, m2s, counts, contracted):
    """bn_merge_pieces: means, m2s (C, K) fp32 piece partials and counts (K,) in merge order -> the fp64 (n, m, m2) (C,) before any
    cast, from (0, 0, 0): a rank's local triplet (bn_local_forward_kernel), (0, 0, 0) for K = 0"""
    means, m2s = np.asarray(means, np.float32), np.asarray(m2s, np.float32)
    c = means.shape[0]
    n, m, m2 = np.zeros(c), np.zeros(c), np.zeros(c)
    for k in range(means.shape[1]):
        n, m, m2 = chan_step(n, m, m2, float(counts[k]), means[:, k].astype(np.float64), m2s[:, k], contracted)
    return n, m, m2


def chan_merge(means, m2s, counts, contracted):
    """bn_finalize_forward_kernel's merge: ``chan_merge64`` -> (mean, var) (C,) fp32"""
    n, m, m2 = chan_merge64(means, m2s, counts, contracted)
    return m.astype(np.float32), (m2 / n).astype(np.float32)


def scale_shift(w, b, mean, var, eps):
    """bn_scale_shift: (scale, shift uncontracted, shift contracted) (C,) fp32 from fp32 mean and var; w / b None: 1 / 0"""
    mean, var = np.asarray(mean, np.float32).astype(np.float64), np.asarray(var, np.float32).astype(np.float64)
    w64 = np.ones_like(mean) if w is None else np.asarray(w, np.float32).astype(np.float64)
    b64 = np.zeros_like(mean) if b is None else np.asarray(b, np.float32).astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        s = w64 / np.sqrt(var + eps)
        plain = b64 - mean * s
    return s.astype(np.float32), plain.astype(np.float32), fma64(-mean, s, b64).astype(np.float32)


def backward_coefficients(scale, s1, s2, var, eps, n):
    """bn_finalize_backward_kernel from the fp64 channel sums: (grad_weight, grad_bias, k1, k0) (C,) fp32"""
    ve = np.asarray(var, np.float32).astype(np.float64) + eps
    sc = np.asarray(scale, np.float32).astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        return ((s2 / np.sqrt(ve)).astype(np.float32), np.asarray(s1, np.float64).astype(np.float32),
                (-sc * s2 / (float(n) * ve)).astype(np.float32), (-sc * s1 / float(n)).astype(np.float32))


def _bc(v):
    return np.asarray(v, np.float32).reshape(1, -1, 1, 1)


def restate(x, w, b, rm, rv, r, dy, training, relu, eps, contracted=False):
    """The header's formulas with the pieces' fp32 order, the finalize's fp64 merge (contracted or not) and fmaf rounded once:
    x, r, dy (b, C, s, pixels) fp32 -> dict of mean, var, y, dx, dw, db (dw / db over the same mask as dx).  Bit-exact where the
    pieces' M2 and S2 are exact (their products may be contracted on the device): the exact cases."""
    x = np.asarray(x, np.float32)
    bsz, c, s, pixels = x.shape
    n = bsz * s * pixels
    counts = np.tile(piece_counts(pixels), bsz * s)
    if training:
        sums = bn_piece_sums_model(x, pixels)
        pm = sums / piece_counts(pixels)                                     # fp32 division
        reps = np.repeat(pm, piece_sizes(pixels), axis=-1)
        d = x - reps
        m2 = bn_piece_sums_model(d * d, pixels)
        mean, var = chan_merge(channel_pieces(pm, pixels), channel_pieces(m2, pixels), counts, contracted)
    else:
        mean, var = np.asarray(rm, np.float32), np.asarray(rv, np.float32)
    scale, shift_u, shift_c = scale_shift(w, b, mean, var, eps)
    shift = shift_c if contracted else shift_u
    pre = fmaf_exact(_bc(scale), x, _bc(shift))
    y = np.where(pre < 0, np.float32(0), pre) if relu else pre
    if r is not None:
        y = (y + np.asarray(r, np.float32)).astype(np.float32)
    out = dict(mean=mean, var=var, scale=scale, shift=shift, y=y)
    if dy is None:
        return out
    dy = np.asarray(dy, np.float32)
    with np.errstate(invalid="ignore"):
        g = np.where(pre <= 0, np.float32(0), dy) if relu else dy
    dmu = (x - _bc(mean)).astype(np.float32)
    s1 = seq_sum64(channel_pieces(bn_piece_sums_model(g, pixels), pixels))
    s2 = seq_sum64(channel_pieces(bn_piece_sums_model(g * dmu, pixels), pixels))
    dw, db, k1, k0 = backward_coefficients(scale, s1, s2, var, eps, n)
    if training:
        dx = fmaf_exact(_bc(scale), g, fmaf_exact(_bc(k1), dmu, _bc(k0)))
    else:
        dx = (_bc(scale) * g).astype(np.float32)
    out.update(dx=dx, dw=dw, db=db, s1=s1, s2=s2)
    return out


# ------------------------------------------------------------------------------------------------------------------------------
# exact cases
# ------------------------------------------------------------------------------------------------------------------------------
def _four_squares(r):
    """four non-negative integers whose squares sum to r (Lagrange), the largest first"""
    for a in range(math.isqrt(r), -1, -1):
        for b in range(min(a, math.isqrt(r - a * a)), -1, -1):
            for c in range(min(b, math.isqrt(r - a * a - b * b)), -1, -1):
                d2 = r - a * a - b * b - c * c
                d = math.isqrt(d2)
                if d * d == d2 and d <= c:
                    return [a, b, c, d]
    raise AssertionError(r)


def _magnitudes(m, total, rng):
    """m non-negative integers whose squares sum to `total` (None when there is no such set): for m >= 4, random values within 2 of
    base = isqrt(total / m), nudged one at a time until what is left is small, and that rest as four squares"""
    if m == 0:
        return [] if total == 0 else None
    if m < 4:
        def search(k, rest, cap):
            if k == 0:
                return [] if rest == 0 else None
            for a in range(min(cap, math.isqrt(rest)), -1, -1):
                tail = search(k - 1, rest - a * a, a)
                if tail is not None:
                    return [a] + tail
            return None
        return search(m, total, math.isqrt(total))
    base = max(1, math.isqrt(total // m))
    a = base + rng.integers(-1, 2, m - 4)
    rest = total - int((a * a).sum())
    cap = 4 * (base + 2) ** 2
    while rest < 0 or rest > cap:
        if rest < 0:                                        # each step gains 2a - 1 <= 2 base + 1
            idx = np.flatnonzero(a > 0)[:max(1, -rest // (2 * base + 1))]
            rest += int((2 * a[idx] - 1).sum())
            a[idx] -= 1
        else:                                               # each step costs 2a + 1 <= 2 base + 3
            idx = np.flatnonzero(a <= base)[:max(1, (rest - cap) // (2 * base + 3))]
            rest -= int((2 * a[idx] + 1).sum())
            a[idx] += 1
    return [int(v) for v in a] + _four_squares(rest)


def exact_deviations(b, c, s, pixels, v, rng):
    """(b, C, s, pixels) int deviations from the channel mean with a zero sum in every piece and sum of squares v * b * s * pixels per
    channel: pairs (+a, -a) inside each piece, a 0 in a piece of odd count (a 1-pixel piece sits on the mean).  None when the pieces'
    pairs cannot carry that sum."""
    sizes = piece_sizes(pixels)
    m = b * s * sum(n // 2 for n in sizes)
    total = v * b * s * pixels
    if total % 2:
        return None
    mags = _magnitudes(m, total // 2, rng)
    if mags is None:
        return None
    d = np.zeros((c, b * s, pixels), np.int64)
    for ch in range(c):
        a = rng.permutation(np.array(mags, np.int64))
        k = 0
        for p in range(b * s):
            o = 0
            for n in sizes:
                h = n // 2
                piece = np.zeros(n, np.int64)
                piece[:h], piece[h:2 * h] = a[k:k + h], -a[k:k + h]
                d[ch, p, o:o + n] = rng.permutation(piece)
                k += h
                o += n
    return d.reshape(c, b, s, pixels).transpose(1, 0, 2, 3)


GAMMAS = np.array([1.0, -1.5, 0.0, 0.25, 2.0, -0.5, 1.5, -2.0], np.float32)


def exact_case(shape, seed, eps=0.0, affine=True):
    """Inputs (b, C, s, X, Y) for which every intermediate of training and eval is exact, so the kernels' bits are the header's
    formula's whatever the order and the contraction.  Per channel: x = mu_c + d with mu_c a small integer and d exact_deviations
    (every piece's mean is mu_c, Chan's delta 0 after the first piece), the biased var v with v + eps = 16 (v = 16 - eps; planes of
    one pixel have v = 0 and then eps = 1); gamma dyadic, negative and 0 among them; beta = -scale * t for a small integer t, so that
    fmaf(scale, x, shift) is exactly 0 wherever d = t; running statistics mu_c and v; dy and the residual small integers.
    Returns a dict of fp32 arrays (x, r, dy as (b, C, s, pixels)) and eps."""
    b, c, s, X, Y = shape
    pixels = X * Y
    rng = np.random.default_rng(seed)
    if pixels == 1:
        v, eps = 0, 1.0
    else:
        v = 16 - eps
        assert v == int(v) and v > 0, eps
        v = int(v)
    d = exact_deviations(b, c, s, pixels, v, rng)
    assert d is not None, f"no exact deviations for {shape} at var {v}"
    mu = rng.integers(-8, 9, c)
    x = (mu.reshape(1, c, 1, 1) + d).astype(np.float32)
    ve = v + eps
    w = np.resize(GAMMAS, c).astype(np.float32) if affine else None
    scale = (w if affine else np.ones(c, np.float32)) / np.float32(math.sqrt(ve))
    typical = [int(np.median(np.abs(d[:, ch]))) for ch in range(c)]            # a deviation with others on both sides of it
    t = np.array([(typical[ch], -typical[ch], 0, 1)[ch % 4] for ch in range(c)])
    bias = (-scale * t).astype(np.float32) if affine else None
    return dict(x=x, w=w, b=bias, rm=mu.astype(np.float32), rv=np.full(c, v, np.float32),
                r=rng.integers(-4, 5, x.shape).astype(np.float32), dy=rng.integers(-3, 4, x.shape).astype(np.float32),
                eps=float(eps), mu=mu, var=v, zero_at=t if affine else np.zeros(c, np.int64))


# ------------------------------------------------------------------------------------------------------------------------------
# shapes: (b, C, s, X, Y) and why each is there
# ------------------------------------------------------------------------------------------------------------------------------
SHAPES = [
    ((2, 3, 1, 1, 1), "1-pixel planes: every piece one pixel, var 0, eps 1"),
    ((1, 129, 1, 1, 2), "2-pixel planes, one plane per channel; C = 129: a second finalize block with one channel"),
    ((4, 127, 1, 1, 3), "3-pixel planes: a partial chunk, one pair per plane; C = 127"),
    ((1, 128, 3, 1, 5), "5 pixels: one full chunk and one lane of the next; C = 128: one full finalize block"),
    ((3, 255, 1, 1, 7), "7 pixels: a chunk and three lanes; C = 255"),
    ((1, 2, 1, 4, 1023), "4092 pixels: one piece, the last chunk of thread 254 of round 3, threads 255 idle"),
    ((2, 3, 1, 1, 4093), "4093: one piece ending one lane into thread 255's last chunk"),
    ((1, 2, 2, 1, 4094), "4094"),
    ((1, 3, 1, 1, 4095), "4095: one lane short of a whole piece"),
    ((1, 2, 2, 64, 64), "4096: exactly one piece"),
    ((2, 1, 1, 1, 4097), "4097: a whole piece and a 1-pixel piece on the mean"),
    ((1, 2, 1, 2, 2049), "4098: a 2-pixel last piece"),
    ((1, 1, 3, 1, 4099), "4099: a 3-pixel last piece"),
    ((1, 256, 1, 4, 1025), "4100: a 4-pixel last piece; C = 256: two full finalize blocks"),
    ((1, 2, 2, 1, 8191), "8191: a piece and a piece one pixel short"),
    ((2, 1, 1, 8, 1024), "8192: two whole pieces"),
    ((1, 3, 1, 1, 8193), "8193: two pieces and a 1-pixel third"),
    ((1, 2, 1, 1, 12289), "12289: three pieces and a 1-pixel fourth"),
    ((2, 4, 3, 200, 200), "40000: the shipped grid, 10 pieces per plane (9 whole and 3136 pixels)"),
    ((1, 2, 1, 200, 400), "80000: 20 pieces per plane"),
    ((8, 1000, 8, 1, 1), "many channels of 1-pixel planes: 8 finalize blocks, the last one partial, 64 pieces per channel"),
    ((4, 2, 5000, 1, 2), "20000 pieces of 2 pixels per channel: Chan's merge over many tiny pieces"),
    ((64, 2, 1, 1, 3), "b = 64, s = 1"),
    ((1, 3, 64, 1, 5), "b = 1, s = 64"),
    ((8, 5, 8, 3, 5), "b * s = 64"),
]
SHAPE_LIST = [shape for shape, _ in SHAPES]
PIXELS = [1, 2, 3, 5, 7, 4092, 4093, 4094, 4095, 4096, 4097, 4098, 4099, 4100, 8191, 8192, 8193, 12289, 40000, 80000]
CHANNELS = [1, 127, 128, 129, 255, 256, 1000]


# ------------------------------------------------------------------------------------------------------------------------------
# a process group (fiery_batch_norm_*_gathered): every rank's local triplet, gathered and merged in ascending rank order
# ------------------------------------------------------------------------------------------------------------------------------
def merge_ranks(triplets, contracted, descending=False, skip_empty=True):
    """bn_gathered_forward_kernel's merge: triplets (world, C, 3) fp64 (n, mean, M2) -> (n, m, m2) (C,) fp64: rank 0's triplet, then
    Chan's step with each later rank in ascending order, a rank with n = 0 skipped.  ``descending`` and ``skip_empty=False`` are the
    two ways of getting it wrong that tests/test_sync_batch_norm_cases_cpu.py shows the splits can see."""
    t = np.asarray(triplets, np.float64)[::-1] if descending else np.asarray(triplets, np.float64)
    n, m, m2 = t[0, :, 0].copy(), t[0, :, 1].copy(), t[0, :, 2].copy()
    for r in range(1, t.shape[0]):
        nn, mm, mm2 = chan_step(n, m, m2, t[r, :, 0], t[r, :, 1], t[r, :, 2], contracted)
        keep = t[r, :, 0] != 0 if skip_empty else np.ones_like(n, bool)
        n, m, m2 = np.where(keep, nn, n), np.where(keep, mm, m), np.where(keep, mm2, m2)
    return n, m, m2


def sum_ranks(triplets):
    """bn_gathered_backward_kernel's sum: (world, C, 3) (n, S1, S2) -> each summed over the ranks in ascending order, in fp64"""
    return tuple(seq_sum64(np.moveaxis(np.asarray(triplets, np.float64)[..., k], 0, -1)) for k in range(3))


def local_triplet(x, contracted):
    """bn_local_forward_kernel: x (b, C, s, pixels) fp32, b or s may be 0 -> (C, 3) fp64 (n, mean, M2)"""
    x = np.asarray(x, np.float32)
    bsz, c, s, pixels = x.shape
    if bsz * s == 0:
        return np.zeros((c, 3))
    sums = bn_piece_sums_model(x, pixels)
    pm = sums / piece_counts(pixels)
    d = x - np.repeat(pm, piece_sizes(pixels), axis=-1)
    m2 = bn_piece_sums_model(d * d, pixels)
    counts = np.tile(piece_counts(pixels), bsz * s)
    return np.stack(chan_merge64(channel_pieces(pm, pixels), channel_pieces(m2, pixels), counts, contracted), axis=1)


MUTATIONS = {
    "descending": "the ranks merged in descending order",
    "no_skip": "no n = 0 skip in the forward merge",
    "rank_n": "the rank's own n instead of the group's in the backward coefficients",
    "piece_count": "a rank's backward count written as per_channel * pixels (pieces times pixels)",
    "group_s2": "dgamma from the group's S2 instead of the rank's own",
}


def restate_group(shards, w, b, rs, dys, relu, eps, contracted=False, mutation=None):
    """The group path restated: shards, rs, dys lists of (b_r, C, s, pixels) fp32 per rank (b_r may be 0; rs / dys entries may be
    None) -> dict of the group's mean, var (C,) fp32 and count (fp64), the gathered forward and backward triplets, and per rank lists
    y, dx, dw, db (each rank's own dgamma / dbeta).  A group of one is ``restate``; ``mutation`` (a key of MUTATIONS) restates a
    wrong kernel."""
    shards = [np.asarray(x, np.float32) for x in shards]
    c, s, pixels = shards[0].shape[1:]
    fwd = np.stack([local_triplet(x, contracted) for x in shards])
    n, m, m2 = merge_ranks(fwd, contracted, descending=mutation == "descending", skip_empty=mutation != "no_skip")
    with np.errstate(invalid="ignore", divide="ignore"):
        mean, var = m.astype(np.float32), (m2 / n).astype(np.float32)
    scale, shift_u, shift_c = scale_shift(w, b, mean, var, eps)
    shift = shift_c if contracted else shift_u
    out = dict(mean=mean, var=var, count=n, scale=scale, shift=shift, gathered_forward=fwd, y=[], dx=[], dw=[], db=[], s1=[], s2=[])
    pres, gs, dmus, bwd = [], [], [], []
    for x, r, dy in zip(shards, rs, dys):
        pre = fmaf_exact(_bc(scale), x, _bc(shift))
        y = np.where(pre < 0, np.float32(0), pre) if relu else pre
        out["y"].append((y + np.asarray(r, np.float32)).astype(np.float32) if r is not None else y)
        dy = np.asarray(dy, np.float32) if dy is not None else np.zeros_like(x)
        with np.errstate(invalid="ignore"):
            g = np.where(pre <= 0, np.float32(0), dy) if relu else dy
            dmu = (x - _bc(mean)).astype(np.float32)
        if x.shape[0] * s:
            s1 = seq_sum64(channel_pieces(bn_piece_sums_model(g, pixels), pixels))
            s2 = seq_sum64(channel_pieces(bn_piece_sums_model(g * dmu, pixels), pixels))
        else:
            s1 = s2 = np.zeros(c)
        per = len(piece_sizes(pixels)) if mutation == "piece_count" else 1
        bwd.append(np.stack([np.full(c, float(x.shape[0] * s * per * pixels)), s1, s2], axis=1))
        pres.append(pre)
        gs.append(g)
        dmus.append(dmu)
        out["s1"].append(s1)
        out["s2"].append(s2)
    bwd = np.stack(bwd)
    out["gathered_backward"] = bwd
    nb, s1g, s2g = sum_ranks(bwd)
    for k, (g, dmu) in enumerate(zip(gs, dmus)):
        dw, db, k1, k0 = backward_coefficients(scale, out["s1"][k], s2g if mutation == "group_s2" else out["s2"][k], var, eps, 1.0)
        n_coef = bwd[k, 0, 0] if mutation == "rank_n" else nb[0]
        _, _, k1, k0 = backward_coefficients(scale, s1g, s2g, var, eps, n_coef)
        out["dw"].append(dw)
        out["db"].append(db)
        out["dx"].append(fmaf_exact(_bc(scale), g, fmaf_exact(_bc(k1), dmu, _bc(k0))))
    return out


def shards_of(t, sizes):
    """t (B, ...) split along the batch into pieces of the given sizes (some 0)"""
    cuts = np.cumsum([0] + list(sizes))
    assert cuts[-1] == t.shape[0], (sizes, t.shape)
    return [t[cuts[i]:cuts[i + 1]] for i in range(len(sizes))]


def exact_group_case(shape, sizes, seed, eps=0.0, offsets=False):
    """An ``exact_case`` for a group: inputs (b, C, s, X, Y) split along the batch into ``sizes``.  offsets=False: every piece has
    mean mu_c, so Chan's delta is 0 across the ranks too.  offsets=True: the ranks' means are mu_c + a_r for integers a_r with the
    non-empty ranks' counts in ratios 1 : 1 : 2 : 4 (sizes must be so), sum n_r a_r = 0 and in-rank variance 14 - eps, so the group's
    var + eps is 16 with the cross-rank delta^2 term non-zero, and every nb / nn a power of two.  Returns the case dict of
    ``exact_case`` (x, r, dy whole-batch (b, C, s, pixels)) with "sizes" added."""
    if not offsets:
        case = exact_case(shape, seed, eps=eps)
        case["sizes"] = list(sizes)
        return case
    b, c, s, X, Y = shape
    pixels = X * Y
    full = [k for k in sizes if k]
    assert len(full) == 4 and [k // full[0] for k in full] == [1, 1, 2, 4] and full[0] * 8 == sum(full) == b, (sizes, shape)
    rng = np.random.default_rng(seed)
    a = iter((3, -1, 1, -1))                                    # 3 - 1 + 2 - 4 = 0, and sum n_r a_r^2 / n = 2
    v = 14 - eps
    assert v == int(v) and v > 0, eps
    mu = rng.integers(-8, 9, c)
    parts = []
    for k in sizes:
        if k == 0:
            parts.append(np.zeros((0, c, s, pixels)))
            continue
        d = exact_deviations(k, c, s, pixels, int(v), rng)
        assert d is not None, f"no exact deviations for {k} of {shape}"
        parts.append(mu.reshape(1, c, 1, 1) + next(a) + d)
    x = np.concatenate(parts).astype(np.float32)
    w = np.resize(GAMMAS, c).astype(np.float32)
    t = np.array([(3, -2, 0, 1)[ch % 4] for ch in range(c)])
    bias = (-(w / np.float32(4.0)) * t).astype(np.float32)
    return dict(x=x, w=w, b=bias, rm=mu.astype(np.float32), rv=np.full(c, 16 - eps, np.float32),
                r=rng.integers(-4, 5, x.shape).astype(np.float32), dy=rng.integers(-3, 4, x.shape).astype(np.float32),
                eps=float(eps), mu=mu, var=16 - eps, sizes=list(sizes))


def _spread(total, ranks, empty):
    """``total`` batch elements over ``ranks`` ranks, none on the ranks in ``empty``, the others as even as can be (earlier ones more)"""
    full = [r for r in range(ranks) if r not in empty]
    out = [0] * ranks
    for i in range(total):
        out[full[i % len(full)]] += 1
    return out


# (name, sizes(B) -> per-rank batch sizes or None where the split does not apply, why it is there)
SPLITS = [
    ("all", lambda B: [B], "one rank: the single-rank finalize's numbers"),
    ("0+all", lambda B: [0, B], "an empty rank 0: the merge starts from (0, 0, 0) and the first step must be exact"),
    ("0+0+a+b", lambda B: [0, 0, B - B // 2, B // 2], "two leading empty ranks: only the n = 0 skip keeps nb / nn from 0 / 0"),
    ("a+0+b+0", lambda B: [B - B // 2, 0, B // 2, 0], "empty ranks between and after the data"),
    ("1+1", lambda B: [1, 1] if B == 2 else None, "two ranks of one batch element: single-value ranks on 1-pixel planes"),
    ("1+rest", lambda B: [1, B - 1] if B >= 2 else None, "one element on rank 0, the rest on rank 1: unequal counts"),
    ("0x5+all", lambda B: [0] * 5 + [B], "all data on the last of six ranks"),
    ("8:3empty", lambda B: _spread(B, 8, (0, 3, 6)), "8 ranks, 3 of them (0, 3 and 6) empty, the others uneven"),
    ("64", lambda B: [1 if (37 * r) % 64 < B else 0 for r in range(64)] if B <= 64 else None,
     "64 ranks, each holding one batch element or none"),
]
SPLIT_NAMES = [name for name, _, _ in SPLITS]


def split_sizes(name, B):
    return dict((n, f) for n, f, _ in SPLITS)[name](B)


def cancelling_case(c, seed):
    """x (7, C, 1, 2) whose batch elements hold 2a, a, a, -a, -a, -a, -a (a full-mantissa value per channel): the group's mean is 0
    exactly, so the fp32 mean is the fp64 merge's rounding residue, whose bits depend on the order of the ranks' merge"""
    a = ((np.random.default_rng(seed).random(c) + 0.5) * 1000).astype(np.float32).reshape(1, c, 1, 1)
    return np.concatenate([np.broadcast_to(2 * a, (1, c, 1, 2)), np.broadcast_to(a, (2, c, 1, 2)),
                           np.broadcast_to(-a, (4, c, 1, 2))]).astype(np.float32)
