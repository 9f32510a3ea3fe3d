"""CPU: the group restatement of tests/_batch_norm_cases.py (``merge_ranks``, ``restate_group``, ``exact_group_case``, ``SPLITS``)
against fp64 brute force and against the single-rank restatement, the exactness of the exact group cases, the splits' power to
see each wrong merge, and the host check of the gathered triplets."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from fiery_b200 import batch_norm as BN
from tests import _batch_norm_cases as BC

EPS = 1e-5


def _bits(a):
    return np.asarray(a, np.float32).view(np.int32)


def _same_bits(a, b):
    return np.asarray(a).shape == np.asarray(b).shape and np.array_equal(_bits(a), _bits(b))


def _random(shape, seed, spread=1.0):
    rng = np.random.default_rng(seed)
    b, c, s, X, Y = shape
    p = X * Y
    x = (rng.standard_normal((b, c, s, p)) * 2 + rng.standard_normal(c).reshape(1, c, 1, 1) * 3 * spread).astype(np.float32)
    w = (1 + 0.5 * rng.standard_normal(c)).astype(np.float32)
    w[::3] *= -1
    bias = (0.3 * rng.standard_normal(c)).astype(np.float32)
    r = rng.standard_normal(x.shape).astype(np.float32)
    dy = rng.standard_normal(x.shape).astype(np.float32)
    return x, w, bias, r, dy


def _group(x, w, bias, r, dy, sizes, relu=True, contracted=False, mutation=None, eps=EPS):
    return BC.restate_group(BC.shards_of(x, sizes), w, bias, BC.shards_of(r, sizes), BC.shards_of(dy, sizes), relu, eps, contracted,
                            mutation)


def _outputs(g):
    """every output of a restated group as one flat list of fp32 arrays"""
    return [g["mean"], g["var"], np.asarray(g["count"], np.float32)] + g["y"] + g["dx"] + g["dw"] + g["db"]


@pytest.mark.parametrize("name", BC.SPLIT_NAMES)
@pytest.mark.parametrize("shape", [(2, 3, 1, 1, 7), (4, 2, 2, 1, 4099), (8, 5, 1, 2, 3)], ids=lambda s: "x".join(map(str, s)))
def test_restate_group_against_fp64_brute_force(shape, name):
    sizes = BC.split_sizes(name, shape[0])
    if sizes is None:
        pytest.skip("split not defined for this batch")
    x, w, bias, r, dy = _random(shape, sum(shape))
    g = _group(x, w, bias, r, dy, sizes)
    x64 = x.astype(np.float64)
    mean64, var64 = x64.mean(axis=(0, 2, 3)), x64.var(axis=(0, 2, 3))
    n = x.size // x.shape[1]
    assert np.all(g["count"] == n)
    np.testing.assert_allclose(g["mean"], mean64, rtol=1e-6, atol=1e-6 * np.sqrt(var64).max())
    np.testing.assert_allclose(g["var"], var64, rtol=1e-5)
    bc = lambda v: v.reshape(1, -1, 1, 1)                                           # noqa: E731
    pre = (x64 - bc(mean64)) / np.sqrt(bc(var64) + EPS) * bc(w.astype(np.float64)) + bc(bias.astype(np.float64))
    y64 = np.maximum(pre, 0) + r
    gm = np.where(pre > 0, dy.astype(np.float64), 0.0)
    xh = (x64 - bc(mean64)) / np.sqrt(bc(var64) + EPS)
    dbeta, dgamma = gm.sum(axis=(0, 2, 3)), (gm * xh).sum(axis=(0, 2, 3))
    dx64 = bc(w.astype(np.float64)) / np.sqrt(bc(var64) + EPS) * (gm - bc(dbeta) / n - xh * bc(dgamma) / n)
    rel = lambda a, e: np.linalg.norm(a - e) / max(np.linalg.norm(e), 1e-30)   # noqa: E731
    assert rel(np.concatenate(g["y"]), y64) < 1e-5
    assert rel(np.concatenate(g["dx"]), dx64) < 1e-4
    assert rel(sum(d.astype(np.float64) for d in g["db"]), dbeta) < 1e-5
    assert rel(sum(d.astype(np.float64) for d in g["dw"]), dgamma) < 1e-5
    for k, (a, b) in enumerate(zip(g["db"], BC.shards_of(gm, sizes))):            # each rank's own dbeta
        np.testing.assert_allclose(a, b.sum(axis=(0, 2, 3)), rtol=1e-4, atol=1e-4 * np.abs(gm).sum() / x.shape[1])


@pytest.mark.parametrize("shape", [(2, 3, 1, 1, 1), (1, 4, 2, 1, 4097), (3, 2, 1, 5, 7)], ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("contracted", [False, True], ids=["plain", "contracted"])
def test_one_rank_group_is_restate_bit_for_bit(shape, contracted):
    x, w, bias, r, dy = _random(shape, 3)
    g = _group(x, w, bias, r, dy, [shape[0]], contracted=contracted)
    want = BC.restate(x, w, bias, None, None, r, dy, True, True, EPS, contracted)
    for name in ("mean", "var"):
        assert _same_bits(g[name], want[name]), name
    for name in ("y", "dx", "dw", "db"):
        assert _same_bits(g[name][0], want[name]), name


@pytest.mark.parametrize("contracted", [False, True], ids=["plain", "contracted"])
def test_empty_ranks_around_one_rank_change_no_bit(contracted):
    """Chan's step from (0, 0, 0) with the only non-empty rank, and every n = 0 rank skipped, is exact: wherever the data sits"""
    shape = (3, 4, 2, 1, 4099)
    x, w, bias, r, dy = _random(shape, 5, spread=30.0)
    ref = _outputs(_group(x, w, bias, r, dy, [3], contracted=contracted))
    for sizes in ([0, 3], [3, 0], [0, 0, 3], [0, 3, 0, 0], [0, 0, 0, 0, 0, 3], [0] * 7 + [3]):
        got = _group(x, w, bias, r, dy, sizes, contracted=contracted)
        k = sizes.index(3)
        flat = [got["mean"], got["var"], np.asarray(got["count"], np.float32)] + [got[n][k] for n in ("y", "dx", "dw", "db")]
        assert all(_same_bits(a, b) for a, b in zip(flat, ref)), sizes
        for n in ("y", "dx"):                                       # the empty ranks' outputs are empty
            assert all(got[n][i].size == 0 for i in range(len(sizes)) if i != k)
        assert all(not np.any(got["dw"][i]) and not np.any(got["db"][i]) for i in range(len(sizes)) if i != k)


EXACT_GROUPS = [
    ((4, 3, 1, 1, 4097), [0, 0, 1, 3], False),
    ((8, 5, 2, 1, 6), [0, 1, 0, 1, 2, 4], True),
    ((16, 3, 1, 1, 4100), [2, 2, 4, 0, 8], True),
    ((8, 2, 1, 2, 9), [1, 1, 2, 4], True),
]


@pytest.mark.parametrize("shape,sizes,offsets", EXACT_GROUPS, ids=str)
def test_exact_group_cases_are_exact_in_the_model(shape, sizes, offsets):
    case = BC.exact_group_case(shape, sizes, seed=2, offsets=offsets)
    x, r, dy = (BC.shards_of(case[k], sizes) for k in ("x", "r", "dy"))
    runs = [BC.restate_group(x, case["w"], case["b"], r, dy, relu, case["eps"], contracted)
            for relu in (True, False) for contracted in (False, True)]
    assert np.array_equal(runs[0]["mean"], case["mu"].astype(np.float32)) and np.all(runs[0]["var"] == np.float32(case["var"]))
    for a, b in ((runs[0], runs[1]), (runs[2], runs[3])):           # the contraction changes no bit
        assert all(_same_bits(u, v) for u, v in zip(_outputs(a), _outputs(b)))
    if offsets:                                                     # the ranks' means differ: the cross-rank delta^2 carries variance
        means = [t[:, 1] for t in runs[0]["gathered_forward"] if t[0, 0]]
        assert any(not np.array_equal(m, means[0]) for m in means[1:])
        within = sum(t[:, 2] for t in runs[0]["gathered_forward"])
        assert np.all(within < runs[0]["count"] * runs[0]["var"])
    # the statistics equal the fp64 ones exactly, and y the fp64 formula (every value is exact)
    x64 = case["x"].astype(np.float64)
    assert np.array_equal(x64.mean(axis=(0, 2, 3)), case["mu"]) and np.all(x64.var(axis=(0, 2, 3)) == case["var"])
    pre = (x64 - case["mu"].reshape(1, -1, 1, 1)) * (case["w"].astype(np.float64) / 4).reshape(1, -1, 1, 1) + \
        case["b"].astype(np.float64).reshape(1, -1, 1, 1)
    assert np.array_equal(np.concatenate(runs[0]["y"]).astype(np.float64), np.maximum(pre, 0) + case["r"])
    assert np.any(pre == 0)                                         # the ReLU's equality case is met


def test_every_mutation_shows_on_a_split():
    """each wrong merge of MUTATIONS changes the restated bits on at least one SPLITS entry, of random data or of the cancelling case
    (whose fp32 mean is the merge's rounding residue, so that the ranks' order shows): the GPU tests can see it"""
    shape = (8, 6, 1, 1, 4100)
    x, w, bias, r, dy = _random(shape, 11, spread=30.0)
    xc = BC.cancelling_case(6, 0)
    datasets = [(x, r, dy), (xc, np.zeros_like(xc), np.ones_like(xc))]
    seen = {m: [] for m in BC.MUTATIONS}
    for name in BC.SPLIT_NAMES:
        for xs, rs, dys in datasets:
            sizes = BC.split_sizes(name, xs.shape[0])
            if sizes is None:
                continue
            runs = [_outputs(_group(xs, w, bias, rs, dys, sizes, contracted=k)) for k in (False, True)]
            for m in BC.MUTATIONS:
                got = _outputs(_group(xs, w, bias, rs, dys, sizes, contracted=True, mutation=m))
                # different from the plain and the contracted arithmetic alike, which the GPU tests both accept
                if all(not all(_same_bits(a, b) for a, b in zip(got, ref)) for ref in runs):
                    seen[m].append(name)
    assert all(seen.values()), seen
    assert "0+0+a+b" in seen["no_skip"] and "0+all" not in seen["no_skip"], seen


def test_splits_cover_what_they_say():
    sizes = {name: BC.split_sizes(name, 4) for name in BC.SPLIT_NAMES}
    assert sizes["0+0+a+b"][:2] == [0, 0] and all(sizes["0+0+a+b"][2:])
    assert sizes["0x5+all"] == [0] * 5 + [4]
    assert len(sizes["8:3empty"]) == 8 and [sizes["8:3empty"][i] for i in (0, 3, 6)] == [0, 0, 0]
    sixty_four = BC.split_sizes("64", 40)
    assert len(sixty_four) == 64 and sum(sixty_four) == 40 and set(sixty_four) == {0, 1}
    assert BC.split_sizes("1+1", 2) == [1, 1]
    for name in BC.SPLIT_NAMES:
        for B in (1, 2, 3, 8, 64):
            s = BC.split_sizes(name, B)
            assert s is None or (sum(s) == B and min(s) >= 0), (name, B)


# ------------------------------------------------------------------------------------------------------------------------------
# the host rejects gathered triplets the kernels would misread, before any device work
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", ["float32", "transposed", "channels", "2-D", "no ranks"])
def test_gathered_must_be_contiguous_world_c_3_fp64(bad):
    c = 4
    x = torch.zeros(2, c, 1, 1, 8)
    good = torch.zeros(3, c, 3, dtype=torch.float64)
    gathered = {"float32": good.float(), "transposed": torch.zeros(3, 3, c, dtype=torch.float64).transpose(1, 2),
                "channels": torch.zeros(3, c + 1, 3, dtype=torch.float64), "2-D": torch.zeros(c, 3, dtype=torch.float64),
                "no ranks": torch.zeros(0, c, 3, dtype=torch.float64)}[bad]
    mean, var = torch.zeros(c), torch.ones(c)
    with pytest.raises(ValueError, match="gathered"):
        BN.forward_gathered(gathered, x, None, None, None, EPS, True)
    with pytest.raises(ValueError, match="gathered"):
        BN.backward_gathered(gathered, torch.zeros_like(x), x, None, None, mean, var, EPS, True)
