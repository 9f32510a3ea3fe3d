"""CPU: the probes of tests/test_geometry_envelope_gpu.py sit where they claim.  Every boundary probe is on its side of the boundary
by the oracle's explicit fp32 chain and its nextafter neighbour on the other; the probes that claim an exact value (s = -1, s = N,
p - offset_z = z_lo / z_hi) have it, so a comparison that loses its equality case is seen; the reference chain on torch-CPU
(frustum_to_ego with the given combined, then voxel_indices; fiery.py:199-205,236-247) equals the explicit chain at every probe;
the run-pattern cases host every event they are meant to; and the intrinsics of the calibration test force the pivot orders they
are named for."""
import numpy as np
import pytest

from tests import _geometry_probes as G

ALL_GRIDS = {**G.GRIDS, **G.BIG_GRIDS}


def test_grids_have_the_intended_shapes():
    for name, g in G.GRIDS.items():
        assert (g.X, g.Y) == G.GRID_DIMS[name], name
    for name, g in G.BIG_GRIDS.items():
        assert (g.X, g.Y) == G.BIG_DIMS[name], name
    pow2 = lambda r: float(r) > 0 and np.frexp(np.float32(r))[0] == 0.5            # noqa: E731
    assert [pow2(r) for r in G.GRIDS["pow2"].res[:2]] == [True, True]
    assert [pow2(r) for r in G.GRIDS["div"].res[:2]] == [False, False]
    assert [pow2(r) for r in G.GRIDS["mixed"].res[:2]] == [True, False]
    assert (G.GRIDS["odd"].X * G.GRIDS["odd"].Y) % 2 == 1
    # float(X) rounds below X only for the 2^24 + 1 grids
    assert float(np.float32(G.EDGE + 1)) < G.EDGE + 1 and float(np.float32(G.EDGE + 3)) > G.EDGE + 3


@pytest.mark.parametrize("grid", list(ALL_GRIDS), ids=list(ALL_GRIDS))
@pytest.mark.parametrize("axis", [0, 1, 2], ids=["x", "y", "z"])
def test_probe_sits_on_its_boundary(grid, axis):
    g = ALL_GRIDS[grid]
    probes = G.z_probes(g) if axis == 2 else G.axis_probes(g, axis)
    labels = [q.label for q in probes]
    if axis < 2:
        N = g.dim[axis]
        must = ["first_kept", "band_mid", "band_top", "s_ge_0", "last_kept", "s_ge_N", "nan", "+inf", "-inf", "s_1e20"]
        assert set(must) <= set(labels), labels
        by = {q.label: q for q in probes}
        assert by["first_kept"].keep and by["first_kept"].idx == 0 and not by["first_kept"].n_keep
        assert by["band_mid"].keep and by["band_mid"].idx == 0
        assert by["band_top"].keep and by["band_top"].idx == 0 and by["s_ge_0"].keep and by["s_ge_0"].idx == 0
        assert by["last_kept"].keep and by["last_kept"].idx == N - 1 and not by["last_kept"].n_keep
        assert not by["s_ge_N"].keep and by["s_ge_N"].idx >= N and by["s_ge_N"].n_keep and by["s_ge_N"].n_idx == N - 1
        for k in {1, N // 2, N - 1}:
            if 1 <= k <= N - 1:
                assert by[f"edge_{k}"].idx == k and by[f"edge_{k}"].n_idx < k          # k - 1, or less where floats are 2 apart
                assert by[f"below_edge_{k}"].idx < k and by[f"below_edge_{k}"].n_idx == k
        # the band's lower end is as close to -1 as fp32 gets where the offset is 0: s = nextafter(-1, 0)
        ego = np.array([[g.interior(0), g.interior(1), g.interior(2)]], np.float32)
        ego[0, axis] = by["first_kept"].p
        assert g.scaled(ego)[0, axis] > -1.0
        if g.res[axis] in (0.25, 0.5, 1.0):                    # exact scale: s = -1 and s = N are reached exactly
            assert "s_eq_-1" in labels
            assert by["s_ge_N"].exact == float(N) or float(np.float32(N)) != N     # N itself is a float up to 2^24
        if g.res[axis] in (0.25, 0.5, 1.0) and g.off[axis] == 0:
            assert g.scaled(ego)[0, axis] == np.nextafter(np.float32(-1), np.float32(0))
    else:
        by = {q.label: q for q in probes}
        assert by["z_lo"].keep and not by["z_lo"].n_keep and not by["z_lo_below"].keep and by["z_lo_above"].keep
        assert by["z_hi"].keep and not by["z_hi"].n_keep and not by["z_hi_above"].keep and by["z_hi_below"].keep
        assert by["z_lo"].exact == float(g.z_lo) and by["z_hi"].exact == float(g.z_hi)
    for q in probes:
        ego = np.array([[g.interior(0), g.interior(1), g.interior(2)]], np.float32)
        ego[0, axis] = q.p
        idx, keep = g.indices(ego)
        assert bool(keep[0]) == q.keep, q
        if q.idx is not None:
            assert int(idx[0, axis]) == q.idx, q
        if q.step:
            ego[0, axis] = np.nextafter(q.p, np.float32(np.inf * q.step), dtype=np.float32)
            idx, keep = g.indices(ego)
            assert bool(keep[0]) == q.n_keep, q
            if q.n_idx is not None:
                assert int(idx[0, axis]) == q.n_idx, q
            assert q.n_keep != q.keep or q.n_idx != q.idx, q               # the neighbour is across the boundary


CASES = {**{f"boundary-{n}": (lambda n=n: G.boundary_case(ALL_GRIDS[n])) for n in ALL_GRIDS},
         **{f"runs-h{h}-{p}": (lambda h=h, p=p: G.run_case(h, p)) for h in G.RUN_HS for p in ("alt", "mixed")}}


@pytest.mark.parametrize("name", list(CASES), ids=list(CASES))
def test_case_places_its_probes_and_torch_agrees(name):
    case = CASES[name]()
    frames = 2
    ego = case.ego(frames)
    idx, keep, pillar, s = case.oracle(frames)
    t_ego, t_idx, t_keep = G.torch_chain(case, frames)
    n_pts = idx.reshape(frames, -1, 3).shape[1]
    assert np.array_equal(t_ego, ego, equal_nan=True)
    assert np.array_equal(t_keep.reshape(frames, n_pts), keep.reshape(frames, n_pts))
    spec = np.isfinite(s) & (np.abs(s.astype(np.float64)) < G.INT64_EDGE)
    t_idx = t_idx.reshape(idx.shape)
    assert np.array_equal(t_idx[spec], idx[spec])
    if name.startswith("boundary"):
        g = case.grid
        # camera 0 at depth 1 carries the x probes on its columns and the y probes on its rows; camera 1 the z probes on its depths
        xs, ys, zs = G.axis_probes(g, 0), G.axis_probes(g, 1), G.z_probes(g)
        assert case.d[0] == 1.0
        fu, fv = np.isfinite(case.u), np.isfinite(case.v)
        at1 = ego[0, 0, 0][np.ix_(fv, fu)]                            # camera 0, depth 1, finite rows and columns
        assert np.array_equal(at1[..., 0], np.broadcast_to(case.u[fu], at1.shape[:2]))
        assert np.array_equal(at1[..., 1], np.broadcast_to(case.v[fv, None], at1.shape[:2]))
        zp = np.array([q.p for q in zs], np.float32)
        fz = np.abs(zp) < 1e30                                        # u d overflows at the largest depths
        assert np.array_equal(ego[0, 1, 1:1 + len(zs), 0, 0, 2][fz], zp[fz])
        for i, q in enumerate(xs):
            row = [j for j, y in enumerate(ys) if y.label == "interior"][0]
            assert bool(keep[0, 0, 0, row, i]) == q.keep, q
        for j, q in enumerate(ys):
            col = [i for i, x in enumerate(xs) if x.label == "interior"][0]
            assert bool(keep[0, 0, 0, j, col]) == q.keep, q
        for k, q in enumerate(zs):
            assert bool(keep[0, 1, 1 + k, 0, 0]) == q.keep, q
        assert keep.any() and (~keep).any()
    else:
        h = case.v.size
        ev = G.boundary_events(pillar)
        if name.endswith("alt"):
            # every row boundary hosts a change, valid -> masked, masked -> valid and no change; from row 2 on also a return to
            # an earlier pillar and a masked gap inside a run (A, -1, A)
            for k in ("change", "valid_to_masked", "masked_to_valid", "no_change"):
                assert ev[k][1:].all(), (k, ev[k])
            for k in ("return", "gap"):
                assert ev[k][2:].all(), (k, ev[k])
        elif h >= 8:
            assert all(ev[k].any() for k in ev), {k: ev[k].any() for k in ev}
        assert (pillar >= 0).any()


def test_run_cases_cover_every_row_boundary():
    """Across the run-pattern cases, every row boundary 1..h-1 of every h hosts every event (returns and gaps from row 2)."""
    for h in G.RUN_HS:
        total = None
        for p in ("alt", "mixed"):
            ev = G.boundary_events(G.run_case(h, p).oracle(2)[2])
            total = ev if total is None else {k: total[k] | ev[k] for k in ev}
        for k, v in total.items():
            lo = 2 if k in ("return", "gap") else 1
            assert v[lo:].all(), (h, k, v)


@pytest.mark.parametrize("item", G.pivot_intrinsics(), ids=lambda it: it[0])
def test_pivot_intrinsics_force_their_pivot_order(item):
    from oracle import lift_oracle as O
    name, K, claim = item
    comb, _ = O.compose_calibration_explicit(K[None], G.pivot_extrinsics(1))
    if claim == "singular":
        assert np.linalg.matrix_rank(K.astype(np.float64)) < 3
        assert not np.isfinite(comb).all()
    elif claim == "nonfinite":
        assert not np.isfinite(K).all()                      # the result may still be finite: 1 / inf = 0
    else:
        assert G.pivot_sequence(K) == claim
        assert np.isfinite(comb).all()


def test_pivot_intrinsics_cover_every_order_and_the_ties():
    items = G.pivot_intrinsics()
    seqs = {claim for _, _, claim in items if isinstance(claim, tuple)}
    assert {(p0, p1) for p0 in range(3) for p1 in (1, 2)} <= seqs
    by = {name: K for name, K, _ in items}
    for name in ("tie0-pos-first", "tie0-neg-first"):
        col = np.abs(by[name][:, 0])
        assert (col == col.max()).sum() == 2 and G.pivot_sequence(by[name])[0] == int(np.argmax(col))
