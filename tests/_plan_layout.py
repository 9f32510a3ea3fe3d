"""A decoder of the geometry plan's bytes (layout: fiery_b200/csrc/lift_plan.cuh) back to one pillar per frustum point, shared by
the tests that read plans.  The record size, the counts offset and the touched maps' offset are the host layer's own
(fiery_b200/lift.py); decoding plans against the oracle pins them and the field offsets below."""
import numpy as np

from fiery_b200.lift import _PLAN_OFF_COUNTS as OFF_COUNTS, _PLAN_TILE_BYTES as TILE_BYTES, _plan_touched_offset

PAIRS, RG, ND, STREAMS, MAX_ROWS = 192, 4, 4, 64, 32
CAP = PAIRS * MAX_ROWS
OFF_MASK, OFF_OFF, OFF_SOFF = 0, PAIRS * 4, PAIRS * 4 + PAIRS * 2
OFF_RUNS = OFF_COUNTS + 16
OFF_STREAMS = OFF_RUNS + CAP * 4


def _decode(plan: np.ndarray, cfg):
    """plan bytes -> (pillar per point (B', n, D, h, w) int32, list of per-tile dicts, touched (B', X*Y) uint8).  ``cfg`` needs
    feat_hw, depth_bins, n_cameras, frames and bev_hw (a fiery_b200.synthetic.LiftConfig, or any object with those fields)."""
    h, w = cfg.feat_hw
    D, n, B = cfg.depth_bins, cfg.n_cameras, cfg.frames
    n_wt = (w + 3) // 4
    n_tiles = B * n * n_wt
    X, Y = cfg.bev_hw
    dense = np.full((B, n, D, h, w), -2, dtype=np.int32)
    tiles = []
    for t in range(n_tiles):
        rec = plan[t * TILE_BYTES:(t + 1) * TILE_BYTES]
        mask = rec[OFF_MASK:OFF_MASK + PAIRS * 4].view(np.uint32)
        off = rec[OFF_OFF:OFF_OFF + PAIRS * 2].view(np.uint16)
        soff = rec[OFF_SOFF:OFF_SOFF + STREAMS * 2].view(np.uint16)
        n_runs, n_stream = rec[OFF_COUNTS:OFF_COUNTS + 8].view(np.uint32)
        runs = rec[OFF_RUNS:OFF_RUNS + CAP * 4].view(np.int32)
        streams = rec[OFF_STREAMS:OFF_STREAMS + (CAP + 2 * STREAMS) * 4].view(np.int32)
        img, wt = divmod(t, n_wt)
        f, cam = divmod(img, n)
        per_pair = np.empty((PAIRS, h), dtype=np.int32)
        for pair in range(PAIRS):
            k = 0
            for row in range(h):
                if row and (int(mask[pair]) >> row) & 1:
                    k += 1
                per_pair[pair, row] = runs[int(off[pair]) + k]
            assert int(mask[pair]) >> h == 0 and not int(mask[pair]) & 1
        for d in range(D):
            for c in range(4):
                if wt * 4 + c < w:
                    dense[f, cam, d, :, wt * 4 + c] = per_pair[d * 4 + c]
        tiles.append(dict(mask=mask.copy(), off=off.copy(), soff=soff.copy(), n_runs=int(n_runs), n_stream=int(n_stream),
                          runs=runs, streams=streams, per_pair=per_pair))
    t0 = _plan_touched_offset(B, n, w)
    touched = plan[t0:t0 + B * X * Y].reshape(B, X * Y)
    return dense, tiles, touched


def assert_tile_streams(t, h):
    """A decoded tile's run list is tight and its backward streams list, per (row group, column, slot), the run containing the
    group's first row followed by the runs that start inside the group, depth group after depth group, then two pads."""
    assert t["n_runs"] == PAIRS + sum(bin(int(m)).count("1") for m in t["mask"])
    total = 0
    for s in range(STREAMS):
        rg, col, j = s >> 4, (s >> 2) & 3, s & 3
        r_lo, r_hi = (h * rg) // RG, (h * (rg + 1)) // RG
        want_s = []
        for g in range(48 // ND):
            row_p = t["per_pair"][(g * ND + j) * 4 + col]
            want_s.append(int(row_p[min(r_lo, h - 1)]) if r_lo < h else int(row_p[h - 1]))
            for row in range(r_lo + 1, r_hi):
                if (int(t["mask"][(g * ND + j) * 4 + col]) >> row) & 1:
                    want_s.append(int(row_p[row]))
        want_s += [-1, -1]
        got = t["streams"][int(t["soff"][s]):int(t["soff"][s]) + len(want_s)].tolist()
        assert got == want_s, (s, got[:8], want_s[:8])
        total += len(want_s)
    assert t["n_stream"] == total
