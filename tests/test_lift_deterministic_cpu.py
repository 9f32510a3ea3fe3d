"""CPU: the deterministic forward's workspace and pass split are host logic (lift_fwd.cu: det_layout), so
fiery_lift_deterministic_workspace_bytes answers without a device, and the argument checks of fiery_lift_forward_deterministic reject a
bad call before anything is launched.  A workspace sized too small would make the tile kernel store partial sums past its end on the
GPU; this module walks every pass of a call and checks that its plan, partial sums, accumulator and index fit the workspace."""
import pytest

from fiery_b200 import _lib
from fiery_b200.lift import _PLAN_TILE_BYTES
from fiery_b200.synthetic import CONFIGS
from tests.test_lift_launch_plan_cpu import passes

# mirror of fiery_b200/csrc/lift_fwd.cu: det_layout
PASS_CAP = 1 << 30               # workspace of one pass, as the default path's scratch
PLAN_PAIRS = 192                 # (depth, column) pairs of a tile; a pair has at most one run per image row
C = 64


def _a(n, m=256):
    return (n + m - 1) // m * m


def det_layout(n_frames, cams, feat_w, feat_h, pillars, nchw, forced=0):
    """(frames per pass, {region: (offset, bytes)}, total bytes)."""
    tpf = cams * ((feat_w + 3) // 4)
    rows = tpf * PLAN_PAIRS * feat_h
    per_frame = tpf * _PLAN_TILE_BYTES + pillars + rows * C * 4 + (pillars * C * 4 if nchw else 0) + pillars * 8 + rows * 4
    f = PASS_CAP // per_frame
    if 0 < forced < f:
        f = forced
    f = max(1, min(f, n_frames))
    sizes = [("plan", f * tpf * _PLAN_TILE_BYTES + _a(f * pillars, 128)), ("partials", f * rows * C * 4),
             ("accum", f * pillars * C * 4 if nchw else 0), ("start", f * pillars * 4), ("cursor", f * pillars * 4),
             ("lists", f * rows * 4)]
    regions, off = {}, 0
    for name, b in sizes:
        regions[name] = (off, b)
        off += _a(b)
    return f, regions, off


def _desc(frames, cams, w, h, bev, layout, depth=48):
    d = _lib.LiftDesc()
    d.n_frames, d.n_cameras, d.depth_bins, d.channels, d.feat_h, d.feat_w = frames, cams, depth, C, h, w
    d.bev_x, d.bev_y, d.bev_z = bev[0], bev[1], 1
    for a in range(3):
        d.bev_resolution[a] = 1.0
    d.bev_layout = layout
    return d


def _bench_shapes():
    out = {}
    for name in ("cfg2_static_lss", "cfg3_baseline", "cfg4_pon"):
        cfg = CONFIGS[name]
        h, w = cfg.feat_hw
        out[name] = (cfg.n_cameras, w, h, cfg.bev_hw)
    out["h32-w200"] = (6, 200, 32, (200, 200))          # the largest tile count and row count of the launch-plan tests
    out["tiny"] = (1, 16, 8, (50, 49))
    return out


def test_mirror_on_the_reference_shape():
    """6 cameras, 28 x 60 features, 200 x 200 BEV: 483 840 possible runs (= frustum points) per frame, 124 MB of partial sums; a pass
    holds 7 frames of plan + partials + accumulator + index under 1 GiB."""
    f, regions, total = det_layout(40, 6, 60, 28, 200 * 200, True)
    assert regions["partials"][1] == 7 * 483840 * 256
    assert f == 7 and total <= PASS_CAP
    assert det_layout(40, 6, 60, 28, 200 * 200, True, forced=3)[0] == 3


@pytest.mark.parametrize("forced", [0, 1, 2, 3, 7])
@pytest.mark.parametrize("shape", list(_bench_shapes()), ids=list(_bench_shapes()))
def test_workspace_matches_the_mirror_and_every_pass_fits(shape, forced):
    lib = _lib.load()
    cams, w, h, bev = _bench_shapes()[shape]
    pillars = bev[0] * bev[1]
    tpf = cams * ((w + 3) // 4)
    lib.fiery_lift_set_max_chunk_frames(forced)
    try:
        for layout in (_lib.BEV_NCHW, _lib.BEV_NHWC):
            for frames in range(41):
                where = dict(shape=shape, forced=forced, layout=layout, frames=frames)
                got = lib.fiery_lift_deterministic_workspace_bytes(_desc(frames, cams, w, h, bev, layout))
                if frames == 0:
                    assert got == 0, where
                    continue
                f, regions, total = det_layout(frames, cams, w, h, pillars, layout == _lib.BEV_NCHW, forced)
                assert got == total, (where, got, total)
                assert f <= frames and (forced == 0 or f <= forced), where
                for _, nf in passes(frames, f):
                    rows = nf * tpf * PLAN_PAIRS * h
                    need = {"plan": nf * tpf * _PLAN_TILE_BYTES + nf * pillars, "partials": rows * C * 4,
                            "accum": nf * pillars * C * 4 if layout == _lib.BEV_NCHW else 0, "start": nf * pillars * 4,
                            "cursor": nf * pillars * 4, "lists": rows * 4}
                    for name, b in need.items():
                        off, size = regions[name]
                        assert b <= size and off + size <= got, (where, nf, name)
                if f > 1:                                                  # the cap only cuts where one pass would not fit
                    assert total <= PASS_CAP, where
    finally:
        lib.fiery_lift_set_max_chunk_frames(0)


def _call(desc, head=16, bev=16, ws=16, theta=0, copy_mask=0):
    lib = _lib.load()
    return lib.fiery_lift_forward_deterministic(desc, head, 16, 16, 16, 16, 16, bev, ws, 0, theta, copy_mask, 0)


def test_argument_checks_need_no_device():
    """Rejected before any launch: a bad descriptor, a NULL workspace, the warped lift with channel-last output, half a warp."""
    good = _desc(2, 6, 60, 28, (200, 200), _lib.BEV_NCHW)
    bad = _desc(2, 0, 60, 28, (200, 200), _lib.BEV_NCHW)
    assert _call(bad) == -1 and b"n_cameras" in _lib.load().fiery_last_error()
    assert _call(good, ws=0) == -1 and b"workspace" in _lib.load().fiery_last_error()
    assert _call(good, head=0) == -1
    nhwc = _desc(2, 6, 60, 28, (200, 200), _lib.BEV_NHWC)
    assert _call(nhwc, theta=16, copy_mask=16) == -1 and b"NCHW" in _lib.load().fiery_last_error()
    assert _call(good, theta=16) == -1
    assert _call(_desc(2, 6, 60, 28, (200, 200), _lib.BEV_NCHW, depth=49)) == -1
    assert _call(_desc(0, 6, 60, 28, (200, 200), _lib.BEV_NCHW), ws=0) == 0               # nothing to do


def test_voxels_summing_workspace_and_checks():
    lib = _lib.load()
    assert lib.fiery_voxels_summing_deterministic_workspace_bytes(0, 64) == 0
    assert lib.fiery_voxels_summing_deterministic_workspace_bytes(1, 64) == 2 * 64 * 4
    assert lib.fiery_voxels_summing_deterministic_workspace_bytes(4_200_000, 1) == (4_200_000 + 63) // 64 * 2 * 4
    assert lib.fiery_voxels_summing_forward_deterministic(10, 64, 64, 16, 16, 16, 3, 16, 16, 0, 0) == -1
    assert b"workspace" in lib.fiery_last_error()
    assert lib.fiery_voxels_summing_forward_deterministic(10, 64, 32, 16, 16, 16, 3, 16, 16, 16, 0) == -1
