"""CPU: the forward lift's launch plan -- passes, frame groups, scratch lanes -- is host logic (lift_fwd.cu: lift_chunk_frames,
lift_forward_groups, lane_layout, scratch_frames), so fiery_lift_scratch_bytes and fiery_lift_forward_launches answer without a
device.  A scratch sized too small would make the tile kernels reduce past its end on the GPU; this module catches that here, by
walking every pass and frame group of a call and checking that each group's slice fits the scratch the library asks for."""
import pytest

from fiery_b200 import _lib

# mirror of fiery_b200/csrc/lift_fwd.cu (constants and the three functions above)
SCRATCH_CAP = 1 << 30           # accumulator + marks of one pass
MAX_CHAINS = 4                  # frame groups of a pass
MAX_LANES = 2                   # scratch slices (and streams) the groups run on
CHAIN_MIN_TILES = 132           # tiles a frame group keeps at least: one per SM of an H100 SXM
C = 64


def chunk_frames(n_frames, pillars, forced=0):
    """Frames per pass: as many as fit SCRATCH_CAP, or the test hook's cap when that is smaller."""
    c = SCRATCH_CAP // (pillars * C * 4 + pillars)
    if 0 < forced < c:
        c = forced
    return max(1, min(c, n_frames))


def forward_groups(frames_in_pass, tiles_per_frame, nchw=True):
    """Frame groups of one pass: at most MAX_CHAINS, each with at least CHAIN_MIN_TILES tiles; channel-last output has one."""
    if not nchw:
        return 1
    g = min(frames_in_pass, MAX_CHAINS)
    while g > 1 and (frames_in_pass // g) * tiles_per_frame < CHAIN_MIN_TILES:
        g -= 1
    return max(g, 1)


def group_bounds(frames_in_pass, groups):
    return [(frames_in_pass * g // groups, frames_in_pass * (g + 1) // groups) for g in range(groups)]


def lane_layout(frames_in_pass, tiles_per_frame, nchw=True):
    """(group bounds, lane of every group, first scratch frame of every lane, scratch frames of the pass)."""
    groups = forward_groups(frames_in_pass, tiles_per_frame, nchw)
    lanes = min(groups, MAX_LANES)
    bounds = group_bounds(frames_in_pass, groups)
    slice0, frames = [], 0
    for lane in range(lanes):
        slice0.append(frames)
        frames += max(s1 - s0 for s0, s1 in bounds[lane::lanes])
    return bounds, [g % lanes for g in range(groups)], slice0, frames


def passes(n_frames, chunk):
    return [(f0, min(chunk, n_frames - f0)) for f0 in range(0, n_frames, chunk)]


def scratch_frames(n_frames, tiles_per_frame, pillars, forced=0):
    """Scratch frames a call needs: the largest pass's lane slices.  Every pass is looked at, not just the first and the last."""
    chunk = chunk_frames(n_frames, pillars, forced)
    return max(lane_layout(nf, tiles_per_frame)[3] for _, nf in passes(n_frames, chunk))


def forward_launches(n_frames, tiles_per_frame, pillars, nchw=True, forced=0):
    """(tile kernel [+ layout pass]) per frame group, over every pass."""
    if n_frames == 0:
        return 0
    chunk = chunk_frames(n_frames, pillars, forced)
    return sum((2 if nchw else 1) * forward_groups(nf, tiles_per_frame, nchw) for _, nf in passes(n_frames, chunk))


def scratch_bytes(frames, pillars):
    return frames * pillars * C * 4 + (frames * pillars + 127) // 128 * 128


# tiles per frame -> (cameras, feat_w): tiles = cameras * ceil(feat_w / 4)
TILE_SHAPES = {4: (1, 16), 45: (3, 60), 90: (6, 60), 132: (6, 88), 133: (7, 76), 300: (6, 200)}
# (bev_x, bev_y): a grid whose pass holds the whole call, and one where SCRATCH_CAP cuts a pass at 4 frames
GRIDS = [(200, 200), (1024, 1000)]


def _desc(frames, tiles, grid, layout):
    cams, w = TILE_SHAPES[tiles]
    d = _lib.LiftDesc()
    d.n_frames, d.n_cameras, d.depth_bins, d.channels, d.feat_h, d.feat_w = frames, cams, 48, C, 28, w
    d.bev_x, d.bev_y, d.bev_z = grid[0], grid[1], 1
    d.bev_layout = layout
    return d


def test_mirror_reproduces_the_documented_examples():
    """The mirror itself, on cases worked out by hand: 8 frames of 90 tiles are 4 groups of 2 frames on 2 lanes (4 scratch frames);
    a pass capped at 8 of 15 frames leaves a tail of 7 frames cut into groups of 2, 2 and 3 -- lane 0 holds the 3-frame group, so the
    tail needs 3 + 2 = 5 scratch frames, more than the full pass's 4."""
    assert lane_layout(8, 90) == ([(0, 2), (2, 4), (4, 6), (6, 8)], [0, 1, 0, 1], [0, 2], 4)
    assert lane_layout(7, 90) == ([(0, 2), (2, 4), (4, 7)], [0, 1, 0], [0, 3], 5)
    assert scratch_frames(15, 90, 200 * 200, forced=8) == 5
    assert forward_launches(15, 90, 200 * 200, forced=8) == 2 * (4 + 3)
    assert chunk_frames(40, 1024 * 1000) == 4
    assert forward_groups(1, 4) == 1 and forward_groups(2, 132) == 2 and forward_groups(9, 90) == 4 and forward_groups(8, 90, False) == 1


@pytest.mark.parametrize("grid", GRIDS, ids=lambda g: f"{g[0]}x{g[1]}")
@pytest.mark.parametrize("forced", [0, 1, 2, 3, 7, 8])
def test_scratch_and_launches_match_the_mirror(forced, grid):
    """fiery_lift_scratch_bytes and fiery_lift_forward_launches over frames 0..40, tiles per frame {4, 45, 90, 132, 133, 300}, with
    the pass cap of the test hook forced or not; and every frame group of every pass fits the scratch the library sizes: its lane's
    slice starts where the lanes before it end, and slice + group frames stay within the scratch frames."""
    lib = _lib.load()
    pillars = grid[0] * grid[1]
    lib.fiery_lift_set_max_chunk_frames(forced)
    try:
        for tiles in TILE_SHAPES:
            for frames in range(41):
                where = dict(frames=frames, tiles=tiles, forced=forced)
                nchw = _desc(frames, tiles, grid, _lib.BEV_NCHW)
                nhwc = _desc(frames, tiles, grid, _lib.BEV_NHWC)
                assert lib.fiery_lift_forward_launches(nchw) == forward_launches(frames, tiles, pillars, True, forced), where
                assert lib.fiery_lift_forward_launches(nhwc) == forward_launches(frames, tiles, pillars, False, forced), where
                assert lib.fiery_lift_scratch_bytes(nhwc) == 0, where            # channel-last output reduces into the output itself
                got = lib.fiery_lift_scratch_bytes(nchw)
                if frames == 0:
                    assert got == 0, where
                    continue
                want = scratch_frames(frames, tiles, pillars, forced)
                assert got == scratch_bytes(want, pillars), (where, got, want)
                # the launcher's use of the scratch, group by group
                sized = got // (pillars * C * 4)
                for _, nf in passes(frames, chunk_frames(frames, pillars, forced)):
                    bounds, lane_of, slice0, _ = lane_layout(nf, tiles)
                    for (s0, s1), lane in zip(bounds, lane_of):
                        end = slice0[lane] + (s1 - s0)
                        assert end <= sized, (where, nf, (s0, s1), lane, sized)
                        assert lane + 1 == len(slice0) or end <= slice0[lane + 1], (where, nf, (s0, s1), lane, slice0)
    finally:
        lib.fiery_lift_set_max_chunk_frames(0)


def test_tail_pass_larger_than_a_full_pass_is_sized_for_the_tail():
    """15 frames of 90 tiles in passes of at most 8: the full pass needs 4 scratch frames, the 7-frame tail 5."""
    lib = _lib.load()
    d = _desc(15, 90, (200, 200), _lib.BEV_NCHW)
    lib.fiery_lift_set_max_chunk_frames(8)
    try:
        assert lib.fiery_lift_scratch_bytes(d) == scratch_bytes(5, 200 * 200)
        assert lib.fiery_lift_forward_launches(d) == 14
    finally:
        lib.fiery_lift_set_max_chunk_frames(0)
