"""CPU: the lift's C-ABI entry points reject a head shape or dtype their tile kernels are not built for before anything is launched,
so these calls need no device (the pointers are dummies that are never dereferenced).  Every entry point that runs the tile kernels
must reject the same shapes with a message that names the field; a 0-frame call does nothing and succeeds whatever the shape; the plan
size, which does not depend on the tile kernels, answers for any shape."""
import pytest

from fiery_b200 import _lib

P = 16          # a dummy non-NULL device pointer
E_INVALID = -1  # FIERY_E_INVALID (include/fiery_b200.h)


def _desc(**kw):
    d = _lib.LiftDesc()
    d.n_frames, d.n_cameras, d.depth_bins, d.channels, d.feat_h, d.feat_w = 2, 6, 48, 64, 28, 60
    d.bev_x, d.bev_y, d.bev_z = 200, 200, 1
    for a in range(3):
        d.bev_resolution[a] = 1.0
    d.head_dtype = _lib.DTYPE_F32
    d.bev_layout = _lib.BEV_NCHW
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _forward(lib, d):
    return lib.fiery_lift_forward(d, P, P, P, P, P, P, P, P, 0, 0)


def _forward_warped(lib, d):
    return lib.fiery_lift_forward_warped(d, P, P, P, P, P, P, P, P, 0, P, P, 0)


def _forward_deterministic(lib, d):
    return lib.fiery_lift_forward_deterministic(d, P, P, P, P, P, P, P, P, 0, 0, 0, 0)


def _backward(lib, d):
    return lib.fiery_lift_backward(d, P, P, P, P, P, P, P, P, P, 0, 0)


ENTRIES = {"forward": _forward, "forward_warped": _forward_warped, "forward_deterministic": _forward_deterministic,
           "backward": _backward}
BAD = {"channels": dict(channels=32), "depth_bins": dict(depth_bins=49), "feat_w": dict(feat_w=62), "feat_h": dict(feat_h=33),
       "dtype": dict(head_dtype=7)}


@pytest.mark.parametrize("field", list(BAD))
@pytest.mark.parametrize("entry", list(ENTRIES))
def test_unsupported_head_is_rejected_and_named(entry, field):
    lib = _lib.load()
    assert ENTRIES[entry](lib, _desc(**BAD[field])) == E_INVALID
    assert field.encode() in lib.fiery_last_error()


def test_backward_rejects_a_half_precision_head():
    lib = _lib.load()
    assert _backward(lib, _desc(head_dtype=_lib.DTYPE_F16)) == E_INVALID
    assert b"dtype" in lib.fiery_last_error()


@pytest.mark.parametrize("field", list(BAD))
@pytest.mark.parametrize("entry", list(ENTRIES))
def test_zero_frames_succeed_whatever_the_shape(entry, field):
    assert ENTRIES[entry](_lib.load(), _desc(n_frames=0, **BAD[field])) == 0


@pytest.mark.parametrize("field", ["channels", "feat_w"])
def test_plan_size_does_not_depend_on_the_tile_shape(field):
    """The plan records pillar runs per (depth, column) pair and row: channels and the column pitch do not enter it."""
    assert _lib.load().fiery_lift_plan_bytes(_desc(**BAD[field])) > 0
