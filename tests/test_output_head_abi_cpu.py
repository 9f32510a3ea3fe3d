"""The output head's C ABI (fiery_output_head_*) rejects every argument outside its limits before any device work, with a message
naming the field, and its size queries return 0 for a rejected shape.  No GPU: a call that got past its checks would fail on the
missing device with a CUDA message instead, and a size query touches no device at all."""
from __future__ import annotations

import ctypes

import pytest

from fiery_b200 import _lib
from fiery_b200 import decoder as dec

E_INVALID = -1
SIZE_QUERIES = ("fiery_output_head_packed_bytes", "fiery_output_head_forward_workspace_bytes",
                "fiery_output_head_backward_workspace_bytes")
A, B = 4096, 4100                 # a 16-byte aligned and a misaligned fake address: no call below gets far enough to use them


def _desc(**kw):
    d = dec.desc(2, 8, 8, 16, 2, True, 1e-5)
    for k, v in kw.items():
        setattr(d, k, v)
    return d


# (field overrides, a fragment of the message)
BAD_DESCS = [
    ({"maps": 0}, b"maps = 0"),
    ({"maps": -3}, b"maps = -3"),
    ({"channels": 0}, b"channels = 0"),
    ({"channels": 129}, b"channels = 129"),
    ({"n_out": 0}, b"n_out = 0"),
    ({"n_out": 9}, b"n_out = 9"),
    ({"grid_x": 0}, b"grid_x = 0"),
    ({"grid_y": -1}, b"grid_y = -1"),
    ({"grid_x": 3, "grid_y": 5}, b"multiple of 4"),
    ({"grid_x": 7, "grid_y": 9}, b"multiple of 4"),
    ({"grid_x": 65536, "grid_y": 32768}, b"must be < 2^31"),
    ({"grid_x": 2 ** 31 - 1, "grid_y": 4}, b"must be < 2^31"),
    ({"training": 2}, b"training = 2"),
    ({"training": -1}, b"training = -1"),
    ({"eps": -1e-7}, b"eps"),
    ({"eps": float("nan")}, b"eps"),
    ({"eps": float("-inf")}, b"eps"),
    ({"maps": 1, "grid_x": 1, "grid_y": 1}, b"multiple of 4"),
]


def _entry_calls(d):
    """each entry point with this desc and otherwise valid-looking arguments: (name, rc)"""
    lib = _lib.load()
    yield "pack", lib.fiery_output_head_pack_weights(d, A, A, None)
    yield "forward", lib.fiery_output_head_forward(d, A, A, A, A, A, A, A, A, A, A, None)
    yield "backward", lib.fiery_output_head_backward(d, A, A, A, A, A, A, A, A, A, A, A, A, A, None)


@pytest.mark.parametrize("fields,msg", BAD_DESCS, ids=[f"{'_'.join(f'{k}{v}' for k, v in f.items())}" for f, _ in BAD_DESCS])
def test_bad_desc_rejected_everywhere(fields, msg):
    d = _desc(**fields)
    lib = _lib.load()
    for name in SIZE_QUERIES:
        assert getattr(lib, name)(d) == 0, name
    for name, rc in _entry_calls(d):
        assert rc == E_INVALID, name
        assert msg in lib.fiery_last_error(), (name, lib.fiery_last_error())


def test_null_desc_rejected():
    lib = _lib.load()
    for name in SIZE_QUERIES:
        assert getattr(lib, name)(None) == 0
    for name, rc in _entry_calls(None):
        assert rc == E_INVALID and b"NULL desc" in lib.fiery_last_error(), name


@pytest.mark.parametrize("training", [1, 0])
def test_limits_accepted_by_the_size_queries(training):
    # the edges inside the limits: every size query answers, with no device
    lib = _lib.load()
    for fields in ({"channels": 1, "n_out": 1}, {"channels": 128, "n_out": 8}, {"maps": 1, "grid_x": 1, "grid_y": 4},
                   {"grid_x": 46340, "grid_y": 46340}, {"eps": 0.0}):
        d = _desc(training=training, **fields)
        for name in SIZE_QUERIES:
            assert getattr(lib, name)(d) > 0, (name, fields)


# (argument index in the forward's pointer list y, packed, bn_w, bn_b, running_mean, running_var, out, mean, var, workspace; the value;
#  a fragment of the message)
FORWARD_BAD = [
    (0, 0, b"NULL pointer"), (1, 0, b"NULL pointer"), (6, 0, b"NULL pointer"), (7, 0, b"NULL pointer"), (8, 0, b"NULL pointer"),
    (9, 0, b"NULL pointer"), (0, B, b"aligned"), (1, B, b"aligned"), (6, B, b"aligned"), (9, B, b"aligned"),
]


@pytest.mark.parametrize("i,value,msg", FORWARD_BAD)
def test_forward_rejects_pointers(i, value, msg):
    lib = _lib.load()
    ptrs = [A] * 10
    ptrs[i] = value
    assert lib.fiery_output_head_forward(_desc(), *ptrs, None) == E_INVALID
    assert msg in lib.fiery_last_error()


@pytest.mark.parametrize("which", [4, 5])
def test_eval_forward_needs_running_statistics(which):
    lib = _lib.load()
    ptrs = [A] * 10
    ptrs[which] = 0
    assert lib.fiery_output_head_forward(_desc(training=0), *ptrs, None) == E_INVALID
    assert b"running_mean and running_var" in lib.fiery_last_error()


# backward pointers: grad_out, y, mean, var, w1, bn_w, bn_b, grad_y, grad_bn_w, grad_bn_b, grad_w, grad_b, workspace
BACKWARD_BAD = [
    (0, 0, b"NULL pointer"), (1, 0, b"NULL pointer"), (2, 0, b"NULL pointer"), (3, 0, b"NULL pointer"), (4, 0, b"NULL pointer"),
    (12, 0, b"NULL pointer"), (0, B, b"aligned"), (1, B, b"aligned"), (7, B, b"aligned"), (12, B, b"aligned"),
]


@pytest.mark.parametrize("i,value,msg", BACKWARD_BAD)
def test_backward_rejects_pointers(i, value, msg):
    lib = _lib.load()
    ptrs = [A] * 13
    ptrs[i] = value
    assert lib.fiery_output_head_backward(_desc(), *ptrs, None) == E_INVALID
    assert msg in lib.fiery_last_error()


@pytest.mark.parametrize("w,packed,msg", [(0, A, b"NULL weight"), (A, 0, b"NULL weight"), (A, B, b"aligned")])
def test_pack_rejects_pointers(w, packed, msg):
    lib = _lib.load()
    assert lib.fiery_output_head_pack_weights(_desc(), w, packed, None) == E_INVALID
    assert msg in lib.fiery_last_error()


def test_desc_mirror_matches_the_header():
    # six int32 fields, then the double: 24 + 8 bytes
    assert ctypes.sizeof(_lib.OutputHeadDesc) == 32 and _lib.OutputHeadDesc.eps.offset == 24
