"""CPU: the host path the tensor-core layers share -- the weight-pack cache (fiery_b200/_lib.py: ``packed``) with a counting pack
function, the depth layer's pack after its weight is replaced, and the schemas of the convolution operators (fiery_b200/ops.py)."""
import pytest
import torch
import torch.nn as nn

from fiery_b200 import _lib, ops  # noqa: F401  (registers the operators)


@pytest.fixture(autouse=True)
def _empty_cache():
    _lib._pack_cache.clear()
    yield
    _lib._pack_cache.clear()


def _counting_pack():
    """a pack function that records its calls; the pack of (a list of) weights is their concatenation times (1 + sum(args))"""
    calls = []

    def pack(weights, *args):
        calls.append(args)
        ws = [weights] if isinstance(weights, torch.Tensor) else weights
        return torch.cat([w.detach().flatten() for w in ws]) * (1 + sum(args))
    return pack, calls


def test_a_pack_is_made_once_per_weight_version():
    pack, calls = _counting_pack()
    w = nn.Parameter(torch.randn(4, 3))
    a = _lib.packed(pack, w)
    assert _lib.packed(pack, w) is a and len(calls) == 1
    with torch.no_grad():
        w.mul_(2.0)                                          # an optimizer step bumps the version
    b = _lib.packed(pack, w)
    assert len(calls) == 2 and torch.equal(b, w.detach().flatten())
    assert _lib.packed(pack, w) is b and len(calls) == 2
    v = _lib.packed(pack, w.view(12))                         # same address, another shape
    assert len(calls) == 3 and torch.equal(v, b)
    ws = [torch.randn(2), torch.randn(3)]                    # a list of weights: an update of any one re-makes the pack
    c = _lib.packed(pack, ws, 1)
    assert _lib.packed(pack, ws, 1) is c and len(calls) == 4
    ws[1].add_(1.0)
    assert torch.equal(_lib.packed(pack, ws, 1), torch.cat(ws) * 2) and len(calls) == 5


def test_a_replaced_weight_is_repacked():
    """Each new weight gets its own pack, even where the old weight is freed first and its address could be handed out again."""
    pack, calls = _counting_pack()
    for i in range(3 * _lib._PACK_CACHE_SIZE):               # past the bound, so evicted entries release their weights' memory
        w = torch.full((64,), float(i))
        assert torch.equal(_lib.packed(pack, w), w)
        del w
    assert len(calls) == 3 * _lib._PACK_CACHE_SIZE


def test_entries_are_per_pack_function_and_args():
    pack1, calls1 = _counting_pack()
    pack2, calls2 = _counting_pack()
    w = torch.randn(5)
    a, b, c = _lib.packed(pack1, w, 1), _lib.packed(pack1, w, 2), _lib.packed(pack2, w, 1)
    assert torch.equal(a, w * 2) and torch.equal(b, w * 3) and torch.equal(c, w * 2) and c is not a
    assert _lib.packed(pack1, w, 1) is a and _lib.packed(pack1, w, 2) is b and _lib.packed(pack2, w, 1) is c
    assert len(calls1) == 2 and len(calls2) == 1


def test_least_recently_used_entry_is_evicted_at_the_bound():
    pack, calls = _counting_pack()
    n = _lib._PACK_CACHE_SIZE
    ws = [torch.full((1,), float(i)) for i in range(n + 1)]
    first = [_lib.packed(pack, w) for w in ws[:n]]
    assert len(calls) == n and len(_lib._pack_cache) == n
    assert _lib.packed(pack, ws[0]) is first[0]              # a hit makes ws[0] the most recently used
    _lib.packed(pack, ws[n])                                 # one more entry evicts the least recently used: ws[1]
    assert len(calls) == n + 1 and len(_lib._pack_cache) == n
    assert _lib.packed(pack, ws[0]) is first[0] and len(calls) == n + 1
    assert _lib.packed(pack, ws[1]) is not first[1] and len(calls) == n + 2


def test_depth_layer_pack_follows_a_replaced_weight():
    """A new weight Parameter may land at the freed address of the old one with the same version count; its pack must still be its
    own."""
    from fiery_b200.depth_layer import DepthLayer, pack_weight
    layer = DepthLayer(112)
    stale = 0
    for _ in range(20):
        layer._packed_weight(torch.float16)
        layer.weight = nn.Parameter(torch.empty(0))           # the old weight is freed
        layer.weight = nn.Parameter(torch.randn(112, 128, 1, 1))
        stale += not torch.equal(layer._packed_weight(torch.float16), pack_weight(layer.weight, torch.float16))
    assert stale == 0


def test_convolution_operator_schemas():
    want = {
        "first_conv": "fiery_b200::first_conv(Tensor x, Tensor weight) -> Tensor",
        "first_conv_backward": "fiery_b200::first_conv_backward(Tensor grad_y, Tensor x, Tensor weight, bool need_input, "
                               "bool need_weight) -> (Tensor, Tensor)",
        "causal_conv3d": "fiery_b200::causal_conv3d(Tensor x, Tensor weight) -> Tensor",
        "causal_conv3d_backward": "fiery_b200::causal_conv3d_backward(Tensor grad_y, Tensor x, Tensor weight, bool need_input, "
                                  "bool need_weight) -> (Tensor, Tensor)",
        "temporal_entry": "fiery_b200::temporal_entry(Tensor x, Tensor[] weights, Tensor? extra) -> Tensor[]",
        "temporal_entry_backward": "fiery_b200::temporal_entry_backward(Tensor[] grads, Tensor x, Tensor[] weights, Tensor? extra, "
                                   "bool need_input, bool need_weight) -> (Tensor, Tensor[])",
    }
    for name, schema in want.items():
        assert str(getattr(torch.ops.fiery_b200, name).default._schema) == schema
