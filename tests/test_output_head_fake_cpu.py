"""The output-head operator's fake implementations: the shapes and dtypes the real operator returns, without a GPU."""
from __future__ import annotations

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

import fiery_b200.decoder  # noqa: F401  (registers torch.ops.fiery_b200.output_head)
from fiery_b200 import decoder as dec
from oracle import decoder_oracle as DO


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_output_head_fake_shapes(dtype):
    with FakeTensorMode():
        y = torch.empty(15, 64, 200, 200, dtype=dtype, device="cuda")
        w1, b1 = torch.empty(2, 64, 1, 1, device="cuda"), torch.empty(2, device="cuda")
        bw, bb = torch.empty(64, device="cuda"), torch.empty(64, device="cuda")
        out, mean, var = torch.ops.fiery_b200.output_head(y, w1, b1, bw, bb, None, None, True, 1e-5)
        assert out.shape == (15, 2, 200, 200) and out.dtype == torch.float32
        assert mean.shape == var.shape == (64,)
        need = [True, False, True, True, False]
        g = torch.ops.fiery_b200.output_head_backward(out, y, mean, var, w1, b1, bw, bb, True, 1e-5, need)
        assert [tuple(t.shape) for t in g] == [(15, 64, 200, 200), (0,), (64,), (2, 64, 1, 1), (0,)]
        assert g[0].dtype == dtype


def test_module_reason_covers_reference_heads_only():
    for n, sig in ((2, False), (1, True)):
        assert dec.module_reason(DO.output_head(64, n, sig)) is None
    head = DO.output_head(64, 2)
    head[1] = torch.nn.SyncBatchNorm(64)
    assert "SyncBatchNorm" in dec.module_reason(head)
    head = DO.output_head(64, 9)
    assert "9 outputs" in dec.module_reason(head)
    head = DO.output_head(64, 2)
    head[2] = torch.nn.GELU()
    assert "GELU" in dec.module_reason(head)


def test_install_swaps_each_head_keys_unchanged():
    from fiery_b200 import install

    class Model(torch.nn.Module):
        def __init__(self, flow):
            super().__init__()
            self.decoder = DO.Decoder(64, 2, flow)
    for flow in (False, True):
        m = Model(flow)
        keys = list(m.state_dict())
        install.use_tensor_core_output_heads(m)
        names = [h for h in install._OUTPUT_HEADS if getattr(m.decoder, h, None) is not None]
        assert len(names) == (4 if flow else 3)
        assert all(isinstance(getattr(m.decoder, h), dec.FusedOutputHead) for h in names)
        assert list(m.state_dict()) == keys
        install.use_tensor_core_output_heads(m)                 # a second call does nothing
        assert all(isinstance(getattr(m.decoder, h), dec.FusedOutputHead) for h in names)
