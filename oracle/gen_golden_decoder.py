"""Pin oracle/decoder_oracle.py against the REAL reference ``Decoder``.  Dev container only.

Run from the repo root:   FIERY_REFERENCE=<a wayveai/fiery checkout> python oracle/gen_golden_decoder.py

The reference's ``Decoder`` (64 channels, 2 classes, with and without future flow) and the oracle's are built, the reference's state
dict is loaded into the oracle, and on seeded (2, 2, 64, 16, 16) inputs:
  1. the state_dict keys must be identical;
  2. every output, the input gradient and every parameter gradient must be bit-equal in train and in eval mode, and so must the
     running statistics after the train step -- a mismatch aborts.
The decoder's state dict is ~11 MB, so no golden file is written: the pin is this script's run.
"""
from __future__ import annotations

import os
import sys

import torch
import torchvision.models.resnet as tv_resnet

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import decoder_oracle as DO  # noqa: E402
from oracle.gen_golden import import_reference  # noqa: E402


def step(model, x, train):
    model.train(train)
    x = x.clone().requires_grad_(True)
    out = model(x)
    loss = sum((v.double() * (i + 1)).sum() for i, v in enumerate(t for t in out.values() if t is not None))
    loss.backward()
    res = {f"out.{k}": v.detach() for k, v in out.items() if v is not None}
    res["gx"] = x.grad
    res.update({f"grad.{n}": p.grad for n, p in model.named_parameters()})
    res.update({f"buf.{n}": b.clone() for n, b in model.named_buffers()})
    model.zero_grad(set_to_none=True)
    return res


def main():
    import_reference()
    # the reference calls resnet18(pretrained=False, ...); torchvision releases without that keyword take weights=None
    real_resnet18 = tv_resnet.resnet18
    tv_resnet.resnet18 = lambda pretrained=False, **kw: real_resnet18(weights=None, **kw)
    import fiery.models.decoder as ref_decoder
    ref_decoder.resnet18 = tv_resnet.resnet18
    for flow in (False, True):
        torch.manual_seed(0)
        ref = ref_decoder.Decoder(64, 2, flow).double()
        ora = DO.Decoder(64, 2, flow).double()
        assert list(ref.state_dict()) == list(ora.state_dict()), "state_dict keys differ"
        ora.load_state_dict(ref.state_dict())
        x = torch.randn(2, 2, 64, 16, 16, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
        for train in (True, False):
            a, b = step(ref, x, train), step(ora, x, train)
            assert a.keys() == b.keys(), "result keys differ"
            for k in a:
                assert torch.equal(a[k], b[k]), f"flow={flow} train={train}: {k} differs"
        print(f"decoder oracle pinned (predict_future_flow={flow}): {len(a)} tensors bit-equal in train and eval")


if __name__ == "__main__":
    main()
