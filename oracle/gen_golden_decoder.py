"""Pin oracle/decoder_oracle.py against the REAL reference ``Decoder``.  Dev container only.

Run from the repo root:   FIERY_REFERENCE=<a wayveai/fiery checkout> python oracle/gen_golden_decoder.py

The reference's ``Decoder`` (64 channels, 2 classes, with and without future flow) and the oracle's are built, the reference's state
dict is loaded into the oracle, and on seeded (2, 2, 64, 16, 16) inputs:
  1. the state_dict keys must be identical;
  2. every output, the input gradient and every parameter gradient must be bit-equal in train and in eval mode, and so must the
     running statistics after the train step -- a mismatch aborts.
The decoder's state dict is ~11 MB, so the whole decoder is pinned by this script's run only.  Its four output heads are small at
16 channels (``shared_out_channels = in_channels``), so the script also writes tests/golden/decoder_heads.npz from a reference
``Decoder(16, 3, True)``: per head its state dict, a seeded input and grad_out, and in train and in eval the output, the input and
parameter gradients and the buffers after the step (``head_step``), each first checked bit-equal against the oracle's
``output_head``.  tests/test_decoder_oracle_cpu.py holds ``output_head`` to that file.
"""
from __future__ import annotations

import os
import sys

import numpy as np
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


HEADS = (("segmentation_head", 3, False), ("instance_offset_head", 2, False), ("instance_center_head", 1, True),
         ("instance_future_head", 2, False))
HEAD_CHANNELS = 16
HEAD_INPUT = (2, HEAD_CHANNELS, 4, 6)


def head_step(head, x, gout, train):
    """One forward + backward of an output head: {out, gx, grad.<param>, buf.<buffer>}."""
    head.train(train)
    x = x.clone().requires_grad_(True)
    out = head(x)
    out.backward(gout)
    res = {"out": out.detach(), "gx": x.grad}
    res.update({f"grad.{n}": p.grad for n, p in head.named_parameters()})
    res.update({f"buf.{n}": b.clone() for n, b in head.named_buffers()})
    head.zero_grad(set_to_none=True)
    return res


def heads_golden(ref_decoder):
    """tests/golden/decoder_heads.npz from the reference's Decoder(16, 3, True), each head checked against the oracle's first"""
    torch.manual_seed(2)
    ref = ref_decoder.Decoder(HEAD_CHANNELS, 3, True)
    golden = {}
    for name, n_out, sigmoid in HEADS:
        head = getattr(ref, name)
        with torch.no_grad():                                   # non-trivial norm parameters and running statistics
            bn = head[1]
            bn.weight.uniform_(0.5, 1.5), bn.bias.uniform_(-0.2, 0.2)
            bn.running_mean.uniform_(-0.1, 0.1), bn.running_var.uniform_(0.5, 1.5)
        ora = DO.output_head(HEAD_CHANNELS, n_out, sigmoid)
        sd = {k: v.clone() for k, v in head.state_dict().items()}
        assert list(sd) == list(ora.state_dict()), f"{name}: state_dict keys differ"
        g = torch.Generator().manual_seed(len(golden) + 1)
        x = torch.randn(HEAD_INPUT, generator=g)
        gout = torch.randn((HEAD_INPUT[0], n_out) + HEAD_INPUT[2:], generator=g)
        for train in (True, False):
            head.load_state_dict(sd)
            ora.load_state_dict(sd)
            want, got = head_step(head, x, gout, train), head_step(ora, x, gout, train)
            assert want.keys() == got.keys(), f"{name}: result keys differ"
            for k in want:
                assert torch.equal(want[k], got[k]), f"{name} train={train}: {k} differs"
                golden[f"{name}__{'train' if train else 'eval'}__{k}"] = want[k].numpy()
        for k, v in sd.items():
            golden[f"{name}__sd__{k}"] = v.numpy()
        golden[f"{name}__x"], golden[f"{name}__gout"] = x.numpy(), gout.numpy()
    path = os.path.join(ROOT, "tests", "golden", "decoder_heads.npz")
    np.savez_compressed(path, **golden)
    print(f"output heads pinned: wrote {path} ({os.path.getsize(path)} bytes)")


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
    heads_golden(ref_decoder)


if __name__ == "__main__":
    main()
