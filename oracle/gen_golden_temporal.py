"""Pin oracle/temporal_oracle.py against the REAL reference classes and write tests/golden/temporal.npz.  Dev container only.

Run from the repo root:   FIERY_REFERENCE=<a wayveai/fiery checkout> python oracle/gen_golden_temporal.py

For a small TemporalModel (14 -> 8 channels, a block with a projection and pyramid pooling like the first block of baseline.yml,
then 8 -> 8, on a 4 x 4 map) and for one TemporalBlock without pyramid pooling, the reference's classes and the oracle's are built, the reference's state dict is loaded into the
oracle, and:
  1. the state_dict keys must be identical;
  2. outputs, the input gradient and every parameter gradient must be bit-equal in train and in eval mode on seeded inputs, and so
     must the running statistics after the train step -- a mismatch aborts;
  3. the state dict, inputs and the reference's results are written so tests/test_temporal_oracle_cpu.py holds the same pin on a
     machine without the reference.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REFERENCE = os.environ.get("FIERY_REFERENCE", "")

from oracle import temporal_oracle as TO  # noqa: E402
from oracle.gen_golden import import_reference  # noqa: E402

GRID = (4, 4)


def _step(model, x, gout, train):
    model.train(train)
    x = x.clone().requires_grad_(True)
    y = model(x)
    y.backward(gout)
    out = {"y": y.detach(), "gx": x.grad}
    for n, p in model.named_parameters():
        out[f"grad.{n}"] = p.grad
    for n, b in model.named_buffers():
        out[f"buf.{n}"] = b.clone()
    model.zero_grad(set_to_none=True)
    return out


def cases():
    from fiery.layers.temporal import TemporalBlock
    from fiery.models.temporal_model import TemporalModel
    torch.manual_seed(0)
    yield "model", TemporalModel(14, 3, GRID, start_out_channels=8), TO.TemporalModel(14, 3, GRID, start_out_channels=8), \
        (2, 3, 14, *GRID), (2, 1, 8, *GRID)
    yield "block", TemporalBlock(8, 8), TO.TemporalBlock(8, 8), (2, 8, 3, *GRID), (2, 8, 3, *GRID)


def main():
    import_reference()
    golden = {}
    for name, ref, ora, xshape, gshape in cases():
        ref_sd, ora_sd = ref.state_dict(), ora.state_dict()
        if list(ref_sd) != list(ora_sd):
            raise SystemExit(f"{name}: state_dict keys differ:\n{sorted(set(ref_sd) ^ set(ora_sd))}")
        for bn in ref.modules():                                  # non-trivial BN statistics, then the same state in both
            if isinstance(bn, torch.nn.BatchNorm3d):
                bn.weight.data.uniform_(0.5, 1.5)
                bn.bias.data.uniform_(-0.2, 0.2)
                bn.running_mean.uniform_(-0.1, 0.1)
                bn.running_var.uniform_(0.5, 1.5)
        sd = {k: v.clone() for k, v in ref.state_dict().items()}
        ora.load_state_dict(sd)
        g = torch.Generator().manual_seed(1)
        x = torch.randn(xshape, generator=g)
        gout = torch.randn(gshape, generator=g)
        for train in (True, False):
            ref.load_state_dict(sd)
            ora.load_state_dict(sd)
            want, got = _step(ref, x, gout, train), _step(ora, x, gout, train)
            for k in want:
                if not torch.equal(want[k], got[k]):
                    raise SystemExit(f"{name} {'train' if train else 'eval'}: {k} differs")
            for k, v in want.items():
                golden[f"{name}__{'train' if train else 'eval'}__{k}"] = v.numpy()
        for k, v in sd.items():
            golden[f"{name}__sd__{k}"] = v.numpy()
        golden[f"{name}__x"], golden[f"{name}__gout"] = x.numpy(), gout.numpy()
        print(f"{name}: keys identical, train and eval bit-equal")
    path = os.path.join(ROOT, "tests", "golden", "temporal.npz")
    np.savez_compressed(path, **golden)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
