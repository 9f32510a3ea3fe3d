"""Pin oracle/future_oracle.py against the REAL reference classes and write tests/golden/future_prediction.npz.  Dev container only.

Run from the repo root:   FIERY_REFERENCE=<a wayveai/fiery checkout> python oracle/gen_golden_future.py

For a small FuturePrediction (8 hidden, 4 latent channels, 3 GRUs with 3 Bottlenecks each, 3 steps on a 4 x 4 map) and for one
SpatialGRU with a non-zero gru_bias_init, the reference's classes and the oracle's are built, the reference's state dict is loaded
into the oracle, and:
  1. the state_dict keys must be identical;
  2. outputs, the input and state gradients and every parameter gradient must be bit-equal in train and in eval mode on seeded
     inputs, and so must the running statistics after the train step -- a mismatch aborts;
  3. the state dict, inputs and the reference's results are written so tests/test_future_oracle_cpu.py holds the same pin on a
     machine without the reference.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import future_oracle as FO  # noqa: E402
from oracle.gen_golden import import_reference  # noqa: E402

GRID = (4, 4)
B, T = 2, 3


def step(model, x, h0, gout, train):
    """One forward + backward: {y, gx, gh0, grad.<param>, buf.<buffer>}."""
    model.train(train)
    x = x.clone().requires_grad_(True)
    h0 = h0.clone().requires_grad_(True)
    y = model(x, h0)
    y.backward(gout)
    out = {"y": y.detach(), "gx": x.grad, "gh0": h0.grad}
    for n, p in model.named_parameters():
        out[f"grad.{n}"] = p.grad
    for n, b in model.named_buffers():
        out[f"buf.{n}"] = b.clone()
    model.zero_grad(set_to_none=True)
    return out


def cases():
    from fiery.layers.temporal import SpatialGRU
    from fiery.models.future_prediction import FuturePrediction
    torch.manual_seed(0)
    yield "future", FuturePrediction(8, 4), FO.FuturePrediction(8, 4), (B, T, 4, *GRID), (B, 8, *GRID), (B, T, 8, *GRID)
    yield "gru", SpatialGRU(5, 6, gru_bias_init=0.25), FO.SpatialGRU(5, 6, gru_bias_init=0.25), (B, T, 5, *GRID), (B, 6, *GRID), \
        (B, T, 6, *GRID)


def main():
    import_reference()
    golden = {}
    for name, ref, ora, xshape, hshape, gshape in cases():
        ref_sd, ora_sd = ref.state_dict(), ora.state_dict()
        if list(ref_sd) != list(ora_sd):
            raise SystemExit(f"{name}: state_dict keys differ:\n{sorted(set(ref_sd) ^ set(ora_sd))}")
        for bn in ref.modules():                                  # non-trivial BN statistics, then the same state in both
            if isinstance(bn, torch.nn.BatchNorm2d):
                bn.weight.data.uniform_(0.5, 1.5)
                bn.bias.data.uniform_(-0.2, 0.2)
                bn.running_mean.uniform_(-0.1, 0.1)
                bn.running_var.uniform_(0.5, 1.5)
        sd = {k: v.clone() for k, v in ref.state_dict().items()}
        g = torch.Generator().manual_seed(1)
        x, h0, gout = torch.randn(xshape, generator=g), torch.randn(hshape, generator=g), torch.randn(gshape, generator=g)
        for train in (True, False):
            ref.load_state_dict(sd)
            ora.load_state_dict(sd)
            want, got = step(ref, x, h0, gout, train), step(ora, x, h0, gout, train)
            for k in want:
                if not torch.equal(want[k], got[k]):
                    raise SystemExit(f"{name} {'train' if train else 'eval'}: {k} differs")
            for k, v in want.items():
                golden[f"{name}__{'train' if train else 'eval'}__{k}"] = v.numpy()
        for k, v in sd.items():
            golden[f"{name}__sd__{k}"] = v.numpy()
        golden[f"{name}__x"], golden[f"{name}__h0"], golden[f"{name}__gout"] = x.numpy(), h0.numpy(), gout.numpy()
        print(f"{name}: keys identical, train and eval bit-equal")
    path = os.path.join(ROOT, "tests", "golden", "future_prediction.npz")
    np.savez_compressed(path, **golden)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
