"""Pin oracle/warp_oracle.py against the REAL reference (fiery/utils/geometry.py:82-253) and write tests/golden/warp.npz.
Needs a wayveai/fiery checkout in FIERY_REFERENCE.  Run from the repo root: python oracle/gen_golden_warp.py"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
for name, attr in (("pyquaternion", "Quaternion"), ("efficientnet_pytorch", "EfficientNet")):
    if name not in sys.modules:
        m = types.ModuleType(name)
        setattr(m, attr, object)
        sys.modules[name] = m
if not os.path.isdir(os.path.join(os.environ.get("FIERY_REFERENCE", ""), "fiery")):
    raise SystemExit("set FIERY_REFERENCE to a wayveai/fiery checkout")
sys.path.insert(0, os.environ["FIERY_REFERENCE"])
from fiery.utils import geometry as R  # noqa: E402
from oracle import warp_oracle as W  # noqa: E402
from fiery_b200.synthetic import make_egomotion  # noqa: E402


def main():
    torch.manual_seed(0)
    out = {}
    for tag, (b, t, c, h, w), extent in (("small", (2, 3, 5, 12, 16), (50.0, 50.0)), ("rect", (1, 4, 3, 20, 10), (50.0, 25.0)),
                                          ("bev", (1, 3, 8, 200, 200), (50.0, 50.0))):
        x = torch.randn(b, t, c, h, w)
        flow = torch.from_numpy(make_egomotion(b, t, seed=3))
        ref = R.cumulative_warp_features(x.clone(), flow, mode="bilinear", spatial_extent=extent)
        got = W.cumulative_warp_features(x.clone(), flow, mode="bilinear", spatial_extent=extent)
        assert torch.equal(ref, got), tag
        assert torch.equal(R.pose_vec2mat(flow), W.pose_vector_to_matrix(flow))
        m = R.pose_vec2mat(flow)
        assert torch.equal(R.mat2pose_vec(m), W.matrix_to_pose_vector(m))
        one = R.warp_features(x[:, 0], flow[:, 0], mode="bilinear", spatial_extent=extent)
        assert torch.equal(one, W.warp_features(x[:, 0], flow[:, 0], mode="bilinear", spatial_extent=extent))
        xg = x.clone().requires_grad_(True)
        gout = torch.randn_like(ref)
        R.cumulative_warp_features(xg.clone(), flow, mode="bilinear", spatial_extent=extent).backward(gout)
        out[f"{tag}__shape"] = np.array([b, t, c, h, w])
        out[f"{tag}__extent"] = np.array(extent, dtype=np.float32)
        out[f"{tag}__flow"] = flow.numpy()
        if tag == "bev":                              # keep the fixture small: seeds + samples
            pick = np.random.default_rng(1).integers(0, ref.numel(), 8192)
            out[f"{tag}__pick"] = pick
            out[f"{tag}__ref_at_pick"] = ref.flatten()[pick].numpy()
            out[f"{tag}__grad_at_pick"] = xg.grad.flatten()[pick].numpy()
            out[f"{tag}__ref_norm"] = np.array([float(ref.double().norm())])
        else:
            out[f"{tag}__x"] = x.numpy()
            out[f"{tag}__gout"] = gout.numpy()
            out[f"{tag}__ref"] = ref.numpy()
            out[f"{tag}__grad"] = xg.grad.numpy()
        print("ok", tag)
    path = os.path.join(ROOT, "tests", "golden", "warp.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
