#!/usr/bin/env python
"""Small ncu target: runs only the launches to be captured, through the C ABI.
    python tools/ncu_target.py <workload> tile    # the column tile kernel alone (channel-last target), whole batch, 4 launches
    python tools/ncu_target.py <workload> tile_planned   # the same with a caller-owned geometry plan (planned variant of the kernel)
    python tools/ncu_target.py <workload> step    # the NCHW step (tile kernels + layout passes of every frame group), 4 calls
    python tools/ncu_target.py <workload> warp_bwd      # backward of cumulative_warp_features (3, 3, 64, X, Y): the gather adjoint, 3 calls
    python tools/ncu_target.py <workload> step_warped   # lift with the warp folded into the layout pass (finalize_warp_kernel), 3 calls
    python tools/ncu_target.py <workload> bwd     # NCHW backward (re-layout + backward tile kernel), 3 calls
    python tools/ncu_target.py <workload> depth   # the wgmma depth_layer (fp16 features -> fp32 head tensor) at the workload's size, 4 calls
    python tools/ncu_target.py <workload> conv    # the wgmma first BEV convolution on a channel-last BEV of the workload's size, 4 calls
"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from fiery_b200 import _lib
from fiery_b200.geometry import _stream_ptr
from fiery_b200.lift import LiftSplat
from fiery_b200.synthetic import CONFIGS, make_calibration, make_grad_bev, make_head

wl, mode = sys.argv[1], sys.argv[2]
cfg = CONFIGS[wl]
dev = torch.device("cuda:0")
lib = _lib.load()
K, E = make_calibration(cfg, seed=100)
head = torch.from_numpy(make_head(cfg, seed=100)).to(dev)
K_d, E_d = torch.from_numpy(K).to(dev), torch.from_numpy(E).to(dev)
lift = LiftSplat.from_config(cfg).to(dev)
c = lift._constants(dev)
X, Y = cfg.bev_hw
if mode == "depth":
    from fiery_b200.depth_layer import depth_layer_forward, pack_weight as pack_depth
    fh, fw = cfg.feat_hw
    feat = torch.randn(cfg.frames * cfg.n_cameras, 128, fh, fw, device=dev).half()
    w = torch.randn(cfg.head_channels, 128, 1, 1, device=dev) * 0.05
    b = torch.randn(cfg.head_channels, device=dev)
    wp = pack_depth(w, torch.float16)
    for _ in range(4):
        depth_layer_forward(feat, w, b, wp)
elif mode == "conv":
    from fiery_b200.bev_conv import first_conv_forward, pack_weight
    xb = torch.randn(cfg.frames, X, Y, 64, device=dev).permute(0, 3, 1, 2)
    wp = pack_weight(torch.randn(64, 64, 7, 7, device=dev) * 0.02)
    for _ in range(4):
        first_conv_forward(xb, wp)
elif mode == "warp_bwd":
    from fiery_b200.synthetic import make_egomotion
    from fiery_b200.warp import cumulative_warp_features
    fl = torch.from_numpy(make_egomotion(3, 3, seed=7)).to(dev)
    xw = torch.randn(3, 3, 64, X, Y, device=dev, requires_grad=True)
    g = torch.randn(3, 3, 64, X, Y, device=dev)
    for _ in range(3):
        xw.grad = None
        cumulative_warp_features(xw, fl, mode="bilinear", spatial_extent=(float(cfg.x_bound[1]), float(cfg.y_bound[1]))).backward(g)
elif mode == "step_warped":
    from fiery_b200.synthetic import make_egomotion
    seq = 3 if cfg.frames % 3 == 0 else 2
    fl = torch.from_numpy(make_egomotion(cfg.frames // seq, seq, seed=11)).to(dev)
    for _ in range(3):
        lift.forward_warped(head, K_d, E_d, fl, (float(cfg.x_bound[1]), float(cfg.y_bound[1])))
elif mode == "bwd":
    g = torch.from_numpy(make_grad_bev(cfg, seed=100)).to(dev)
    for _ in range(3):
        lift._launch_backward(head, K_d, E_d, g)
else:
    layout = _lib.BEV_NHWC if mode.startswith("tile") else _lib.BEV_NCHW
    plan = lift.plan(K_d, E_d) if mode == "tile_planned" else None
    desc = lift._desc(c, cfg.frames, cfg.n_cameras, torch.float32, _lib.CALIB_RAW, layout)
    out = torch.zeros((cfg.frames, X, Y, cfg.out_channels) if mode.startswith("tile") else (cfg.frames, cfg.out_channels, X, Y), device=dev)
    scratch = torch.zeros(max(1, int(lib.fiery_lift_scratch_bytes(desc)) // 4), dtype=torch.float32, device=dev)
    for _ in range(4):
        _lib.check(lib.fiery_lift_forward(desc, head.data_ptr(), K_d.data_ptr(), E_d.data_ptr(), c["u"].data_ptr(), c["v"].data_ptr(),
                                          c["d"].data_ptr(), out.data_ptr(), scratch.data_ptr(), plan.data_ptr() if plan is not None else None, _stream_ptr(dev)), "fwd")
torch.cuda.synchronize()
