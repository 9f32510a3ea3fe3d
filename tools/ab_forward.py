#!/usr/bin/env python
"""A/B harness for experiment builds (FIERY_NVCC_EXTRA=-DFIERY_COLS_AB): times every unit shape of the column tile kernel
and every layout pass on one workload, checks each against the default variant, writes gpurun_out/ab.json."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from fiery_b200 import _lib
from fiery_b200.geometry import _stream_ptr
from fiery_b200.lift import LiftSplat
from fiery_b200.synthetic import CONFIGS, make_calibration, make_head

wl = sys.argv[1] if len(sys.argv) > 1 else "cfg2_static_lss_b8"
variants = [int(v) for v in (sys.argv[2].split(",") if len(sys.argv) > 2 else "0,2".split(","))]
cfg = CONFIGS[wl]
dev = torch.device("cuda:0")
lib = _lib.load()
K, E = make_calibration(cfg, seed=100)
head = torch.from_numpy(make_head(cfg, seed=100)).to(dev)
K_d, E_d = torch.from_numpy(K).to(dev), torch.from_numpy(E).to(dev)
lift = LiftSplat.from_config(cfg).to(dev)
c = lift._constants(dev)
X, Y = cfg.bev_hw
F = cfg.frames
flush = torch.empty((256 << 20) // 4, dtype=torch.float32, device=dev)
stream = _stream_ptr(dev)


def timed(fn, n=20):
    ts = []
    for _ in range(n):
        flush.fill_(1.0)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.mean(ts)) * 1e3, float(np.min(ts)) * 1e3


PLAN = lift.plan(K_d, E_d)       # caller-owned plan: the timings below are the tile kernel (+ layout pass) alone


def runner(layout, out, scratch):
    desc = lift._desc(c, F, cfg.n_cameras, torch.float32, _lib.CALIB_RAW, layout)
    def run():
        _lib.check(lib.fiery_lift_forward(desc, head.data_ptr(), K_d.data_ptr(), E_d.data_ptr(), c["u"].data_ptr(), c["v"].data_ptr(),
                                          c["d"].data_ptr(), out.data_ptr(), scratch.data_ptr(), PLAN.data_ptr(), stream), "fwd")
    return run, desc


res = {"workload": wl, "tile": {}, "layout_pass": {}}
ref = None
acc = torch.zeros((F, X, Y, cfg.out_channels), dtype=torch.float32, device=dev)
_d_nhwc = lift._desc(c, F, cfg.n_cameras, torch.float32, _lib.CALIB_RAW, _lib.BEV_NHWC)
run_nhwc, _ = runner(_lib.BEV_NHWC, acc, torch.zeros(max(1, int(lib.fiery_lift_scratch_bytes(_d_nhwc)) // 4), dtype=torch.float32, device=dev))
for v in variants:
    os.environ["FIERY_COLS_VARIANT"] = str(v)
    try:
        acc.zero_()
        run_nhwc()
        torch.cuda.synchronize()
        out = acc.clone()
        if ref is None:
            ref = out
        err = float((out - ref).norm() / ref.norm())
        for _ in range(3):
            run_nhwc()
        mean, mn = timed(run_nhwc)
        res["tile"][v] = {"us_mean": mean, "us_min": mn, "rel_err_vs_v0": err}
    except Exception as e:  # noqa
        res["tile"][v] = {"error": str(e)[:200]}
    print("tile", v, res["tile"][v], flush=True)

best = min((v for v in res["tile"] if "us_mean" in res["tile"][v] and res["tile"][v]["rel_err_vs_v0"] < 1e-5), key=lambda v: res["tile"][v]["us_mean"])
res["best_tile"] = best
out_nchw = torch.empty((F, cfg.out_channels, X, Y), dtype=torch.float32, device=dev)
ref_nchw = ref.permute(0, 3, 1, 2)
combos = os.environ.get("AB_COMBOS", "1:132 2:132 4:132").split()
from fiery_b200.synthetic import make_grad_bev
gout = torch.from_numpy(make_grad_bev(cfg, seed=100)).to(dev)
for combo in combos:
    chains, min_tiles = (int(x) for x in combo.split(":"))
    os.environ["FIERY_COLS_VARIANT"] = "-1"
    os.environ["FIERY_CHAINS"] = str(chains)
    os.environ["FIERY_CHAIN_MIN_TILES"] = str(min_tiles)
    run, desc = runner(_lib.BEV_NCHW, out_nchw, None)
    scratch = torch.zeros(int(lib.fiery_lift_scratch_bytes(desc)) // 4, dtype=torch.float32, device=dev)
    run, desc = runner(_lib.BEV_NCHW, out_nchw, scratch)
    out_nchw.fill_(float("nan"))
    run(); torch.cuda.synchronize()
    err = float((out_nchw - ref_nchw).norm() / ref_nchw.norm())
    clean = bool((scratch == 0).all().item())
    for _ in range(3):
        run()
    mean, mn = timed(run)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        sp = s.cuda_stream
        def run_s():
            _lib.check(lib.fiery_lift_forward(desc, head.data_ptr(), K_d.data_ptr(), E_d.data_ptr(), c["u"].data_ptr(), c["v"].data_ptr(),
                                              c["d"].data_ptr(), out_nchw.data_ptr(), scratch.data_ptr(), PLAN.data_ptr(), sp), "fwd")
        run_s(); torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            run_s()
    torch.cuda.current_stream().wait_stream(s)
    out_nchw.fill_(float("nan"))
    gmean, gmn = timed(g.replay)
    torch.cuda.synchronize()
    err2 = float((out_nchw - ref_nchw).norm() / ref_nchw.norm())
    clean2 = bool((scratch == 0).all().item())
    # backward (eager, through the host layer: workspace allocation + re-layout + tile kernel)
    gh = lift._launch_backward(head, K_d, E_d, gout)
    if combo == combos[0]:
        gh_ref = gh.clone()
    berr = float((gh - gh_ref).norm() / gh_ref.norm())
    for _ in range(3):
        lift._launch_backward(head, K_d, E_d, gout)
    bmean, bmn = timed(lambda: lift._launch_backward(head, K_d, E_d, gout))
    res["layout_pass"][combo] = {"us_mean": mean, "graph_us_mean": gmean, "graph_us_min": gmn, "rel_err": max(err, err2),
                                 "scratch_clean": clean and clean2, "launches": int(lib.fiery_lift_forward_launches(desc)),
                                 "bwd_us_mean": bmean, "bwd_rel_err_vs_first": berr}
    print("chains:min_tiles", combo, res["layout_pass"][combo], flush=True)
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
with open(os.path.join(ROOT, "gpurun_out", f"ab_{wl}.json"), "w") as fh:
    json.dump(res, fh, indent=1)
