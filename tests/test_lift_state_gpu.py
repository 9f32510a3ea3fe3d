"""GPU: the lift across repeated calls and through its host entry points, against the fp64 oracle.

The kernels keep state between calls: the pooled scratch (zero on entry, zero again when a call's work completes), a caller-owned
geometry plan, the CUDA graph's own scratch and static inputs, and the thread-local side stream that the frame-group chains fork onto.
Each section drives one of them the way a user does and compares every frame with oracle.lift_exact (fp64 direct pooling) or the
fp64 autograd gradient, at the bars of tests/test_lift_envelope_gpu.py.
  1. Caller-owned plans: a plan made for another (B', n) is rejected before any launch; a plan of this batch reused by several calls.
  2. Graph replay follows in-place writes to its head and calibration, interleaved with eager calls and another graph.
  3. lift_from_host: chunk sequences, caller-supplied output, channels-last modules, fp16 heads, scratch-pool eviction.
  4. Streams: two modules on two streams, and a graph replay beside eager calls on another stream."""
import numpy as np
import pytest
import torch

from fiery_b200 import _lib
from fiery_b200 import lift as lift_mod
from fiery_b200.lift import LiftSplat
from fiery_b200.synthetic import LiftConfig
from oracle import lift_oracle as O
from tests.test_lift_envelope_gpu import (_ORACLE, ROUTE_ODD, ROUTE_TMA, _assert_bev, _assert_grad, _assert_scratch_clean, _exact,
                                          _exact_grad, _frames, _inputs, _launches)
from tests.test_lift_launch_plan_cpu import forward_groups

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TAG = "state"                   # first element of this module's oracle cache keys
TILES = 90                      # tiles per frame of every configuration here: 6 cameras x 15 column tiles
# ROUTE_TMA on a 100 x 100 grid: a second module with another grid, and the host pipeline's batch (cheaper to compare)
GRID100 = LiftConfig("grid100", n_cameras=6, final_dim=(64, 480), d_bound=(2.0, 50.0, 4.0), x_bound=(-50.0, 50.0, 1.0),
                     y_bound=(-50.0, 50.0, 1.0))
MSG = "another batch shape"


@pytest.fixture(scope="module", autouse=True)
def _oracle_cache():
    yield
    for k in [k for k in _ORACLE if k[0] == TAG]:
        del _ORACLE[k]


def _case(cfg, seed):
    head, K, E, gout = _inputs(cfg, seed)
    return dict(cfg=cfg, seed=seed, head=head, K=K, E=E, gout=gout, hd=head.to(DEV), Kd=K.to(DEV), Ed=E.to(DEV), gd=gout.to(DEV))


def _bev(cfg, seed, head, K, E, comb=None, tag=""):
    """The fp64 BEV of every frame (cached): the raw calibration, or ``comb`` = R @ K^-1 as a calibration="torch" module composes it."""
    key = (TAG, cfg.name, cfg.frames, seed, tag)
    if comb is None:
        return _exact(key, cfg, head, K, E)
    if key not in _ORACLE:
        oracle, n = O.LiftOracle.from_config(cfg), cfg.n_cameras
        _ORACLE[key] = torch.cat([oracle.lift_exact(head[f * n:(f + 1) * n], K[f:f + 1], E[f:f + 1], combined=comb[f:f + 1])
                                  for f in range(K.shape[0])])
    return _ORACLE[key]


def _grad(c, gout=None, tag=""):
    cfg = c["cfg"]
    return _exact_grad((TAG, cfg.name, cfg.frames, c["seed"], "grad" + tag), cfg, c["head"], c["K"], c["E"],
                       c["gout"] if gout is None else gout)


def _assert_frames(got, exact, what):
    got = got.detach().cpu()
    assert got.shape == exact.shape, what
    for f in range(exact.shape[0]):
        _assert_bev(got[f:f + 1], exact[f:f + 1], (what, f))


def _channels_last(g):
    return g.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)


def _pool_entries(stream):
    return [buf for key, buf in lift_mod._scratch._bufs.items() if key[1] == stream.cuda_stream]


# ==== 1. caller-owned plans ======================================================================================================
PLAN_CFG = _frames(ROUTE_TMA, 3)
FOREIGN = ["more_frames", "fewer_frames", "other_cameras", "int8"]


@pytest.fixture(scope="module")
def plan_case():
    """3 frames whose calibrations are the first 3 of a 5-frame rig: the 5-frame plan is the static rig's plan met by a short batch."""
    big = _case(_frames(ROUTE_TMA, 5), seed=11)
    c = _case(PLAN_CFG, seed=11)
    c.update(K5=big["Kd"], E5=big["Ed"], head=big["head"][:3 * 6], K=big["K"][:3], E=big["E"][:3], hd=big["hd"][:3 * 6],
             Kd=big["Kd"][:3], Ed=big["Ed"][:3])
    c["lift"] = LiftSplat.from_config(PLAN_CFG).to(DEV)
    c["lift_cl"] = LiftSplat.from_config(PLAN_CFG, output_layout="channels_last").to(DEV)
    return c


def _foreign_plan(c, which):
    lift = c["lift"]
    if which == "more_frames":
        return lift.plan(c["K5"], c["E5"])
    if which == "fewer_frames":
        return lift.plan(c["K5"][:2], c["E5"][:2])
    if which == "other_cameras":
        return lift.plan(c["Kd"][:, :5], c["Ed"][:, :5])
    return lift.plan(c["Kd"], c["Ed"]).view(torch.int8)


@pytest.mark.parametrize("which", FOREIGN)
def test_foreign_plan_is_rejected_before_any_launch(plan_case, which):
    """Forward (NCHW and NHWC), backward (NCHW and NHWC gradient) and autograd all raise, and leave the scratch pool untouched; the
    next call without a plan is exact."""
    c = plan_case
    lift = c["lift"]
    p = _foreign_plan(c, which)
    lift_mod._scratch.clear()
    try:
        # the rule itself first: without it, the backward's kernels would read a plan made for fewer frames or cameras past its end
        desc, _ = lift._abi_args(DEV, c["Kd"], c["Ed"], torch.float32, _lib.BEV_NCHW)
        with pytest.raises(ValueError, match=MSG):
            LiftSplat._check_plan(p, desc, DEV)
        with torch.no_grad():
            for m in (lift, c["lift_cl"]):
                with pytest.raises(ValueError, match=MSG):
                    m(c["hd"], c["Kd"], c["Ed"], plan=p)
        for g in (c["gd"], _channels_last(c["gd"])):
            with pytest.raises(ValueError, match=MSG):
                lift._launch_backward(c["hd"], c["Kd"], c["Ed"], g, plan=p)
        h = c["hd"].clone().requires_grad_(True)
        with pytest.raises(ValueError, match=MSG):
            lift(h, c["Kd"], c["Ed"], plan=p).backward(c["gd"])
        assert h.grad is None
        assert not lift_mod._scratch._bufs
        with torch.no_grad():
            bev = lift(c["hd"], c["Kd"], c["Ed"])
        _assert_frames(bev, _bev(PLAN_CFG, 11, c["head"], c["K"], c["E"]), which)
        _assert_scratch_clean()
    finally:
        lift_mod._scratch.clear()


def test_plan_rule_checks_size_dtype_and_device(plan_case):
    c = plan_case
    lift = c["lift"]
    p = lift.plan(c["Kd"], c["Ed"])
    desc, _ = lift._abi_args(DEV, c["Kd"], c["Ed"], torch.float32, _lib.BEV_NCHW)
    assert p.numel() == int(_lib.load().fiery_lift_plan_bytes(desc))
    LiftSplat._check_plan(p, desc, DEV)
    LiftSplat._check_plan(None, desc, DEV)
    for bad in (p.cpu(), p[:-1], torch.cat([p, p[:1]]), p.view(torch.int8)):
        with pytest.raises(ValueError, match=MSG):
            LiftSplat._check_plan(bad, desc, DEV)


def test_zero_frame_plan_is_one_byte(plan_case):
    c = plan_case
    lift = c["lift"]
    p0 = lift.plan(c["Kd"][:0], c["Ed"][:0])
    assert p0.numel() == 1 and p0.dtype == torch.uint8
    with torch.no_grad():
        out = lift(c["hd"][:0], c["Kd"][:0], c["Ed"][:0], plan=p0)
        assert tuple(out.shape) == (0, PLAN_CFG.out_channels, *PLAN_CFG.bev_hw)
        with pytest.raises(ValueError, match=MSG):
            lift(c["hd"], c["Kd"], c["Ed"], plan=p0)
        with pytest.raises(ValueError, match=MSG):
            lift(c["hd"][:0], c["Kd"][:0], c["Ed"][:0], plan=lift.plan(c["Kd"], c["Ed"]))


def test_static_rig_plan_reused_across_calls(plan_case):
    """One plan of this batch's calibrations, three calls with new head values each: forward in both layouts, the backward with the
    plan (NCHW and NHWC gradients) and autograd through a caller-owned plan."""
    c = plan_case
    lift, lift_cl = c["lift"], c["lift_cl"]
    p = lift.plan(c["Kd"], c["Ed"])
    snapshot = p.clone()
    try:
        for call in range(3):
            k = _case(PLAN_CFG, seed=20 + call)
            k.update(K=c["K"], E=c["E"], Kd=c["Kd"], Ed=c["Ed"])
            exact = _bev(PLAN_CFG, k["seed"], k["head"], c["K"], c["E"], tag="rig")
            with torch.no_grad():
                _assert_frames(lift(k["hd"], c["Kd"], c["Ed"], plan=p), exact, ("nchw", call))
                _assert_frames(lift_cl(k["hd"], c["Kd"], c["Ed"], plan=p), exact, ("nhwc", call))
            want = _grad(k, tag="rig")
            for g in (k["gd"], _channels_last(k["gd"])):
                _assert_grad(lift._launch_backward(k["hd"], c["Kd"], c["Ed"], g, plan=p), want, ("backward", call))
            h = k["hd"].clone().requires_grad_(True)
            lift(h, c["Kd"], c["Ed"], plan=p).backward(k["gd"])
            _assert_grad(h.grad, want, ("autograd", call))
        torch.cuda.synchronize()
        assert torch.equal(p, snapshot)
        _assert_scratch_clean()
    finally:
        lift_mod._scratch.clear()


# ==== 2. graph replay ============================================================================================================
GRAPHS = {
    "nchw-3groups": dict(cfg=_frames(ROUTE_TMA, 6), launches=2 * 3),
    "channels_last": dict(cfg=_frames(ROUTE_TMA, 2), layout="channels_last"),
    "fallback-3groups": dict(cfg=_frames(ROUTE_ODD, 6), launches=2 * 3),
    "multipass": dict(cfg=_frames(ROUTE_TMA, 5), max_chunk=2, launches=2 * 3),        # passes of 2, 2 and 1 frames
    "fp16": dict(cfg=_frames(ROUTE_TMA, 2), half=True),
    "torch_calibration": dict(cfg=_frames(ROUTE_TMA, 3), calibration="torch"),
}


@pytest.fixture(scope="module")
def other_graph():
    """A graph of another module (100 x 100 grid), replayed between the replays of the graph under test."""
    c = _case(_frames(GRID100, 2), seed=31)
    lift = LiftSplat.from_config(c["cfg"]).to(DEV)
    g = lift.capture(c["hd"], c["Kd"], c["Ed"])
    return dict(lift=lift, g=g, exact=_bev(c["cfg"], 31, c["head"], c["K"], c["E"]))


@pytest.mark.parametrize("static", [False, True], ids=["dynamic", "static"])
@pytest.mark.parametrize("variant", list(GRAPHS))
def test_graph_replay_follows_its_inputs(variant, static, other_graph):
    """Replay; write new head values into the static head with copy_ and replay; for a dynamic graph also write a new rig into the
    static calibrations and replay.  Every replay against the oracle of what its inputs hold; eager calls of the same module and
    replays of another graph in between; the graphs' scratch and the pool all zero afterwards."""
    v = GRAPHS[variant]
    cfg, half, calib = v["cfg"], v.get("half", False), v.get("calibration", "fused")
    layout = v.get("layout", "contiguous")
    lib = _lib.load()
    if "max_chunk" in v:
        lib.fiery_lift_set_max_chunk_frames(v["max_chunk"])
    lift_mod._scratch.clear()
    try:
        lift = LiftSplat.from_config(cfg, output_layout=layout, calibration=calib).to(DEV)
        if "launches" in v:
            assert _launches(lift, cfg.frames, cfg.n_cameras) == v["launches"]
        if variant.endswith("3groups"):
            assert forward_groups(cfg.frames, TILES) == 3
        assert (np.prod(cfg.bev_hw) % 4 != 0) == variant.startswith("fallback")
        a, b = _case(cfg, seed=41), _case(cfg, seed=42)
        for c in (a, b):
            if half:
                c["hd"] = c["hd"].half()
                c["head"] = c["hd"].float().cpu()

        def want(h, k):
            comb = lift._calibration(k["Kd"], k["Ed"])[1].cpu() if calib == "torch" else None
            return _bev(cfg, (h["seed"], k["seed"]), h["head"], k["K"], k["E"], comb, tag=("graph", half, calib))

        hd, Kd, Ed = a["hd"].clone(), a["Kd"].clone(), a["Ed"].clone()           # the graph's static inputs
        g = lift.capture(hd, Kd, Ed, static_calibration=static)
        assert (g.plan is not None) == static
        _assert_frames(g(), want(a, a), "first replay")
        hd.copy_(b["hd"])
        _assert_frames(g(), want(b, a), "new head")
        with torch.no_grad():
            eager = lift(a["hd"], a["Kd"], a["Ed"])
        other = other_graph["g"]()
        _assert_frames(eager, want(a, a), "eager between replays")
        _assert_frames(other, other_graph["exact"], "other graph")
        _assert_frames(g(), want(b, a), "replay after eager")
        if not static:
            Kd.copy_(b["Kd"])
            Ed.copy_(b["Ed"])
            _assert_frames(g(), want(b, b), "new calibration")
            _assert_frames(other_graph["g"](), other_graph["exact"], "other graph again")
        torch.cuda.synchronize()
        for buf in (g.scratch, other_graph["g"].scratch):
            assert buf is None or float(buf.abs().max()) == 0.0
        assert (g.scratch is None) == (layout == "channels_last")
        if layout == "contiguous":
            _assert_scratch_clean()
        for buf in lift_mod._scratch._bufs.values():
            assert float(buf.abs().max()) == 0.0
    finally:
        lib.fiery_lift_set_max_chunk_frames(0)
        lift_mod._scratch.clear()


# ==== 3. host pipeline ===========================================================================================================
HOST_CFG = _frames(GRID100, 16)
CHUNKS = {"1": 1, "1-3": [1, 3], "2-5-1": [2, 5, 1], "3": 3, "longer-than-batch": 40}


@pytest.fixture(scope="module")
def host_case():
    head, K, E, _ = _inputs(HOST_CFG, seed=51)
    return dict(head=head.pin_memory(), K=K.pin_memory(), E=E.pin_memory(), exact=_bev(HOST_CFG, 51, head, K, E))


def _from_host(lift, c, head=None, **kw):
    out = lift.lift_from_host(c["head"] if head is None else head, c["K"], c["E"], device=DEV, **kw)
    assert out.is_pinned() and tuple(out.shape) == (HOST_CFG.frames, HOST_CFG.out_channels, *HOST_CFG.bev_hw)
    return out


@pytest.mark.parametrize("chunks", list(CHUNKS))
def test_host_pipeline_chunk_sequences(host_case, chunks):
    lift = LiftSplat.from_config(HOST_CFG).to(DEV)
    _assert_frames(_from_host(lift, host_case, chunk_frames=CHUNKS[chunks]), host_case["exact"], chunks)
    _assert_scratch_clean()


@pytest.mark.parametrize("layout", ["contiguous", "channels_last"])
def test_host_pipeline_overwrites_a_nan_filled_out(host_case, layout):
    lift = LiftSplat.from_config(HOST_CFG, output_layout=layout).to(DEV)
    out = torch.full((HOST_CFG.frames, HOST_CFG.out_channels, *HOST_CFG.bev_hw), float("nan")).pin_memory()
    got = _from_host(lift, host_case, out=out, chunk_frames=[2, 5, 1])
    assert got is out and not bool(out.isnan().any())
    _assert_frames(out, host_case["exact"], layout)


def test_host_pipeline_fp16_head(host_case):
    h16 = host_case["head"].half().pin_memory()
    exact = _bev(HOST_CFG, 51, h16.float(), host_case["K"], host_case["E"], tag="f16")
    lift = LiftSplat.from_config(HOST_CFG).to(DEV)
    _assert_frames(_from_host(lift, host_case, head=h16, chunk_frames=3), exact, "fp16")


def test_host_pipeline_evicts_pooled_scratch_while_work_is_queued(host_case):
    """Chunks of 1, 2, 3, 4 and 5 frames need 5 scratch sizes on the run stream: the pool (4 entries) drops buffers whose kernels
    may still be queued; the caching allocator must keep them alive until that work has run."""
    lift = LiftSplat.from_config(HOST_CFG).to(DEV)
    c = lift._constants(DEV)
    lib = _lib.load()
    sizes = {int(lib.fiery_lift_scratch_bytes(lift._desc(c, nf, HOST_CFG.n_cameras, torch.float32, _lib.CALIB_RAW, _lib.BEV_NCHW)))
             for nf in range(1, 6)}
    assert len(sizes) == 5 > lift_mod._scratch.max_entries
    lift_mod._scratch.clear()
    try:
        _assert_frames(_from_host(lift, host_case, chunk_frames=[1, 2, 3, 4, 5, 1]), host_case["exact"], "eviction")
        assert len(_pool_entries(lift._host_streams(DEV)[1])) == lift_mod._scratch.max_entries
        _assert_scratch_clean()
    finally:
        lift_mod._scratch.clear()


# ==== 4. streams =================================================================================================================
def test_two_modules_on_two_streams():
    """Two modules (200 x 200 grid, 6 frames in 3 frame groups; 100 x 100 grid, 4 frames in 2), each on its own stream, alternating
    forward and backward with no synchronisation between the streams.  Both fork their chains onto the thread's side stream."""
    cases = [_case(_frames(ROUTE_TMA, 6), seed=61), _case(_frames(GRID100, 4), seed=62)]
    assert forward_groups(6, TILES) == 3 and forward_groups(4, TILES) == 2
    lifts = [LiftSplat.from_config(c["cfg"]).to(DEV) for c in cases]
    streams = [torch.cuda.Stream(DEV), torch.cuda.Stream(DEV)]
    lift_mod._scratch.clear()
    try:
        for s in streams:
            s.wait_stream(torch.cuda.current_stream(DEV))
        results = []
        for _ in range(2):
            bevs = []
            for c, lift, s in zip(cases, lifts, streams):
                with torch.cuda.stream(s):
                    h = c["hd"].clone().requires_grad_(True)
                    bevs.append((h, lift(h, c["Kd"], c["Ed"])))
            for (h, bev), c, s in zip(bevs, cases, streams):
                with torch.cuda.stream(s):
                    bev.backward(c["gd"])
                    results.append((c, bev.detach(), h.grad))
        torch.cuda.synchronize()
        for c, bev, grad in results:
            _assert_frames(bev, _bev(c["cfg"], c["seed"], c["head"], c["K"], c["E"]), c["cfg"].name)
            _assert_grad(grad, _grad(c), c["cfg"].name)
        for s in streams:
            entries = _pool_entries(s)
            assert entries and all(float(buf.abs().max()) == 0.0 for buf in entries)
    finally:
        lift_mod._scratch.clear()


def test_graph_replay_beside_eager_calls_on_another_stream():
    """One thread replays a graph on one stream while eager calls of another module run on a second stream."""
    a, a2 = _case(_frames(ROUTE_TMA, 6), seed=71), _case(_frames(ROUTE_TMA, 6), seed=72)
    e = _case(_frames(GRID100, 4), seed=73)
    lift_g = LiftSplat.from_config(a["cfg"]).to(DEV)
    lift_e = LiftSplat.from_config(e["cfg"]).to(DEV)
    hd = a["hd"].clone()
    g = lift_g.capture(hd, a["Kd"], a["Ed"])
    s1, s2 = torch.cuda.Stream(DEV), torch.cuda.Stream(DEV)
    lift_mod._scratch.clear()
    try:
        for s in (s1, s2):
            s.wait_stream(torch.cuda.current_stream(DEV))
        outs, eager = [], []
        for step in range(2):
            with torch.cuda.stream(s1):
                if step:
                    hd.copy_(a2["hd"])
                outs.append(g().clone())
            with torch.cuda.stream(s2), torch.no_grad():
                eager.append(lift_e(e["hd"], e["Kd"], e["Ed"]))
        torch.cuda.synchronize()
        for out, c in zip(outs, (a, a2)):                                # the graph keeps a's calibration
            _assert_frames(out, _bev(c["cfg"], (c["seed"], 71), c["head"], a["K"], a["E"]), ("graph", c["seed"]))
        for out in eager:
            _assert_frames(out, _bev(e["cfg"], e["seed"], e["head"], e["K"], e["E"]), "eager")
        assert float(g.scratch.abs().max()) == 0.0
        entries = _pool_entries(s2)
        assert entries and all(float(buf.abs().max()) == 0.0 for buf in entries)
    finally:
        lift_mod._scratch.clear()
