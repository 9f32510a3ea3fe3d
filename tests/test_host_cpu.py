"""CPU: host-side logic, the C ABI surface, and the no-fallback rule."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import fiery_b200
from fiery_b200 import _lib
from fiery_b200.geometry import (VoxelsSumming, bev_offset_fp32, calculate_birds_eye_view_parameters, create_frustum,
                                 split_frustum, z_valid_interval)
from fiery_b200.lift import LiftSplat
from fiery_b200.synthetic import CONFIGS, make_calibration, shard_frames
from oracle import lift_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    """Every function include/fiery_b200.h declares is exported by the built shared library with a ctypes signature."""
    header = open(os.path.join(ROOT, "include", "fiery_b200.h")).read()
    declared = set(re.findall(r"FIERY_API\s+[\w\s\*]+?\b(fiery_\w+)\s*\(", header))
    assert declared, "no declarations parsed"
    assert declared == set(_lib.SIGNATURES), (declared ^ set(_lib.SIGNATURES))
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name)
    assert lib.fiery_abi_version() == _lib.ABI_VERSION


def test_desc_struct_matches_header_layout():
    # 9 int32, 6 float, 2 float, 4 int32 = 21 x 4 bytes
    assert ctypes.sizeof(_lib.LiftDesc) == 21 * 4


def test_argument_validation_without_gpu():
    lib = _lib.load()
    d = _lib.LiftDesc()
    d.n_frames, d.n_cameras, d.depth_bins, d.channels, d.feat_h, d.feat_w = 1, 1, 48, 64, 8, 16
    d.bev_x, d.bev_y, d.bev_z = 50, 50, 2          # two height cells: the reference cannot do that either (fiery.py:269)
    for a in range(3):
        d.bev_resolution[a] = 1.0
    rc = lib.fiery_lift_forward(d, 16, 16, 16, 16, 16, 16, 16, 16, None, None)
    assert rc == -1 and b"bev_z" in lib.fiery_last_error()
    assert lib.fiery_lift_scratch_bytes(d) == 1 * 50 * 50 * 64 * 4 + 2560      # accumulator + one mark byte per pillar (padded to 128)
    assert lib.fiery_lift_plan_bytes(d) > 4 * 1296 + 2560                       # 4 tile records (header + run lists) + touched map
    assert lib.fiery_lift_workspace_bytes(d) >= 1 * 50 * 50 * 64 * 4           # NCHW gradient re-layout + room for a plan
    n = ctypes.c_int64(-1)
    assert lib.fiery_voxels_summing_plan(0, None, None, ctypes.byref(n), None) == 0 and n.value == 0


def test_forward_launch_plan_without_gpu():
    """fiery_lift_forward_launches is host logic: one tile kernel for channel-last output; for NCHW one (tile kernel, layout
    pass) chain per frame group, a group holding at least one tile per SM of an H100 (132) and at most four groups per call."""
    lib = _lib.load()
    d = _lib.LiftDesc()
    d.n_cameras, d.depth_bins, d.channels, d.feat_h, d.feat_w = 6, 48, 64, 28, 60        # 90 tiles per frame
    d.bev_x, d.bev_y, d.bev_z = 200, 200, 1
    d.bev_layout = _lib.BEV_NCHW
    expect = {0: 0, 1: 2, 2: 2, 3: 2, 4: 4, 5: 4, 6: 6, 8: 8, 9: 8, 12: 8, 100: 8}
    for frames, launches in expect.items():
        d.n_frames = frames
        assert lib.fiery_lift_forward_launches(d) == launches, frames
    d.n_frames, d.bev_layout = 8, _lib.BEV_NHWC
    assert lib.fiery_lift_forward_launches(d) == 1
    assert lib.fiery_lift_forward_launches(None) == 0
    # the test hook that forces the multi-pass path: 8 frames in passes of 3, 3, 2 -> (1 + 1 + 1) groups
    d.bev_layout = _lib.BEV_NCHW
    lib.fiery_lift_set_max_chunk_frames(3)
    try:
        assert lib.fiery_lift_forward_launches(d) == 6
        assert lib.fiery_lift_scratch_bytes(d) == (3 * (200 * 200 * 64 * 4 + 200 * 200) + 127) // 128 * 128
    finally:
        lib.fiery_lift_set_max_chunk_frames(0)


def test_no_cpu_fallback():
    """The product path refuses CPU tensors instead of silently computing on the host."""
    m = LiftSplat.from_config(CONFIGS["cfg1_tiny"])
    cfg = CONFIGS["cfg1_tiny"]
    K, E = make_calibration(cfg)
    head = torch.zeros(cfg.frames * cfg.n_cameras, cfg.head_channels, *cfg.feat_hw)
    with pytest.raises(_lib.FieryError):
        m(head, torch.from_numpy(K), torch.from_numpy(E))
    with pytest.raises(_lib.FieryError):
        VoxelsSumming.apply(torch.zeros(4, 8), torch.zeros(4, 3, dtype=torch.long), torch.zeros(4, dtype=torch.long))


def test_product_code_never_imports_the_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "fiery_b200")):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in src.replace("no CPU", ""), f"{f} mentions the oracle"


def test_host_constants_match_oracle():
    for cfg in CONFIGS.values():
        r, s, d = calculate_birds_eye_view_parameters(cfg.x_bound, cfg.y_bound, cfg.z_bound)
        ro, so, do = O.bev_grid(cfg.x_bound, cfg.y_bound, cfg.z_bound)
        assert torch.equal(r, ro) and torch.equal(s, so) and torch.equal(d, do)
        fr = create_frustum(cfg.final_dim, cfg.downsample, cfg.d_bound)
        assert torch.equal(fr, O.frustum_grid(cfg.final_dim, cfg.downsample, cfg.d_bound))
        u, v, dd = split_frustum(fr)
        assert u.numel() == cfg.feat_hw[1] and v.numel() == cfg.feat_hw[0] and dd.numel() == cfg.depth_bins
        off = bev_offset_fp32(s, r)
        assert np.array_equal(off, (so - ro / 2.0).numpy())
    with pytest.raises(ValueError):
        bad = create_frustum((64, 128), 8, (2.0, 50.0, 1.0)).clone()
        bad[3, 2, 1, 0] += 1.0
        split_frustum(bad)


@pytest.mark.parametrize("res,dim", [(20.0, 1), (0.5, 200), (0.3, 7), (1.7, 3)])
def test_z_valid_interval_is_exact(res, dim):
    """[lo, hi] is exactly the set of fp32 a with 0 <= trunc(a / res) < dim (fiery.py:236-247 on the z axis)."""
    lo, hi = z_valid_interval(res, dim)
    r = np.float32(res)

    def ok(a):
        q = np.float32(a) / r
        return q > -1 and int(np.trunc(q)) >= 0 and int(np.trunc(q)) < dim

    assert ok(lo) and ok(hi)
    assert not ok(np.nextafter(lo, np.float32(-np.inf), dtype=np.float32))
    assert not ok(np.nextafter(hi, np.float32(np.inf), dtype=np.float32))
    rng = np.random.default_rng(0)
    for a in rng.uniform(-2 * res, (dim + 1) * res, size=2000).astype(np.float32):
        assert ok(a) == (lo <= a <= hi)


def test_state_dict_names_match_reference():
    """fiery.py:21-23,128: the four non-trainable parameters the reference keeps in its state_dict."""
    m = LiftSplat()
    assert set(m.state_dict()) == {"bev_resolution", "bev_start_position", "bev_dimension", "frustum"}
    assert all(not p.requires_grad for p in m.parameters())


def test_shard_frames_partitions():
    for n in (1, 9, 12, 72):
        for ws in (1, 2, 4, 8):
            parts = [list(shard_frames(n, ws, r)) for r in range(ws)]
            assert sorted(sum(parts, [])) == list(range(n))
            assert max(map(len, parts)) - min(map(len, parts)) <= 1


def test_constants_follow_checkpoint_loads_and_in_place_edits():
    """The device-side constants are re-derived when the Parameters change under the module: ``load_state_dict`` copies in
    place (no ``_apply``), and in the reference the checkpoint's values win (fiery/models/fiery.py:21-23 are Parameters)."""
    import torch
    from fiery_b200.lift import LiftSplat
    a = LiftSplat(x_bound=(-50.0, 50.0, 0.5), y_bound=(-50.0, 50.0, 0.5))
    b = LiftSplat(x_bound=(-40.0, 40.0, 0.5), y_bound=(-50.0, 50.0, 0.5))
    cpu = torch.device("cpu")
    before = a._constants(cpu)
    assert before is a._constants(cpu)                            # cached while nothing changes
    assert before["dim"][0] == 200 and abs(float(before["off"][0]) + 50.0) < 1e-6
    a.load_state_dict(b.state_dict())
    after = a._constants(cpu)
    assert after is not before and after["dim"][0] == 160 and abs(float(after["off"][0]) + 40.0) < 1e-6
    with torch.no_grad():
        a.bev_start_position[1] += 1.0
    assert abs(float(a._constants(cpu)["off"][1]) + 49.0) < 1e-6
    # from_fiery shares the model's Parameters: a later edit of the model is seen
    import types
    model = types.SimpleNamespace(frustum=b.frustum, bev_resolution=b.bev_resolution, bev_start_position=b.bev_start_position,
                                  bev_dimension=b.bev_dimension, encoder_out_channels=64)
    shared = LiftSplat.from_fiery(model)
    assert shared.frustum is b.frustum
    x0 = float(shared._constants(cpu)["off"][0])
    with torch.no_grad():
        b.bev_start_position[0] -= 2.0
    assert abs(float(shared._constants(cpu)["off"][0]) - (x0 - 2.0)) < 1e-6


def test_fused_warp_entry_points_have_no_cpu_path():
    """LiftSplat.forward_warped / birds_eye_view_features_warped (fiery.py:140-146 in one chain): CPU tensors raise, like every
    other entry point; the sequence shape is checked before anything is launched."""
    import torch
    from fiery_b200.lift import LiftSplat, birds_eye_view_features_warped  # noqa: F401
    from fiery_b200.synthetic import CONFIGS
    cfg = CONFIGS["cfg1_tiny"]
    lift = LiftSplat.from_config(cfg)
    h, w = cfg.feat_hw
    head = torch.zeros(2 * cfg.n_cameras, cfg.head_channels, h, w)
    K, E = torch.eye(3).expand(2, cfg.n_cameras, 3, 3), torch.eye(4).expand(2, cfg.n_cameras, 4, 4)
    with pytest.raises(Exception, match="CUDA|cuda"):
        lift.forward_warped(head, K, E, torch.zeros(1, 2, 6), (50.0, 50.0))


def test_python_sources_reference_only_defined_names():
    """bench.py's code paths need a GPU, so a misplaced block shows up only on the box (it happened: a benchmark extra pasted into
    run_train used a helper that lives in main).  A conservative static pass: every name a function loads must be bound somewhere in
    that function, at module level, or be a builtin."""
    import ast
    import builtins
    import glob
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    files = [os.path.join(root, "bench.py"), os.path.join(root, "__graft_entry__.py")] + sorted(glob.glob(os.path.join(root, "fiery_b200", "*.py")))

    def bound(node):
        names = {n.id for n in ast.walk(node) if isinstance(n, ast.Name) and isinstance(n.ctx, (ast.Store, ast.Del))}
        names |= {a.arg for n in ast.walk(node) if isinstance(n, ast.arguments)
                  for a in n.args + n.kwonlyargs + n.posonlyargs + ([n.vararg] if n.vararg else []) + ([n.kwarg] if n.kwarg else [])}
        names |= {n.name for n in ast.walk(node) if isinstance(n, (ast.FunctionDef, ast.ClassDef))}
        names |= {(a.asname or a.name.split(".")[0]) for n in ast.walk(node) if isinstance(n, (ast.Import, ast.ImportFrom)) for a in n.names}
        names |= {n.name for n in ast.walk(node) if isinstance(n, ast.ExceptHandler) and n.name}
        return names

    problems = []
    for path in files:
        tree = ast.parse(open(path).read())
        module = set()
        for node in tree.body:
            module |= bound(node) if not isinstance(node, (ast.FunctionDef, ast.ClassDef)) else {node.name}
        funcs = [n for n in tree.body if isinstance(n, ast.FunctionDef)]
        funcs += [m for c in tree.body if isinstance(c, ast.ClassDef) for m in c.body if isinstance(m, ast.FunctionDef)]
        for fn in funcs:
            known = bound(fn) | module
            loaded = {n.id for n in ast.walk(fn) if isinstance(n, ast.Name) and isinstance(n.ctx, ast.Load)}
            missing = sorted(x for x in loaded if x not in known and not hasattr(builtins, x))
            if missing:
                problems.append((os.path.basename(path), fn.name, missing))
    assert not problems, problems
