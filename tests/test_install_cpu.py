"""CPU: install()/uninstall() rebind the reference's call sites (INTEGRATION.md) -- exercised on a stand-in `fiery`
package with the same module paths and symbol names as the reference (fiery/models/fiery.py:10,275,
fiery/utils/geometry.py:283); the real reference cannot be imported on the test box."""
import importlib
import sys
import textwrap

import pytest


@pytest.fixture
def fake_fiery(tmp_path, monkeypatch):
    root = tmp_path / "fiery"
    (root / "models").mkdir(parents=True)
    (root / "utils").mkdir()
    for d in (root, root / "models", root / "utils"):
        (d / "__init__.py").write_text("")
    (root / "utils" / "geometry.py").write_text(textwrap.dedent("""
        class VoxelsSumming:            # stands for fiery/utils/geometry.py:283
            tag = "reference"

        def warp_features(x, flow, mode='nearest', spatial_extent=None):              # geometry.py:181
            return "reference"

        def cumulative_warp_features(x, flow, mode='nearest', spatial_extent=None):   # geometry.py:225
            return "reference"
    """))
    (root / "models" / "fiery.py").write_text(textwrap.dedent("""
        from fiery.utils.geometry import cumulative_warp_features, VoxelsSumming          # bound at import, like fiery/models/fiery.py:10

        class Fiery:
            def calculate_birds_eye_view_features(self, x, intrinsics, extrinsics):   # fiery.py:275
                return "reference"
    """))
    monkeypatch.syspath_prepend(str(tmp_path))
    for name in [m for m in sys.modules if m == "fiery" or m.startswith("fiery.")]:
        monkeypatch.delitem(sys.modules, name)
    yield
    for name in [m for m in sys.modules if m == "fiery" or m.startswith("fiery.")]:
        sys.modules.pop(name, None)


def test_install_rebinds_and_uninstall_restores(fake_fiery):
    import fiery_b200.install as fb
    from fiery_b200.geometry import VoxelsSumming as ours
    from fiery_b200.lift import calculate_birds_eye_view_features as ours_bev

    geometry = importlib.import_module("fiery.utils.geometry")
    fiery_mod = importlib.import_module("fiery.models.fiery")
    ref_vs, ref_bev = geometry.VoxelsSumming, fiery_mod.Fiery.calculate_birds_eye_view_features

    fb.install(level="voxels_summing")
    assert geometry.VoxelsSumming is ours and fiery_mod.VoxelsSumming is ours      # both bindings (fiery.py:10)
    assert fiery_mod.Fiery.calculate_birds_eye_view_features is ref_bev
    fb.install()                                                                    # level="fused"
    assert fiery_mod.Fiery.calculate_birds_eye_view_features is fb._bev_features    # dispatches to ours_bev where supported
    assert ours_bev.__name__ == "calculate_birds_eye_view_features"
    fb.install(level="all")
    from fiery_b200.warp import cumulative_warp_features as ours_cwf
    assert fiery_mod.cumulative_warp_features.__wrapped__ is ours_cwf and geometry.cumulative_warp_features.__wrapped__ is ours_cwf
    # label warps (mode='nearest', the trainer's cumulative_warp_features_reverse) stay on the reference's function
    assert fiery_mod.cumulative_warp_features("x", None, mode="nearest") == "reference"
    assert geometry.warp_features("x", None, mode="nearest") == "reference"
    fb.uninstall()
    assert not hasattr(fiery_mod.cumulative_warp_features, "__wrapped__") and geometry.cumulative_warp_features("x", None) == "reference"
    assert geometry.VoxelsSumming is ref_vs and fiery_mod.VoxelsSumming is ref_vs
    assert fiery_mod.Fiery.calculate_birds_eye_view_features is ref_bev
    with pytest.raises(ValueError):
        fb.install(level="nope")


def test_unsupported_configuration_runs_the_reference_method(fake_fiery):
    """A lift configuration the kernels do not cover (e.g. MODEL.ENCODER.OUT_CHANNELS != 64, fiery/config.py:78) keeps the
    reference's own method, with one warning; a covered one is routed to the fused lift (which raises on CPU tensors: there
    is no CPU path)."""
    import types
    import torch
    import fiery_b200.install as fb
    from fiery_b200 import _lib
    fiery_mod = importlib.import_module("fiery.models.fiery")
    fb.install()
    try:
        m = fiery_mod.Fiery()
        m.encoder_downsample, m.encoder_out_channels = 8, 32
        m.frustum = torch.zeros(48, 28, 60, 3)
        m.bev_dimension = torch.tensor([200, 200, 1])
        x = torch.zeros(1, 1, 6, 3, 224, 480)
        assert "OUT_CHANNELS" in fb.unsupported_reason(m, x)
        with pytest.warns(RuntimeWarning, match="not covered"):
            assert m.calculate_birds_eye_view_features(x, None, None) == "reference"
        m.encoder_out_channels = 64
        assert fb.unsupported_reason(m, x) is None
        m.encoder = types.SimpleNamespace(get_features=lambda t: t[:, :, ::8, ::8], depth_layer=lambda t: t.repeat(1, 38, 1, 1)[:, :112],
                                          use_depth_distribution=True)
        m.bev_resolution, m.bev_start_position = torch.tensor([0.5, 0.5, 20.0]), torch.tensor([-49.75, -49.75, 0.0])
        with pytest.raises(_lib.FieryError, match="no CPU path"):
            m.calculate_birds_eye_view_features(x, torch.eye(3).expand(1, 1, 6, 3, 3), torch.eye(4).expand(1, 1, 6, 4, 4))
    finally:
        fb.uninstall()


def test_depth_layer_swap_keeps_parameters_and_state_dict_keys():
    """use_tensor_core_depth_layer: Encoder.depth_layer (encoder.py:36) becomes the tensor-core (wgmma) layer with the SAME Parameters."""
    import types
    import torch.nn as nn
    import fiery_b200.install as fb
    from fiery_b200.depth_layer import DepthLayer
    model = types.SimpleNamespace(encoder=nn.Module())
    conv = nn.Conv2d(128, 48 + 64, kernel_size=1, padding=0)
    model.encoder.depth_layer = conv
    keys = set(model.encoder.state_dict())
    assert fb.use_tensor_core_depth_layer(model) is model
    layer = model.encoder.depth_layer
    assert isinstance(layer, DepthLayer) and layer.weight is conv.weight and layer.bias is conv.bias
    assert set(model.encoder.state_dict()) == keys == {"depth_layer.weight", "depth_layer.bias"}
    assert fb.use_tensor_core_depth_layer(model).encoder.depth_layer is layer          # idempotent
    other = types.SimpleNamespace(encoder=nn.Module())
    other.encoder.depth_layer = nn.Conv2d(64, 112, kernel_size=1)
    with pytest.warns(RuntimeWarning, match="not covered"):
        fb.use_tensor_core_depth_layer(other)
    assert isinstance(other.encoder.depth_layer, nn.Conv2d)
    fb._warned.clear()


def test_depth_layer_has_no_cpu_path():
    import torch
    from fiery_b200.depth_layer import DepthLayer
    with pytest.raises(Exception, match="CUDA|cuda"):
        DepthLayer(112)(torch.zeros(1, 128, 4, 8))
    with pytest.raises(ValueError):
        DepthLayer(200)


def test_depth_layer_packed_operand_follows_the_parameter():
    """The (128, 128) operand of the kernel is cached per dtype and re-made when the weight changes in place (optimizer step) or is
    loaded from a checkpoint -- the class of staleness ADVICE.md flagged for the lift's constants."""
    import torch
    from fiery_b200.depth_layer import DepthLayer, pack_weight
    layer = DepthLayer(112)
    a = layer._packed_weight(torch.float16)
    assert tuple(a.shape) == (128, 128) and a.dtype == torch.float16
    assert torch.equal(a[:112], layer.weight.detach().reshape(112, 128).half()) and float(a[112:].abs().max()) == 0.0
    assert layer._packed_weight(torch.float16) is a                          # cached
    assert layer._packed_weight(torch.bfloat16).dtype == torch.bfloat16     # one entry per operand type
    with torch.no_grad():
        layer.weight.mul_(3.0)
    b = layer._packed_weight(torch.float16)
    assert b is not a and torch.equal(b[:112], layer.weight.detach().reshape(112, 128).half())
    other = DepthLayer(112)
    layer.load_state_dict(other.state_dict())
    c = layer._packed_weight(torch.float16)
    assert c is not b and torch.equal(c, pack_weight(other.weight, torch.float16))
    with pytest.raises(ValueError):
        pack_weight(torch.zeros(112, 64, 1, 1), torch.float16)
