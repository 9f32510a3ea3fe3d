"""The SpatialGRU's kernels (fiery_spatial_gru_*, fiery_conv3x3_*) element by element across their accepted envelope: every forward
stage of every step and every gradient against the fp64 restatement of tests/_spatial_gru_cases.py fed the kernels' own stage inputs,
each element within its bound; the recurrence split in two calls bit for bit; the layouts x may arrive in, bit for bit; the TF32
rounding modes the header promises, on ties; saturated gates, NaN and infinities; the exact regime bit for bit; every backward subset; the module over several
optimizer steps; one run whose saved buffer spans more than 2^31 bytes.  Every output the C ABI writes lies between sentinel margins
that are checked unchanged."""
from __future__ import annotations

import copy
import itertools

import pytest
import torch
import torch.nn as nn

from fiery_b200 import _lib
from fiery_b200 import future_prediction as fp
from oracle.future_oracle import SpatialGRU
from tests import _spatial_gru_cases as gc

pytestmark = pytest.mark.gpu

EPS = 1e-5
MARGINS = {}                     # stage -> the largest err / bound seen, reported at the end of the module


@pytest.fixture(scope="module", autouse=True)
def _report_margins():
    yield
    if MARGINS:
        print("\nlargest err/bound per stage: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(MARGINS.items())))


def _note(ratios, prefix=""):
    for k, (r, _) in ratios.items():
        MARGINS[prefix + k] = max(MARGINS.get(prefix + k, 0.0), r)


def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


MARGIN = 64                      # floats of sentinel on each side of every output the C ABI writes (keeps 16-byte alignment)
SENTINEL = 12345.0


class Guarded:
    """NaN-filled outputs between sentinel margins; ``intact()`` says whether every margin is unchanged"""

    def __init__(self):
        self.bufs = []

    def __call__(self, *shape):
        n = 1
        for d in shape:
            n *= d
        buf = torch.full((n + 2 * MARGIN,), SENTINEL, device="cuda")
        self.bufs.append(buf)
        view = buf[MARGIN:MARGIN + n].view(shape)
        view.fill_(float("nan"))
        return view

    def intact(self):
        torch.cuda.synchronize()
        return all(bool((b[:MARGIN] == SENTINEL).all() and (b[-MARGIN:] == SENTINEL).all()) for b in self.bufs)


class Run:
    """one forward and backward through the C ABI, every output NaN-filled between sentinel margins and every workspace sized exactly
    and filled with 0xFF bytes"""

    def __init__(self, x, h0, p, frames, training, bias_init, eps=EPS):
        self.x, self.h0, self.p, self.T, self.training, self.bias_init, self.eps = x, h0, p, frames, training, bias_init, eps
        b, tx, cx, X, Y = x.shape
        ch = h0.shape[1]
        self.shape = (b, tx, cx, X, Y, ch)
        self.d = fp._desc(b, frames, tx, X, Y, cx, ch, (x.stride(0), x.stride(1), x.stride(2)), training, eps, bias_init)
        lib = _lib.load()
        self.packed = fp.pack_weights([p["w_gates"][:ch], p["w_gates"][ch:], p["w_state"]], cx)
        self.guard = Guarded()
        self.out, self.means, self.vars = self.guard(b, frames, ch, X, Y), self.guard(frames, ch), self.guard(frames, ch)
        self.saved = self.guard(int(lib.fiery_spatial_gru_saved_bytes(self.d)) // 4)
        ws = torch.full((int(lib.fiery_spatial_gru_forward_workspace_bytes(self.d)),), 255, dtype=torch.uint8, device="cuda")
        ptr = lambda t: t.data_ptr() if t is not None else 0        # noqa: E731
        self.ptr = ptr
        _lib.call("fiery_spatial_gru_forward", x.device, self.d, x.data_ptr(), h0.data_ptr(), self.packed.data_ptr(),
                  p["b_gates"].data_ptr(), ptr(p.get("gamma")), ptr(p.get("beta")), ptr(p["running_mean"]), ptr(p["running_var"]),
                  self.out.data_ptr(), self.saved.data_ptr(), self.means.data_ptr(), self.vars.data_ptr(), ws.data_ptr())

    def kernel(self):
        return gc.as_kernel(self.out, self.saved, self.means, self.vars)

    def backward(self, go, want=("x", "h0", "w_gates", "b_gates", "w_state", "gamma", "beta")):
        b, tx, cx, X, Y, ch = self.shape
        p = self.p
        shapes = {"x": (b, tx, cx, X, Y), "h0": (b, ch, X, Y), "w_gates": (2 * ch, cx + ch, 3, 3), "b_gates": (2 * ch,),
                  "w_state": (ch, cx + ch, 3, 3), "gamma": (ch,), "beta": (ch,)}
        g = {k: (self.guard(*s) if k in want and (k not in ("gamma", "beta") or p.get(k) is not None) else None) for k, s in shapes.items()}
        lib = _lib.load()
        ws = torch.full((int(lib.fiery_spatial_gru_backward_workspace_bytes(self.d)),), 255, dtype=torch.uint8, device="cuda")
        ptr = self.ptr
        _lib.call("fiery_spatial_gru_backward", go.device, self.d, go.data_ptr(), self.x.data_ptr(), self.h0.data_ptr(),
                  self.out.data_ptr(), self.saved.data_ptr(), self.means.data_ptr(), self.vars.data_ptr(), self.packed.data_ptr(),
                  ptr(p.get("gamma")), ptr(p.get("beta")), ptr(g["x"]), ptr(g["h0"]), ptr(g["w_gates"]), ptr(g["b_gates"]),
                  ptr(g["w_state"]), ptr(g["gamma"]), ptr(g["beta"]), ws.data_ptr())
        return g


def _setup(case, seed=1, dev="cuda"):
    cx, ch, X, Y, b, T, Tx, bias_init = case
    p = gc.params(cx, ch, seed=seed + cx + 3 * ch, dtype=torch.float32, device=dev)
    x, h0, go = gc.inputs(b, T, Tx, cx, ch, X, Y, seed=seed, dtype=torch.float32, device=dev)
    return p, x, h0, go


def _check_run(run, go, label=""):
    stages, fw = gc.stage_ratios(run.kernel(), run.x, run.h0, run.p, run.T, run.training, run.eps, run.bias_init)
    _note(stages, label)
    bad = {k: v for k, v in stages.items() if not (v[1] and v[0] <= 1.0)}
    assert not bad, ("forward stages", bad)
    assert run.guard.intact(), "forward wrote outside its outputs"
    if go is None:
        return fw
    grads = run.backward(go)
    gr = gc.grad_ratios(fw, grads, run.x, run.h0, run.p, go, run.training, run.eps)
    _note(gr, label + "d_")
    bad = {k: v for k, v in gr.items() if not (v[1] and v[0] <= 1.0)}
    assert not bad, ("gradients", bad)
    assert run.guard.intact(), "backward wrote outside its outputs"
    return fw


# 1, 2: every stage of every step and every gradient, element by element, at every shape of the list
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("case", gc.CASES, ids=gc.case_id)
def test_stages_and_gradients(case, training):
    p, x, h0, go = _setup(case)
    _check_run(Run(x, h0, p, case[5], training, case[7]), go)


# 3: the recurrence split in two calls
@pytest.mark.parametrize("tx_full", [True, False], ids=["TxT", "Tx1"])
def test_split_recurrence_is_bit_exact(tx_full):
    case = (9, 33, 9, 20, 3, 4, 4 if tx_full else 1, 0.5)
    p, x, h0, go = _setup(case, seed=4)
    T = case[5]
    full = Run(x, h0, p, T, True, case[7])
    fg = full.backward(go)
    fw = gc.forward(x.double(), h0.double(), {k: (v.double() if v is not None else None) for k, v in p.items()}, T, True, EPS, case[7],
                    True, {k: v.double() for k, v in full.kernel().items()})
    _, bound = gc.adjoint(fw, x.double(), h0.double(), {k: (v.double() if v is not None else None) for k, v in p.items()}, go.double(),
                          True, EPS)
    fk = full.kernel()
    for k in range(1, T):
        xa = x[:, :k].contiguous() if tx_full else x
        xb = x[:, k:].contiguous() if tx_full else x
        a = Run(xa, h0, p, k, True, case[7])
        bb = Run(xb, full.out[:, k - 1].contiguous(), p, T - k, True, case[7])
        ak, bk = a.kernel(), bb.kernel()
        assert torch.equal(torch.cat([a.out, bb.out], 1), full.out)
        assert torch.equal(torch.cat([a.means, bb.means]), full.means) and torch.equal(torch.cat([a.vars, bb.vars]), full.vars)
        for n in ("u", "r", "q", "s"):
            assert torch.equal(torch.cat([ak[n], bk[n]]), fk[n]), n
        gb = bb.backward(go[:, k:].contiguous())
        go_a = go[:, :k].clone()
        go_a[:, k - 1] += gb["h0"]
        ga = a.backward(go_a)
        assert torch.equal(ga["h0"], fg["h0"]), k
        if tx_full:
            assert torch.equal(torch.cat([ga["x"], gb["x"]], 1), fg["x"]), k
        for n in ("w_gates", "b_gates", "w_state", "gamma", "beta"):
            r, same = gc.excess(ga[n].double() + gb[n].double(), fg[n].double(), 2 * bound[n])
            assert same and r <= 1.0, (n, k, r)


# 4: layouts
def _values_as(x, dtype):
    return x.to(dtype).float()


def _op(x, h0, p, T, training=True, bias_init=0.25):
    ch = h0.shape[1]
    args = (p["w_gates"][:ch], p["b_gates"][:ch], p["w_gates"][ch:], p["b_gates"][ch:], p["w_state"], p["gamma"], p["beta"])
    out, means, var, saved = fp.forward(x, h0, *args, None if training else p["running_mean"], None if training else p["running_var"],
                                        T, training, EPS, bias_init)
    go = gc.inputs(x.shape[0], T, 1, 1, ch, x.shape[3], x.shape[4], seed=9, dtype=torch.float32, device="cuda")[2]
    grads = fp.backward(go, x, h0, out, saved, means, var, args[0], args[2], args[4], p["gamma"], p["beta"], T, training, EPS,
                        bias_init, True, True, True, True, True)
    return [out, means, var, saved] + [g for g in grads if g is not None]


def _same(a, b):
    return all(torch.equal(u, v) for u, v in zip(a, b)) and len(a) == len(b)


LAYOUT_CASE = (8, 12, 9, 20, 3, 3)


def _layout_inputs(dtype=torch.float32):
    cx, ch, X, Y, b, T = LAYOUT_CASE
    p, x, h0, _ = _setup((cx, ch, X, Y, b, T, T, 0.25), seed=6)
    return p, _values_as(x, dtype), _values_as(h0, dtype), T


@pytest.mark.parametrize("layout", ["frame_major", "channel_slice", "batch_slice", "time_step2"])
def test_uncopied_layouts_are_bit_exact(layout):
    p, x, h0, T = _layout_inputs()
    b, _, cx, X, Y = x.shape
    if layout == "frame_major":
        xv = x.transpose(0, 1).contiguous().transpose(0, 1)
    elif layout == "channel_slice":
        big = torch.zeros(b, T, cx + 4, X, Y, device="cuda")
        big[:, :, 4:] = x
        xv = big[:, :, 4:]
    elif layout == "batch_slice":
        big = torch.zeros(b + 1, T, cx, X, Y, device="cuda")
        big[1:] = x
        xv = big[1:]
    else:
        big = torch.zeros(b, 2 * T, cx, X, Y, device="cuda")
        big[:, ::2] = x
        xv = big[:, ::2]
    assert not xv.is_contiguous() or layout == "batch_slice"
    assert fp.gru_input(xv) is xv
    assert _same(_op(xv, h0, p, T), _op(x, h0, p, T))


@pytest.mark.parametrize("layout", ["misaligned", "h0_misaligned", "fp16", "bf16", "fp64", "h0_strided"])
def test_copied_layouts_are_bit_exact(layout):
    dtype = {"fp16": torch.float16, "bf16": torch.bfloat16, "fp64": torch.float64}.get(layout, torch.float32)
    p, x, h0, T = _layout_inputs(dtype)
    want = _op(x, h0, p, T)
    xv, hv = x, h0
    if layout == "misaligned":
        buf = torch.empty(x.numel() + 1, device="cuda")
        xv = buf[1:].view(x.shape)
        xv.copy_(x)
        assert xv.data_ptr() % 16 != 0
    elif layout == "h0_misaligned":
        buf = torch.empty(h0.numel() + 1, device="cuda")
        hv = buf[1:].view(h0.shape)
        hv.copy_(h0)
    elif layout == "h0_strided":
        hv = h0.transpose(2, 3).contiguous().transpose(2, 3)
    else:
        xv, hv = x.to(dtype), h0.to(dtype)
    if not layout.startswith("h0"):
        assert fp.gru_input(xv) is not xv and fp.gru_input(xv).data_ptr() % 16 == 0
    assert _same(_op(xv, hv, p, T), want)


def test_one_x_frame_against_x_materialized_over_time():
    cx, ch, X, Y, b, T = LAYOUT_CASE
    p, x, h0, go = _setup((cx, ch, X, Y, b, T, 1, 0.25), seed=7)
    one = Run(x, h0, p, T, True, 0.25)
    xt = x.expand(b, T, cx, X, Y).contiguous()
    every = Run(xt, h0, p, T, True, 0.25)
    assert torch.equal(one.out, every.out) and torch.equal(one.saved, every.saved)
    assert torch.equal(one.means, every.means) and torch.equal(one.vars, every.vars)
    g1, gT = one.backward(go), every.backward(go)
    for n in ("h0", "w_gates", "b_gates", "w_state", "gamma", "beta"):
        assert torch.equal(g1[n], gT[n]), n
    fw = gc.forward(x.double(), h0.double(), {k: v.double() for k, v in p.items()}, T, True, EPS, 0.25, True,
                    {k: v.double() for k, v in one.kernel().items()})
    want, bound = gc.adjoint(fw, x.double(), h0.double(), {k: v.double() for k, v in p.items()}, go.double(), True, EPS)
    r, same = gc.excess(g1["x"], want["x"], bound["x"])
    assert same and r <= 1.0
    r, same = gc.excess(gT["x"].double().sum(1, keepdim=True), want["x"], bound["x"])
    assert same and r <= 1.0


@pytest.mark.parametrize("axis", ["batch", "channel", "time"])
def test_stride_zero_inputs(axis):
    cx, ch, X, Y, b, T = LAYOUT_CASE
    p, x, h0, _ = _layout_inputs()
    if axis == "batch":
        xv = x[:1].expand(b, T, cx, X, Y)
    elif axis == "channel":
        xv = x[:, :, :1].expand(b, T, cx, X, Y)
    else:
        xv = x[:, :1].expand(b, T, cx, X, Y)
    assert _same(_op(xv, h0, p, T), _op(xv.contiguous(), h0, p, T))


# 6: rounding probes
PROBES = [1 + 2 ** -11, 1 + 2 ** -12, 1 - 2 ** -12, 1 + 3 * 2 ** -12, -(1 + 2 ** -11), 1 - 3 * 2 ** -13, 1.5 + 2 ** -10, 2 + 2 ** -10]


def test_rounding_modes_of_the_3x3_kernels():
    n = len(PROBES)
    v = torch.tensor(PROBES, dtype=torch.float64)
    rna, rne, rz = gc.tf32_rna(v), gc.tf32_rne(v), gc.tf32_rz(v)
    assert not torch.equal(rna, rne) and not torch.equal(rna, rz)
    d = fp.conv3x3_desc(1, 1, 4, (n, 0), (n, 0))
    pw = 2.0 ** -torch.arange(n, dtype=torch.float64)                     # a power of two per row, one tap each
    w = torch.zeros(n, n, 3, 3, dtype=torch.float64)
    w[range(n), range(n), 1, 1] = pw
    packed = fp.conv3x3_pack(w.float().cuda(), d)
    x = v.view(1, n, 1, 1).expand(1, n, 1, 4).float().cuda().contiguous()
    y = _nan(1, n, 1, 4)
    fp.conv3x3_forward(d, x, None, packed, y, None)
    gx = _nan(1, n, 1, 4)
    fp.conv3x3_backward_data(d, x, None, packed, gx, None)
    torch.cuda.synchronize()
    want = (rna * pw).view(1, n, 1, 1).expand(1, n, 1, 4)
    y, gx = y.double().cpu(), gx.double().cpu()
    assert torch.equal(y, want), "activations: round to nearest, ties away"
    assert torch.equal(gx, want), "output gradients in the input gradient: round to nearest, ties away"
    # the weights: probes as weights, activations 1
    w2 = torch.zeros(n, n, 3, 3, dtype=torch.float64)
    w2[range(n), range(n), 1, 1] = v
    y2 = _nan(1, n, 1, 4)
    fp.conv3x3_forward(d, torch.ones(1, n, 1, 4, device="cuda"), None, fp.conv3x3_pack(w2.float().cuda(), d), y2, None)
    torch.cuda.synchronize()
    assert torch.equal(y2.double().cpu(), rna.view(1, n, 1, 1).expand(1, n, 1, 4)), "weights: round to nearest, ties away"
    # the weight gradient: one pixel; the activation rounded to nearest, the output gradient truncated
    ws = torch.full((max(int(_lib.load().fiery_conv3x3_backward_weight_workspace_bytes(d)), 16),), 255, dtype=torch.uint8, device="cuda")
    for probe_x in (True, False):
        xa = torch.zeros(1, n, 1, 4, device="cuda")
        gy = torch.zeros(1, n, 1, 4, device="cuda")
        xa[0, :, 0, 0] = v.float().cuda() if probe_x else 1.0
        gy[0, :, 0, 0] = 1.0 if probe_x else v.float().cuda()
        gw = _nan(n, n, 3, 3)
        fp.conv3x3_backward_weight(d, xa, None, gy, gw, ws)
        torch.cuda.synchronize()
        diag = gw[range(n), range(n), 1, 1].double().cpu()
        assert torch.equal(diag, rna if probe_x else rz), "weight gradient: x to nearest, grad_y truncated"


def test_rounding_of_q_through_the_gru():
    # zero gate weights and biases: r = 0.5 exactly; h0 = 1 + 2^-11, so q = 0.5 + 2^-12, a tie of the state convolution's operand
    cx, ch, X, Y, b = 1, 1, 1, 4, 2
    p = gc.params(cx, ch, seed=1, dtype=torch.float32, device="cuda")
    p["w_gates"].zero_()
    p["b_gates"].zero_()
    p["w_state"].zero_()
    p["w_state"][0, 1, 1, 1] = 1.0
    p["running_mean"].zero_()
    p["running_var"].fill_(1.0)
    p["gamma"].fill_(1.0)
    p["beta"].zero_()
    x = torch.zeros(b, 1, cx, X, Y, device="cuda")
    h0 = torch.full((b, ch, X, Y), 1 + 2 ** -11, device="cuda")
    run = Run(x, h0, p, 1, False, 0.0, eps=0.0)
    k = run.kernel()
    assert bool((k["r"] == 0.5).all()) and bool((k["q"] == 0.5 + 2 ** -12).all())
    assert bool((k["s"] == 0.5 + 2 ** -11).all()), k["s"]


# 7: values
@pytest.mark.parametrize("sat", [30.0, -30.0])
def test_saturated_gates(sat):
    case = (9, 16, 9, 20, 2, 3, 3, 20.0 if sat > 0 else -20.0)
    p, x, h0, go = _setup(case, seed=8)
    p["b_gates"] += sat
    _check_run(Run(x, h0, p, 3, True, case[7]), go, "sat_")


@pytest.mark.parametrize("training", [False, True], ids=["eval", "train"])
@pytest.mark.parametrize("value", ["nan", "inf"])
def test_non_finite_inputs(value, training):
    # NaN / +-inf at chosen pixels of x and h0: every stage's and every gradient's NaN and infinity positions and signs are the
    # restatement's, the finite elements within their bounds.  A non-finite input pixel reaches every output channel of its 3x3
    # neighbourhood (0 * NaN is NaN, zero weights included); in training it makes every channel's batch statistics NaN.
    case = (8, 8, 16, 20, 2, 2, 2, 0.0)
    p, x, h0, go = _setup(case, seed=9)
    v = float(value)
    x[0, 0, 1, 3, 4] = v
    x[1, 1, 5, 15, 19] = -v
    h0[1, 2, 0, 0] = -v
    h0[0, 4, 8, 10] = v
    run = Run(x, h0, p, 2, training, 0.0)
    _check_run(run, go, "nonfinite_")
    if training:
        assert bool(torch.isnan(run.means).all()) and bool(torch.isnan(run.vars).all())


@pytest.mark.parametrize("training", [False, True], ids=["eval", "train"])
def test_nan_norm_weight_poisons_exactly_its_channel(training):
    # a NaN in one channel of the norm's weight: that channel of the output is NaN everywhere, every other channel finite and
    # within its bound (one step, so the NaN does not reach the next step's convolutions)
    case = (8, 8, 9, 20, 2, 1, 1, 0.0)
    p, x, h0, _ = _setup(case, seed=10)
    p["gamma"][3] = float("nan")
    run = Run(x, h0, p, 1, training, 0.0)
    _check_run(run, None, "nonfinite_")
    bad = torch.isnan(run.out).any(4).any(3).any(1).any(0)
    assert bad.tolist() == [c == 3 for c in range(8)]
    assert bool(torch.isnan(run.out[:, :, 3]).all())


# 5: the exact regime, whole GRU
@pytest.mark.parametrize("config", [0, 1], ids=["zero_gates", "x_weights"])
def test_exact_regime_is_bit_exact(config):
    x, h0, p, go = gc.exact_case(config)
    T = x.shape[1]
    fw = gc.forward(x, h0, p, T, False, 0.0, 0.0, True)
    want, _ = gc.adjoint(fw, x, h0, p, go, False, 0.0)
    assert gc.exact_regime_holds(fw, want, x, h0, p, go) == []
    pc = {k: v.float().cuda() for k, v in p.items()}
    run = Run(x.float().cuda(), h0.float().cuda(), pc, T, False, 0.0, eps=0.0)
    k = run.kernel()
    v = fw["value"]
    assert torch.equal(run.out.cpu().double(), torch.stack(v["out"], 1))
    for n in ("u", "r", "q", "s"):
        assert torch.equal(k[n].cpu().double(), torch.stack(v[n])), n
    g = run.backward(go.float().cuda())
    for n, w in want.items():
        assert torch.equal(g[n].cpu().double(), w), n
    assert run.guard.intact()


# 8: module and ABI paths
def test_every_backward_subset_matches_the_full_call():
    case = (7, 9, 8, 12, 2, 3, 3, 0.5)
    p, x, h0, go = _setup(case, seed=10)
    run = Run(x, h0, p, 3, True, 0.5)
    names = ("x", "h0", "w_gates", "b_gates", "w_state", "gamma", "beta")
    full = run.backward(go)
    for k in range(1, len(names)):
        for sub in itertools.combinations(names, k):
            g = run.backward(go, sub)
            for n in names:
                if n in sub:
                    assert torch.equal(g[n], full[n]), (sub, n)
    assert run.guard.intact()


def _module(cx, ch, seed, affine=True, track=True):
    m = SpatialGRU(cx, ch, gru_bias_init=0.5)
    if not (affine and track):
        m.conv_state_tilde.norm = nn.BatchNorm2d(ch, affine=affine, track_running_stats=track)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for prm in m.parameters():
            prm.copy_(torch.randn(prm.shape, generator=g) * (0.3 if prm.dim() == 1 else 1.5 / (9 * (cx + ch)) ** 0.5))
    return m.cuda()


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def _within(e, e32):
    """the bar of tests/test_spatial_gru_gpu.py: 3x torch's own fp32 CUDA error against fp64, never below 1e-3 (TF32 operands)"""
    return e <= max(3 * e32, 1e-3)


@pytest.mark.parametrize("variant", ["affine_false", "untracked_eval", "state_none", "sum_backward"])
def test_module_variants(variant):
    cx, ch, b, T, X, Y = 8, 16, 2, 3, 9, 12
    m = _module(cx, ch, 3, affine=variant != "affine_false", track=variant != "untracked_eval")
    if variant == "untracked_eval":
        m.eval()
    ref = copy.deepcopy(m).double()
    ours = fp.TensorCoreSpatialGRU.from_module(copy.deepcopy(m))
    x, h0, go = gc.inputs(b, T, T, cx, ch, X, Y, seed=2, dtype=torch.float32, device="cuda")
    outs = []
    tf32_ops = gc.tf32_operands(copy.deepcopy(m).double())
    for mod, dt in ((ref, torch.float64), (copy.deepcopy(m), torch.float32), (ours, torch.float32), (tf32_ops, torch.float64)):
        xx = x.detach().to(dt).clone().requires_grad_(True)
        hh = h0.detach().to(dt).clone().requires_grad_(True)
        o = mod(xx) if variant == "state_none" else mod(xx, hh)
        (o.sum() if variant == "sum_backward" else (o * go.to(dt)).sum()).backward()
        outs.append((o.detach(), xx.grad, None if variant == "state_none" else hh.grad, [q.grad for q in mod.parameters()]))
    # the reference error: the larger of torch's fp32 CUDA module and fp64 on TF32-rounded operands, as tests/test_spatial_gru_gpu.py
    ref_outs, ours_outs = outs[0], outs[2]
    for i in range(3):
        got, want = ours_outs[i], ref_outs[i]
        if want is not None:
            e_ref = max(_rel(outs[1][i], want), _rel(outs[3][i], want))
            assert _within(_rel(got, want), e_ref), i
    for a, w, w32, wt in zip(ours_outs[3], ref_outs[3], outs[1][3], outs[3][3]):
        assert _within(_rel(a, w), max(_rel(w32, w), _rel(wt, w)))


def test_sgd_steps_and_load_state_dict():
    # three SGD steps against the fp64 reference module stepped the same way (weights, running statistics, num_batches_tracked, on
    # tests/test_spatial_gru_gpu.py's bar); after each in-place step and after load_state_dict the swapped module computes what a
    # fresh swap of the same weights (a new pack) computes, bit for bit, so the pack cache follows the updates
    cx, ch, b, T, X, Y = 8, 16, 2, 3, 9, 12
    m = _module(cx, ch, 4)
    ref64, ref32, reft = copy.deepcopy(m).double(), copy.deepcopy(m), gc.tf32_operands(copy.deepcopy(m).double())
    ours = fp.TensorCoreSpatialGRU.from_module(m)
    mods = [(ref64, torch.float64), (ref32, torch.float32), (reft, torch.float64), (ours, torch.float32)]
    opts = [torch.optim.SGD(mod.parameters(), lr=0.02) for mod, _ in mods]
    x, h0, go = gc.inputs(b, T, T, cx, ch, X, Y, seed=3, dtype=torch.float32, device="cuda")

    def fresh_eval():
        f = fp.TensorCoreSpatialGRU.from_module(copy.deepcopy(m)).eval()
        ours.eval()
        want, got = f(x, h0), ours(x, h0)
        ours.train()
        return torch.equal(got, want)

    for step in range(3):
        for (mod, dt), opt in zip(mods, opts):
            opt.zero_grad()
            (mod(x.to(dt), h0.to(dt)) * go.to(dt)).sum().backward()
            opt.step()
        assert fresh_eval(), step
    s64, s32, st, so = (mod.state_dict() for mod, _ in mods)
    assert list(so) == list(s64)
    for k in s64:
        if k.endswith("num_batches_tracked"):
            assert int(so[k]) == int(s64[k]) == 3 * T
        else:
            assert _within(_rel(so[k], s64[k]), max(_rel(s32[k], s64[k]), _rel(st[k], s64[k]))), k
    ours.load_state_dict(_module(cx, ch, 5).state_dict())
    assert fresh_eval()
    assert int(m.conv_state_tilde.norm.num_batches_tracked) == 0


# 9: a saved buffer past 2^31 bytes
def test_saved_buffer_past_two_gigabytes():
    case = (64, 64, 264, 256, 4, 8, 8, 0.25)
    cx, ch, X, Y, b, T, Tx, g0 = case
    p, x, h0, go = _setup(case, seed=12)
    full = Run(x, h0, p, T, True, g0)
    assert full.saved.numel() * 4 > 2 ** 31
    fk = full.kernel()
    # the stage checks on steps 0 and 7 (and 7's predecessor as its input)
    for t0 in (0, T - 1):
        sub = {n: (v[:, t0:t0 + 1] if n == "out" else v[t0:t0 + 1]) for n, v in fk.items()}
        hs = h0 if t0 == 0 else fk["out"][:, t0 - 1]
        stages, _ = gc.stage_ratios(sub, x[:, t0:t0 + 1], hs, p, 1, True, EPS, g0)
        _note(stages, "large_")
        assert all(s and r <= 1.0 for r, s in stages.values()), (t0, stages)
    fg = full.backward(go, ("x", "h0"))
    k = 5
    bb = Run(x[:, k:].contiguous(), full.out[:, k - 1].contiguous(), p, T - k, True, g0)
    assert torch.equal(bb.out, full.out[:, k:])
    bk = bb.kernel()
    for n in ("u", "r", "q", "s"):
        assert torch.equal(bk[n], fk[n][k:]), n
    assert torch.equal(bb.means, full.means[k:]) and torch.equal(bb.vars, full.vars[k:])
    gb = bb.backward(go[:, k:].contiguous(), ("x", "h0"))
    assert torch.equal(gb["x"], fg["x"][:, k:])
    a = Run(x[:, :k].contiguous(), h0, p, k, True, g0)
    assert torch.equal(a.out, full.out[:, :k]) and torch.equal(a.means, full.means[:k]) and torch.equal(a.vars, full.vars[:k])
    go_a = go[:, :k].clone()
    go_a[:, k - 1] += gb["h0"]
    ga = a.backward(go_a, ("x", "h0"))
    assert torch.equal(ga["h0"], fg["h0"]) and torch.equal(ga["x"], fg["x"][:, :k])
    assert full.guard.intact() and a.guard.intact() and bb.guard.intact()
