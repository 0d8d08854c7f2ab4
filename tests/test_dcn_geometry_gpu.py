"""GPU: the `mmdet.ops.dcn` operator surface (ops/dcn.py) in the geometries its signature accepts, against
oracle/torch_reference.py::deform_conv_ref evaluated in float64 on the device.

tests/test_conv_plans_gpu.py pins the detector's own DCN launches (3x3, stride 1, padding 1, 256 channels).  The cases
here walk the other axes pairwise: kernels 1x1 / 3x3 / 5x5 / 1x3 / 3x1, stride 1-3 and 257, padding 0-2, dilation 1-2, ragged,
1x1 and wider-than-128 output maps, Cin 3 to 256, Cout 1 to 300 (several N tiles), N = 1 / 3 / 5, DCNv1 and DCNv2 with
0/1 and random masks, bias on and off, and offsets that are random (many samples leave the image), integer, exactly on
the validity and corner boundaries, or NaN / +-inf.  Each case

- asserts the kernel it reaches (the tensor-core kernel in f16x3 or bf16, or the fp32 CUDA-core kernel), and on the
  tensor-core kernel the deformable plan it launched;
- runs twice: the results must be bitwise equal and finite (the path has no atomics, the inputs no NaN);
- is compared with the fp64 oracle (relative to the output's max), and with zero offsets and no mask also with
  F.conv2d in fp64 at the same stride / padding / dilation, an oracle independent of deform_conv_ref.

Module-level cases: the Pack modules with non-zero conv_offset weights, build_conv_layer('DCN') as mmdet's ResNet builds
conv2, the small-input pad-and-crop path of DeformConv.forward, the weight cache under address reuse, and the errors."""
import collections
import contextlib
import zlib

import pytest
import torch
import torch.nn.functional as F

from orientedreppoints_b200 import _lib

pytestmark = pytest.mark.gpu

FP32_TOL = 1e-5          # fp32 CUDA-core kernel: summation order only
F16X3_TOL = 2.5e-5       # f16x3 deformable (tests/test_conv_plans_gpu.py), scaled by max(1, K / 4096) as OP_TOL
BF16_TOL = 1.5e-2        # bf16 deformable: the sample is rounded to bf16 before the MMA

# api: deform_conv / modulated_deform_conv (functions) or the DeformConv / ModulatedDeformConv modules; prec: the
# set_precision mode; k: (KH, KW); s / p / d: stride / padding / dilation; off: offset pattern (_offsets); mask: None,
# "binary" or "random"; route: the kernel the case must reach ("f16x3" / "bf16" tensor core, "fp32" CUDA cores)
Case = collections.namedtuple("Case", "api prec n cin cout h w k s p d off mask bias route")
CASES = [
    # tensor core, f16x3
    Case("deform_conv", "f16x3", 3, 64, 96, 13, 17, (1, 1), 1, 0, 1, "random", None, False, "f16x3"),
    Case("modulated", "f16x3", 5, 192, 300, 23, 19, (3, 3), 2, 1, 1, "random", "random", True, "f16x3"),
    Case("DeformConv", "f16x3", 1, 64, 18, 9, 11, (5, 5), 1, 2, 1, "edges", None, False, "f16x3"),
    Case("modulated", "f16x3", 3, 256, 10, 12, 15, (1, 3), 2, 0, 1, "integer", "binary", False, "f16x3"),
    Case("deform_conv", "f16x3", 1, 64, 256, 20, 14, (3, 1), 3, 2, 1, "nonfinite", None, False, "f16x3"),
    Case("ModulatedDeformConv", "f16x3", 3, 64, 1, 10, 7, (3, 3), 1, 0, 1, "edges", "random", True, "f16x3"),
    Case("deform_conv", "f16x3", 5, 64, 96, 3, 3, (3, 3), 1, 0, 1, "random", None, False, "f16x3"),          # 1x1 map
    Case("deform_conv", "f16x3", 1, 64, 96, 9, 300, (3, 3), 2, 1, 1, "random", None, False, "f16x3"),        # Wo 150
    Case("modulated", "f16x3", 1, 64, 96, 7, 400, (3, 3), 3, 1, 1, "edges", "binary", True, "f16x3"),       # Wo 134, s 3
    Case("deform_conv", "f16x3", 3, 64, 96, 11, 9, (3, 3), 2, 1, 1, "zero", None, False, "f16x3"),
    Case("DeformConv", "f16x3", 5, 256, 256, 8, 6, (5, 5), 3, 2, 1, "nonfinite", None, False, "f16x3"),     # K 6400
    Case("modulated", "f16x3", 1, 192, 300, 5, 5, (5, 5), 3, 0, 1, "random", "random", True, "f16x3"),      # 1x1 map
    # tensor core, bf16
    Case("deform_conv", "bf16", 3, 64, 300, 15, 13, (3, 3), 2, 1, 1, "random", None, False, "bf16"),
    Case("modulated", "bf16", 5, 256, 18, 9, 10, (1, 3), 1, 1, 1, "edges", "binary", True, "bf16"),
    Case("ModulatedDeformConv", "bf16", 1, 192, 96, 12, 11, (3, 1), 3, 2, 1, "nonfinite", "random", False, "bf16"),
    Case("DeformConv", "bf16", 1, 64, 10, 6, 260, (5, 5), 2, 2, 1, "integer", None, False, "bf16"),         # Wo 130
    Case("deform_conv", "bf16", 3, 64, 1, 7, 9, (1, 1), 1, 1, 1, "zero", None, False, "bf16"),
    Case("modulated", "bf16", 1, 64, 256, 6, 400, (3, 3), 3, 0, 1, "random", "random", True, "bf16"),       # Wo 133, s 3
    # fp32 kernel: Cin % 64 != 0 (Cin 3, 18 and 30 are not multiples of 4 either)
    Case("DeformConv", "f16x3", 1, 3, 16, 12, 12, (3, 3), 1, 1, 1, "random", None, False, "fp32"),
    Case("modulated", "f16x3", 3, 8, 300, 11, 14, (3, 3), 2, 1, 1, "edges", "random", True, "fp32"),
    Case("ModulatedDeformConv", "bf16", 5, 24, 10, 9, 8, (1, 3), 3, 0, 1, "integer", "binary", True, "fp32"),
    Case("deform_conv", "f16x3", 3, 30, 96, 10, 13, (5, 5), 2, 2, 1, "nonfinite", None, False, "fp32"),
    Case("deform_conv", "bf16", 1, 18, 1, 7, 7, (3, 1), 1, 2, 1, "zero", None, False, "fp32"),
    # fp32 kernel: dilation 2
    Case("deform_conv", "f16x3", 3, 64, 96, 13, 12, (3, 3), 1, 2, 2, "random", None, False, "fp32"),
    Case("modulated", "bf16", 1, 256, 18, 11, 10, (3, 3), 2, 1, 2, "edges", "random", True, "fp32"),
    Case("DeformConv", "f16x3", 5, 24, 10, 9, 9, (5, 5), 1, 0, 2, "integer", None, False, "fp32"),          # 1x1 map
    Case("deform_conv", "f16x3", 3, 64, 256, 10, 9, (3, 1), 1, 2, 2, "zero", None, False, "fp32"),
    Case("ModulatedDeformConv", "f16x3", 1, 192, 300, 8, 140, (3, 3), 3, 2, 2, "nonfinite", "binary", True, "fp32"),
    # fp32 kernel: set_precision('fp32')
    Case("deform_conv", "fp32", 3, 64, 96, 12, 11, (3, 3), 2, 1, 1, "random", None, False, "fp32"),
    Case("modulated", "fp32", 5, 256, 10, 7, 8, (5, 5), 1, 2, 1, "edges", "random", True, "fp32"),
    Case("DeformConv", "fp32", 1, 192, 300, 9, 260, (1, 1), 2, 0, 1, "nonfinite", None, False, "fp32"),     # Wo 130
    Case("modulated", "fp32", 3, 3, 18, 6, 5, (3, 3), 3, 1, 2, "integer", "binary", False, "fp32"),
    Case("deform_conv", "fp32", 1, 8, 1, 4, 4, (3, 3), 1, 0, 1, "zero", None, False, "fp32"),
    # fp32 kernel: a stride beyond the tensor-core tile's 256 input columns
    Case("modulated", "f16x3", 3, 64, 96, 300, 520, (3, 3), 257, 1, 1, "random", "random", True, "fp32"),   # 2x3 map
]


def _case_id(c):
    return "%s-%s-n%d-%dx%d-%dx%d-k%dx%d-s%dp%dd%d-%s-%s%s" % (
        c.route, c.api, c.n, c.cin, c.cout, c.h, c.w, c.k[0], c.k[1], c.s, c.p, c.d, c.off, c.mask or "v1",
        "-bias" if c.bias else "")


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / (b.double().abs().max() + 1e-30))


def _out_hw(h, w, k, s, p, d):
    return (h + 2 * p - d * (k[0] - 1) - 1) // s + 1, (w + 2 * p - d * (k[1] - 1) - 1) // s + 1


def _offsets(mode, n, h, w, k, s, p, d, g):
    """[N, 2*KH*KW, Ho, Wo] (dy, dx) per tap.  "edges": every sample lands exactly on a row of {-1, -0.5, 0, 0.5, H-1.5,
    H-1, H-0.5, H} or on the half-integer grid inside, and likewise for columns - the validity and corner tests of the
    bilinear sample at their boundaries.  "nonfinite": random with 5 % each NaN, +inf and -inf"""
    ho, wo = _out_hw(h, w, k, s, p, d)
    shape = (n, 2 * k[0] * k[1], ho, wo)
    if mode == "zero":
        return torch.zeros(shape)
    if mode == "random":
        return torch.randn(shape, generator=g) * 3.0
    if mode == "integer":
        return torch.randint(-3, 4, shape, generator=g).float()
    if mode == "nonfinite":
        off = torch.randn(shape, generator=g) * 3.0
        r = torch.rand(shape, generator=g)
        off[r < 0.05] = float("nan")
        off[(r >= 0.05) & (r < 0.10)] = float("inf")
        off[(r >= 0.10) & (r < 0.15)] = -float("inf")
        return off
    assert mode == "edges"

    def targets(size, shp):
        pick = torch.tensor([-1.0, -0.5, 0.0, 0.5, size - 1.5, size - 1.0, size - 0.5, float(size)])
        t = pick[torch.randint(0, len(pick), shp, generator=g)]
        inner = torch.randint(0, 2 * size, shp, generator=g).float() * 0.5 - 0.5
        return torch.where(torch.rand(shp, generator=g) < 0.75, t, inner)

    off = torch.empty(shape)
    hh = torch.arange(ho).view(1, ho, 1).float() * s - p
    ww = torch.arange(wo).view(1, 1, wo).float() * s - p
    for t in range(k[0] * k[1]):
        i, j = divmod(t, k[1])
        off[:, 2 * t] = targets(h, (n, ho, wo)) - (hh + i * d)
        off[:, 2 * t + 1] = targets(w, (n, ho, wo)) - (ww + j * d)
    return off


def _oracle(x, off, wt, s, p, d, mask=None, bias=None):
    """deform_conv_ref in fp64 on the device (+ bias), at the sample positions the reference's im2col forms: the tap's
    integer base position plus the offset, rounded to fp32 (deform_conv_cuda_kernel.cu computes h_im / w_im in the
    tensor's type; at 260 columns one fp32 ulp moves a bilinear weight by 3e-5).  A NaN or infinite offset fails the
    sample's validity test, so the tap adds 0; deform_conv_ref would carry the NaN through its bilinear weights, so such
    offsets are replaced by one far outside the image, which fails the same test"""
    from oracle import torch_reference as tr
    kh, kw = wt.shape[2:]
    ho, wo = off.shape[2:]
    hb = (torch.arange(ho, device=off.device) * s - p).view(1, ho, 1).double()
    wb = (torch.arange(wo, device=off.device) * s - p).view(1, 1, wo).double()
    pos = off.double().clone()
    for t in range(kh * kw):
        i, j = divmod(t, kw)
        for c, base in ((2 * t, hb + i * d), (2 * t + 1, wb + j * d)):
            pos[:, c] = (base.float() + off[:, c].float()).double() - base     # base + pos = fl32(base + offset) in fp64
    off = torch.where(torch.isfinite(pos), pos, torch.full_like(pos, -1e4))
    y = tr.deform_conv_ref(x.double(), off, wt.double(), s, p, d, mask=None if mask is None else mask.double())
    if bias is not None:
        y = y + bias.double().view(1, -1, 1, 1)
    return y


def _tol(c):
    if c.route == "fp32":
        return FP32_TOL
    if c.route == "f16x3":
        return F16X3_TOL * max(1.0, c.cin * c.k[0] * c.k[1] / 4096.0)
    return BF16_TOL


@pytest.fixture
def routes(monkeypatch):
    """records the kernel every deformable launch of ops/dcn.py reaches: ("f16x3" | "bf16", plan) for the tensor-core
    kernel, ("fp32", None) for orp_deform_conv2d_f32"""
    from orientedreppoints_b200.engine_tc import EngineTC, EngineTCSplit
    seen = []

    def wrap(cls):
        orig = cls._launch

        def launch(self, *a, **kw):
            orig(self, *a, **kw)
            seen.append((self.name, _lib.tc_last_plan()))
        monkeypatch.setattr(cls, "_launch", launch)
    wrap(EngineTC)
    wrap(EngineTCSplit)
    lib = _lib.lib()
    f32 = lib.orp_deform_conv2d_f32

    def f32_launch(*a):
        seen.append(("fp32", None))
        return f32(*a)
    monkeypatch.setattr(lib, "orp_deform_conv2d_f32", f32_launch)
    return seen


@contextlib.contextmanager
def _precision(p):
    from orientedreppoints_b200.ops import dcn
    dcn.set_precision(p)
    try:
        yield
    finally:
        dcn.set_precision("f16x3")


def _check_route(seen, route, cout=None, stride=None, bias=None):
    assert [r for r, _ in seen] == [route], "expected one %s launch, got %s" % (route, [r for r, _ in seen])
    plan = seen[0][1]
    if plan is None:
        return
    assert plan["deform"] == 1 and plan["split"] == int(route == "f16x3") and plan["out_f32"] == 1
    if cout is not None:
        assert plan["Cout"] == cout and plan["bias"] == int(bool(bias))
        if cout > 128:
            assert plan["n_tiles_n"] > 1                 # the A operand is sampled once per N tile
    if stride is not None:
        bw = plan["BW"][0]
        assert bw & (bw - 1) == 0 and bw * stride <= 256, plan


def _twice(fn, seen):
    """two calls: bitwise equal, finite; the kernel reached by the first"""
    outs, first = [], None
    for _ in range(2):
        seen.clear()
        with torch.no_grad():
            outs.append(fn())
        torch.cuda.synchronize()
        first = first if first is not None else list(seen)
    a, b = outs
    assert a.dtype == torch.float32 and a.is_contiguous()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "two calls differ"
    assert bool(torch.isfinite(a).all()), "non-finite output"
    return a, first


# ---------------------------------------------------------------------------------------------------------------- matrix
WORST = {}


@pytest.mark.parametrize("c", CASES, ids=[_case_id(c) for c in CASES])
def test_dcn_geometry(cuda, routes, c):
    from orientedreppoints_b200.ops import DeformConv, ModulatedDeformConv, deform_conv, modulated_deform_conv
    g = torch.Generator().manual_seed(zlib.crc32(_case_id(c).encode()))
    K = c.cin * c.k[0] * c.k[1]
    x = torch.randn(c.n, c.cin, c.h, c.w, generator=g).to(cuda)
    wt = (torch.randn(c.cout, c.cin, *c.k, generator=g) / K ** 0.5).to(cuda)
    off = _offsets(c.off, c.n, c.h, c.w, c.k, c.s, c.p, c.d, g).to(cuda)
    ho, wo = off.shape[2:]
    mask = None
    if c.mask == "binary":
        mask = torch.randint(0, 2, (c.n, c.k[0] * c.k[1], ho, wo), generator=g).float().to(cuda)
    elif c.mask == "random":
        mask = torch.rand(c.n, c.k[0] * c.k[1], ho, wo, generator=g).to(cuda)
    bias = (torch.randn(c.cout, generator=g) * 0.5).to(cuda) if c.bias else None
    assert c.api in ("modulated", "ModulatedDeformConv") or (mask is None and bias is None)

    if c.api == "deform_conv":
        fn = lambda: deform_conv(x, off, wt, c.s, c.p, c.d)                          # noqa: E731
    elif c.api == "modulated":
        fn = lambda: modulated_deform_conv(x, off, mask, wt, bias, c.s, c.p, c.d)    # noqa: E731
    elif c.api == "DeformConv":
        m = DeformConv(c.cin, c.cout, c.k, c.s, c.p, c.d).to(cuda)
        with torch.no_grad():
            m.weight.copy_(wt)
        fn = lambda: m(x, off)                                                        # noqa: E731
    else:
        m = ModulatedDeformConv(c.cin, c.cout, c.k, c.s, c.p, c.d, bias=c.bias).to(cuda)
        with torch.no_grad():
            m.weight.copy_(wt)
            if c.bias:
                m.bias.copy_(bias)
        fn = lambda: m(x, off, mask)                                                  # noqa: E731

    with _precision(c.prec):
        y, seen = _twice(fn, routes)
        if c.route == "f16x3":
            from orientedreppoints_b200.engine_tc import EngineTCSplit
            assert EngineTCSplit(cuda).overflow_count() == 0
    _check_route(seen, c.route, c.cout, c.s, c.bias)
    assert tuple(y.shape) == (c.n, c.cout, ho, wo)
    ref = _oracle(x, off, wt, c.s, c.p, c.d, mask, bias)
    err, tol = _rel(y, ref), _tol(c)
    if c.off == "zero" and mask is None:
        plain = F.conv2d(x.double(), wt.double(), None, c.s, c.p, c.d)
        assert _rel(ref, plain) < 1e-12                                  # the two oracles agree
        err = max(err, _rel(y, plain))
    WORST[c.route] = max(WORST.get(c.route, 0.0), err)
    print("%s: rel err %.2e (tol %.1e); worst %s so far %.2e" % (_case_id(c), err, tol, c.route, WORST[c.route]))
    assert err < tol, (err, tol)


# --------------------------------------------------------------------------------------------------------------- modules
def _capture(module):
    """forward hook: the output of module's conv_offset, as the DCN layer received it"""
    got = []
    module.conv_offset.register_forward_hook(lambda mod, inp, out: got.append(out.detach().clone()))
    return got


@pytest.mark.parametrize("cin,route", [(64, "f16x3"), (24, "fp32")])
@pytest.mark.parametrize("modulated", [False, True], ids=["DeformConvPack", "ModulatedDeformConvPack"])
def test_pack_modules_with_learned_offsets(cuda, routes, cin, route, modulated):
    """non-zero conv_offset weights at stride 2: the offsets (and sigmoid mask) come from the module's own conv_offset
    output, captured as the module used it, so torch's convolution arithmetic (TF32) does not enter the comparison -
    what is checked is the chunk -> cat -> sigmoid plumbing and the DCN launch"""
    from orientedreppoints_b200.ops import DeformConvPack, ModulatedDeformConvPack
    g = torch.Generator().manual_seed(11 + cin)
    cls = ModulatedDeformConvPack if modulated else DeformConvPack
    m = cls(cin, 96, 3, stride=2, padding=1).to(cuda)
    with torch.no_grad():
        m.conv_offset.weight.copy_(torch.randn(m.conv_offset.weight.shape, generator=g) * (2.0 / (cin * 9) ** 0.5))
        m.conv_offset.bias.copy_(torch.randn(m.conv_offset.bias.shape, generator=g) * 0.5)
        if modulated:
            m.bias.copy_(torch.randn(96, generator=g) * 0.5)
    got = _capture(m)
    x = torch.randn(3, cin, 21, 26, generator=g).to(cuda)
    y, seen = _twice(lambda: m(x), routes)
    _check_route(seen, route, 96, 2, modulated)
    assert len(got) == 2 and torch.equal(got[0], got[1])
    out = got[0].double()
    if modulated:
        o1, o2, mk = torch.chunk(out, 3, dim=1)
        ref = _oracle(x, torch.cat((o1, o2), dim=1), m.weight.detach(), 2, 1, 1, torch.sigmoid(mk), m.bias.detach())
    else:
        ref = _oracle(x, out, m.weight.detach(), 2, 1, 1)
    assert float(out.abs().max()) > 2.0                               # the offsets do move the samples
    assert _rel(y, ref) < (F16X3_TOL if route == "f16x3" else FP32_TOL)


def test_build_conv_layer_dcn_as_resnet_conv2(cuda, routes):
    """build_conv_layer(dict(type='DCN'), 128, 128, 3, stride=2, padding=1, bias=False): mmdet ResNet's conv2 with DCN.
    Freshly built (zero conv_offset) it is the plain strided convolution; with learned offsets, the deformable one"""
    from orientedreppoints_b200.ops import DeformConvPack, build_conv_layer
    g = torch.Generator().manual_seed(5)
    m = build_conv_layer(dict(type='DCN'), 128, 128, 3, stride=2, padding=1, bias=False).to(cuda)
    assert isinstance(m, DeformConvPack)
    x = torch.randn(2, 128, 25, 31, generator=g).to(cuda)
    y, seen = _twice(lambda: m(x), routes)
    _check_route(seen, "f16x3", 128, 2, False)
    plain = F.conv2d(x.double(), m.weight.detach().double(), None, 2, 1)
    assert tuple(y.shape) == (2, 128, 13, 16) and _rel(y, plain) < F16X3_TOL
    with torch.no_grad():
        m.conv_offset.weight.copy_(torch.randn(m.conv_offset.weight.shape, generator=g) * (2.0 / (128 * 9) ** 0.5))
    got = _capture(m)
    y, _ = _twice(lambda: m(x), routes)
    assert _rel(y, _oracle(x, got[0], m.weight.detach(), 2, 1, 1)) < F16X3_TOL


@pytest.mark.parametrize("cin,h,w,k,p,s", [(64, 2, 2, 3, 1, 1), (64, 4, 2, 3, 1, 1), (3, 1, 3, 3, 1, 1), (64, 3, 3, 5, 2, 1),
                                           (64, 2, 2, 3, 1, 2)])
def test_small_input_pad_and_crop(cuda, routes, cin, h, w, k, p, s):
    """an input smaller than the kernel is zero padded on the right / bottom (offsets too) and the output cropped back
    (deform_conv.py:239-255): the values are the oracle's on the padded input, cropped the same way"""
    from orientedreppoints_b200.ops import DeformConv
    g = torch.Generator().manual_seed(cin + h * 10 + w + k + s)
    m = DeformConv(cin, 32, k, stride=s, padding=p).to(cuda)
    ho, wo = _out_hw(h, w, (k, k), s, p, 1)
    x = torch.randn(2, cin, h, w, generator=g).to(cuda)
    off = (torch.randn(2, 2 * k * k, ho, wo, generator=g) * 1.5).to(cuda)
    ph, pw = max(k - h, 0), max(k - w, 0)
    y, seen = _twice(lambda: m(x, off), routes)
    _check_route(seen, "f16x3" if cin % 64 == 0 else "fp32", 32, s, False)
    ref = _oracle(F.pad(x, (0, pw, 0, ph)), F.pad(off, (0, pw, 0, ph)), m.weight.detach(), s, p, 1)
    ref = ref[:, :, :ref.shape[2] - ph, :ref.shape[3] - pw]
    assert y.shape == ref.shape
    assert _rel(y, ref) < (F16X3_TOL if cin % 64 == 0 else FP32_TOL)


def test_any_cin_on_the_fp32_kernel(cuda, routes):
    """DeformConv(3, 16, 3, padding=1) - a 3-channel input, as a DCN stem would see it - in every precision mode: the
    channels are zero-padded to 4 for the fp32 kernel, the result is the 3-channel convolution's"""
    from orientedreppoints_b200.ops import DeformConv
    g = torch.Generator().manual_seed(3)
    m = DeformConv(3, 16, 3, padding=1).to(cuda)
    x = torch.randn(2, 3, 17, 19, generator=g).to(cuda)
    off = (torch.randn(2, 18, 17, 19, generator=g) * 3.0).to(cuda)
    ref = _oracle(x, off, m.weight.detach(), 1, 1, 1)
    for prec in ("f16x3", "bf16", "fp32"):
        with _precision(prec):
            y, seen = _twice(lambda: m(x, off), routes)
        _check_route(seen, "fp32")
        assert _rel(y, ref) < FP32_TOL


def test_weight_cache_follows_the_tensor(cuda, routes):
    """a weight freed and a new one of the same shape and version allocated after it must not be served the first
    one's cached layout, on either kernel.  The weights live in a private memory pool, where the second one would land
    exactly where the first one was; the cache entry keeps the first one's memory, so it lands elsewhere"""
    from orientedreppoints_b200.ops import deform_conv
    g = torch.Generator().manual_seed(9)
    for cin in (64, 24):
        x = torch.randn(1, cin, 9, 10, generator=g).to(cuda)
        off = torch.randn(1, 18, 9, 10, generator=g).to(cuda)
        pool = torch.cuda.MemPool()
        with torch.cuda.use_mem_pool(pool):
            w1 = torch.randn(32, cin, 3, 3, generator=g).to(cuda)
        ptr, version = w1.data_ptr(), w1._version
        with torch.no_grad():
            deform_conv(x, off, w1, 1, 1)
        torch.cuda.synchronize()
        del w1
        with torch.cuda.use_mem_pool(pool):
            w2 = torch.randn(32, cin, 3, 3, generator=g).to(cuda)
        assert w2._version == version and w2.data_ptr() != ptr
        y, seen = _twice(lambda: deform_conv(x, off, w2, 1, 1), routes)
        _check_route(seen, "f16x3" if cin == 64 else "fp32")
        assert _rel(y, _oracle(x, off, w2, 1, 1, 1)) < F16X3_TOL
        del w2


def test_geometry_errors(cuda):
    """non-square stride / padding / dilation, groups and deformable_groups > 1: NotImplementedError; offset or mask of
    the wrong shape: RuntimeError (deform_conv_cuda.cpp:130-136)"""
    from orientedreppoints_b200.ops import DeformConv, deform_conv, modulated_deform_conv
    x = torch.randn(2, 64, 8, 9, device=cuda)
    wt = torch.randn(32, 64, 3, 3, device=cuda)
    off = torch.zeros(2, 18, 8, 9, device=cuda)
    mask = torch.ones(2, 9, 8, 9, device=cuda)
    for s, p, d in [((1, 2), 1, 1), (1, (1, 0), 1), (1, 1, (1, 2)), (1, (0, 1), 1)]:
        with pytest.raises(NotImplementedError):
            deform_conv(x, off, wt, s, p, d)
        with pytest.raises(NotImplementedError):
            modulated_deform_conv(x, off, mask, wt, None, s, p, d)
    with pytest.raises(NotImplementedError):
        deform_conv(x, off, wt[:, :32], 1, 1, 1, 2, 1)                    # groups = 2
    with pytest.raises(NotImplementedError):
        deform_conv(x, torch.zeros(2, 36, 8, 9, device=cuda), wt, 1, 1, 1, 1, 2)   # deformable_groups = 2
    with pytest.raises(NotImplementedError):
        modulated_deform_conv(x, off, mask, wt, None, 1, 1, 1, 1, 2)
    with pytest.raises(NotImplementedError):
        DeformConv(64, 32, 3, stride=(2, 1), padding=1).to(cuda)(x, torch.zeros(2, 18, 4, 9, device=cuda))
    for bad in [(2, 16, 8, 9), (2, 18, 8, 8), (2, 18, 7, 9), (1, 18, 8, 9), (2, 18, 4, 5)]:
        with pytest.raises(RuntimeError):
            deform_conv(x, torch.zeros(bad, device=cuda), wt, 1, 1)
    for bad in [(2, 8, 8, 9), (2, 9, 8, 8), (1, 9, 8, 9), (2, 18, 8, 9)]:
        with pytest.raises(RuntimeError):
            modulated_deform_conv(x, off, torch.ones(bad, device=cuda), wt, None, 1, 1)
    # the same offset map is the right one at stride 2
    assert tuple(deform_conv(x, torch.zeros(2, 18, 4, 5, device=cuda), wt, 2, 1).shape) == (2, 32, 4, 5)
