"""FPN_CARAFE on the H100 (include/orp_b200_carafe.h, carafe_fpn.py): every orp_carafe_add launch shape of R-50 FPN_CARAFE at
16 x 1024^2, 1 x 1024^2 and 4 x 960^2 and of Swin-T at 8 x 1024^2 against the fp64 contract in all three formats, with
up_kernel 3 / 5 / 7, up_group 1 / 4 and peaked logits; one-hot logits pinning the shuffle, tap, group and border mapping; the
new convolution plans launched against fp64 and the launch checker over R-50 FPN_CARAFE; whole R-50 and Swin-T necks against
the fp64 graph; bitwise reruns, capture with aug_test, init_detector from checkpoints on ResNet, ResNeXt and Swin, and the
entry point on a side stream and from two host threads."""
import threading
import time

import pytest
import torch

from orientedreppoints_b200 import _lib
from orientedreppoints_b200 import carafe_fpn as cf
from orientedreppoints_b200.detector import EngineF32, OrientedRepPointsDetector
from orientedreppoints_b200.swin import random_swin_state_dict
from orientedreppoints_b200.weights import fpn_carafe_spec, random_state_dict
import fpn_carafe_ref as fr
from test_fpn_carafe_cpu import CARAFE_PARITY

pytestmark = pytest.mark.gpu
FORMATS = ["f16x3", "bf16", "fp32"]
TOL = {"f16x3": 1e-4, "fp32": 1e-4, "bf16": 1.5e-2}
GN = dict(type='GN', num_groups=32, requires_grad=True)


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    d = torch.device("cuda", 0)
    torch.cuda.set_device(d)
    return d


def _engine(fmt, dev):
    if fmt == "fp32":
        return EngineF32(dev)
    from orientedreppoints_b200.engine_tc import EngineTC, EngineTCSplit
    return EngineTCSplit(dev) if fmt == "f16x3" else EngineTC(dev)


def _held(e, t):
    """t (fp32 NHWC on the device) in the engine's format, and the exact values it holds (fp64)"""
    if e.name == "fp32":
        y = t.contiguous()
        return y, y.double()
    y = e.from_float(t)
    return y, e.to_float(y).double()


def _f(e, y):
    return (y if e.name == "fp32" else e.to_float(y)).double()


def _contract(x64, logits, k, g, r64, j):
    """fp64 carafe_add of image j (NHWC in, NCHW out)"""
    nchw = lambda t: t[j:j + 1].double().permute(0, 3, 1, 2)               # noqa: E731
    return fr.carafe_add(nchw(x64), nchw(logits), k, g, nchw(r64))


def _rel(a, b):
    return float((a - b).abs().max()) / max(1e-30, float(b.abs().max()))


def _launch_case(e, dev, n, h, w, hr, wr, k, g, scale, seed, c=256):
    gen = torch.Generator(device=dev).manual_seed(seed)
    x, x64 = _held(e, torch.randn(n, h, w, c, device=dev, generator=gen))
    r, r64 = _held(e, torch.randn(n, hr, wr, c, device=dev, generator=gen))
    logits = (scale * torch.randn(n, h, w, k * k * g * 4, device=dev, generator=gen)).contiguous()
    return x, x64, r, r64, logits


# (N, H, W, Hr, Wr) of every orp_carafe_add of the workloads: the four top-down steps, coarsest first
def _shapes(n, hw):
    s = fr.level_sizes(hw, hw)
    return [(n,) + s[i + 1] + s[i] for i in (3, 2, 1, 0)]


WORKLOADS = {"r50_16x1024": _shapes(16, 1024), "r50_1x1024": _shapes(1, 1024), "r50_4x960": _shapes(4, 960),
             "swin_t_8x1024": _shapes(8, 1024)}
LAUNCHES = [(wl, i) for wl in WORKLOADS for i in range(4)]
# (k, G, logit scale): the default, the other kernels and groups, and peaked logits
VARIANTS = [(5, 1, 1.0), (3, 4, 1.0), (7, 1, 1.0), (7, 4, 1.0), (5, 1, 8.0), (3, 1, 8.0)]


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("wl,i", LAUNCHES, ids=["%s-%d" % l for l in LAUNCHES])
def test_launches_vs_fp64(dev, fmt, wl, i):
    e = _engine(fmt, dev)
    n, h, w, hr, wr = WORKLOADS[wl][i]
    variants = VARIANTS if (wl, i) in (("r50_4x960", 0), ("r50_4x960", 1), ("r50_16x1024", 3)) else VARIANTS[:1]
    for vi, (k, g, scale) in enumerate(variants):
        x, x64, r, r64, logits = _launch_case(e, dev, n, h, w, hr, wr, k, g, scale, seed=100 * i + vi)
        if fmt == "f16x3":
            e.overflow_count()
        y = cf.carafe_add(e, x, logits, k, g, r)
        got = _f(e, y)
        for j in sorted({0, n - 1}):                                 # the first and the last image
            ref = _contract(x64, logits, k, g, r64, j)
            err = _rel(got[j:j + 1].permute(0, 3, 1, 2), ref)
            assert err < TOL[fmt], "%s %s launch %d k %d G %d scale %g image %d: rel err %.3e" % (fmt, wl, i, k, g, scale, j, err)
        if fmt == "f16x3":
            assert e.overflow_count() == 0
        again = cf.carafe_add(e, x, logits, k, g, r)
        assert torch.equal(again, y)                                   # no atomics: bitwise reruns


@pytest.mark.parametrize("fmt", ["f16x3", "fp32"])
@pytest.mark.parametrize("k,g,h,w,hr,wr", [(5, 1, 8, 8, 15, 15), (3, 4, 15, 15, 30, 30), (7, 4, 8, 8, 16, 16), (1, 2, 5, 7, 9, 14)])
def test_one_hot_logits(dev, fmt, k, g, h, w, hr, wr):
    """a margin of 60 on one tap per (output pixel, group): y = the chosen neighbour (0 outside the map) + residual"""
    e = _engine(fmt, dev)
    n, c = 2, 64
    gen = torch.Generator(device=dev).manual_seed(k * 10 + g)
    x, x64 = _held(e, torch.randn(n, h, w, c, device=dev, generator=gen))
    r, r64 = _held(e, torch.randn(n, hr, wr, c, device=dev, generator=gen))
    tap = torch.randint(0, k * k, (n, 2 * h, 2 * w, g), device=dev, generator=gen)
    logits = torch.zeros(n, h, w, g, k * k, 2, 2, device=dev)
    for oy in range(2):
        for ox in range(2):
            sel = tap[:, oy::2, ox::2]                                    # [n, h, w, g]
            logits[:, :, :, :, :, oy, ox].scatter_(4, sel.unsqueeze(-1), 60.0)
    y = _f(e, cf.carafe_add(e, x, logits.reshape(n, h, w, -1).contiguous(), k, g, r))
    rad = (k - 1) // 2
    oy, ox = torch.meshgrid(torch.arange(hr, device=dev), torch.arange(wr, device=dev), indexing="ij")
    want = r64.clone()
    for gi in range(g):
        t = tap[:, :hr, :wr, gi]
        iy, ix = oy // 2 + t // k - rad, ox // 2 + t % k - rad
        inside = (iy >= 0) & (iy < h) & (ix >= 0) & (ix < w)
        nb = x64[torch.arange(n, device=dev).view(n, 1, 1), iy.clamp(0, h - 1), ix.clamp(0, w - 1)]     # [n, hr, wr, c]
        cs = slice(gi * c // g, (gi + 1) * c // g)
        want[..., cs] += torch.where(inside.unsqueeze(-1), nb[..., cs], torch.zeros_like(nb[..., cs]))
    assert _rel(y, want) < 1e-6


def test_refusals_on_device(dev):
    lib = _lib.lib()
    x = torch.zeros(1, 4, 4, 2, 256, dtype=torch.float16, device=dev)
    r = torch.zeros(1, 8, 8, 2, 256, dtype=torch.float16, device=dev)
    y = torch.zeros_like(r)
    lg = torch.zeros(1, 4, 4, 100, device=dev)
    p = _lib.ptr
    assert lib.orp_carafe_add_f16x3(p(x), 1, 4, 4, 256, p(lg), 5, 1, p(r), 8, 8, p(y), None) == 0
    torch.cuda.synchronize()
    for args in ((4, 1, 8, 8), (5, 3, 8, 8), (5, 1, 9, 8), (5, 1, 8, 0), (9, 1, 8, 8)):
        k, g, hr, wr = args
        assert lib.orp_carafe_add_f16x3(p(x), 1, 4, 4, 256, p(lg), k, g, p(r), hr, wr, p(y), None) == -1, args
    assert lib.orp_carafe_add_f16x3(p(x), 1, 4, 4, 256, p(lg), 5, 1, p(r), 8, 8, p(r), None) == -1       # y is the residual
    assert lib.orp_carafe_add_f16x3(p(x), 1, 4, 4, 12, p(lg), 5, 1, p(r), 8, 8, p(y), None) == -1        # C % 8


# ------------------------------------------------------------------------------------------------ whole necks
def _neck_spec(swin=False, **kw):
    return fpn_carafe_spec((192, 384, 768) if swin else (512, 1024, 2048), 256, kw.pop("norm_cfg", GN), **kw)


def _det(kind, fmt, dev, spec=None, seed=0):
    spec = spec or _neck_spec(kind == "swin")
    if kind == "swin":
        sd = random_swin_state_dict(seed, neck=spec, carafe_gain=fr.CARAFE_GAIN)
        return OrientedRepPointsDetector(sd, "swin_tiny", dev, fmt, test_cfg=dict(score_thr=0.02), neck=spec), sd, spec
    extra = dict(groups=32, base_width=4) if kind == "x50" else {}
    sd = random_state_dict(50, seed=seed, reference_init=False, residual_gain=0.5, neck=spec, carafe_gain=fr.CARAFE_GAIN, **extra)
    return OrientedRepPointsDetector(sd, 50, dev, fmt, test_cfg=dict(score_thr=0.02), neck=spec), sd, spec


def _backbone_feats(det, img):
    """the backbone's stride-8, -16 and -32 outputs of det's own pass, captured at the neck's input"""
    got, real = [], det.neck

    def recording(e, feats):
        got.extend(feats)
        return real(e, feats)
    det.neck = recording
    try:
        outs, levels = det.forward_dense(img)
    finally:
        det.neck = real
    return got, outs, levels


@pytest.mark.parametrize("kind", ["r50", "swin"])
@pytest.mark.parametrize("fmt", FORMATS)
def test_whole_neck_vs_fp64(dev, kind, fmt):
    """the five levels against the fp64 neck on the backbone outputs the engine holds: f16x3 and fp32 within 1e-4, bf16 within
    0.06; no f16x3 overflow"""
    if kind == "swin" and fmt == "fp32":
        pytest.skip("the Swin backbones run on the tensor-core engines")
    det, sd, spec = _det(kind, fmt, dev)
    hw = (224, 224) if kind == "swin" else (256, 320)
    img = torch.randn(2, 3, *hw, generator=torch.Generator().manual_seed(3)).to(dev)
    if fmt == "f16x3":
        det.eng.overflow_count()
    feats, outs, levels = _backbone_feats(det, img)
    sd64 = {k: v.double().to(dev) for k, v in sd.items() if k.startswith("neck.")}
    ref = fr.neck(sd64, spec, [_f(det.eng, f).permute(0, 3, 1, 2) for f in feats])
    tol = 0.06 if fmt == "bf16" else 1e-4
    for lv, (a, b) in enumerate(zip(levels, ref)):
        err = _rel(_f(det.eng, a).permute(0, 3, 1, 2), b)
        assert err < tol, "%s %s level %d: rel err %.3e" % (kind, fmt, lv, err)
    if fmt == "f16x3":
        assert det.eng.overflow_count() == 0
    assert len(det.simple_test(img, rescale=False)) == 2


def test_no_norm_relu_neck_vs_fp64(dev):
    spec = _neck_spec(norm_cfg=None, act_cfg=dict(type='ReLU'), upsample_cfg=dict(type='carafe', up_kernel=3, up_group=4,
                                                                                    encoder_kernel=1, compressed_channels=32))
    det, sd, spec = _det("r50", "f16x3", dev, spec)
    img = torch.randn(1, 3, 240, 240, generator=torch.Generator().manual_seed(4)).to(dev)
    feats, outs, levels = _backbone_feats(det, img)
    sd64 = {k: v.double().to(dev) for k, v in sd.items() if k.startswith("neck.")}
    ref = fr.neck(sd64, spec, [_f(det.eng, f).permute(0, 3, 1, 2) for f in feats])
    for a, b in zip(levels, ref):
        assert _rel(_f(det.eng, a).permute(0, 3, 1, 2), b) < 1e-4


@pytest.mark.parametrize("fmt", FORMATS)
def test_two_runs_bitwise_equal(dev, fmt):
    det, _, _ = _det("r50", fmt, dev)
    img = torch.randn(2, 3, 256, 256, generator=torch.Generator().manual_seed(5)).to(dev)
    a = [t.clone() for t in det.forward_dense(img)[1]]
    b = det.forward_dense(img)[1]
    for x, y in zip(a, b):
        if fmt == "fp32":          # the fp32 engine's GroupNorm statistics accumulate with atomics: equal to rounding only
            assert torch.allclose(x, y, rtol=1e-5, atol=1e-5 * float(x.abs().max()))
        else:
            assert torch.equal(x, y)


def test_capture_and_aug_test(dev):
    det, _, _ = _det("r50", "f16x3", dev)
    img = torch.randn(2, 3, 256, 256, generator=torch.Generator().manual_seed(6)).to(dev)
    eager = [x[0].clone() for x in det.forward_dense(img)[0]]
    det.capture(tuple(img.shape))
    outs, _ = det.forward_dense_graph(img)
    for a, b in zip(eager, [o[0] for o in outs]):
        assert torch.equal(a, b)
    small = torch.nn.functional.interpolate(img, size=(120, 120))          # 960-like: cut maps at the coarse levels
    metas = [[dict(img_shape=(256, 256, 3), scale_factor=1.0, flip=False)] * 2,
             [dict(img_shape=(120, 120, 3), scale_factor=120 / 256, flip=False)] * 2]
    assert len(det.aug_test([img, small], metas)) == 2
    outs2, _ = det.forward_dense_graph(img)
    for a, b in zip(eager, [o[0] for o in outs2]):
        assert torch.equal(a, b)


@pytest.mark.parametrize("prec", FORMATS)
@pytest.mark.parametrize("variant", ["resnet", "resnext", "swin"])
def test_init_detector_with_checkpoint(dev, tmp_path, prec, variant):
    """a config with neck=dict(type='FPN_CARAFE', ...) through init_detector (a checkpoint with the reference's keys),
    simple_test and uint8 inference_detector"""
    import os
    from orientedreppoints_b200.apis import Config, inference_detector, init_detector
    if variant == "swin" and prec == "fp32":
        pytest.skip("the Swin backbones run on the tensor-core engines")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    name = "orientedrepoints_swin_tiny_demo.py" if variant == "swin" else "orientedrepoints_r50_demo.py"
    cfg = Config.fromfile(os.path.join(root, "configs", "dota", name))
    widths = [192, 384, 768] if variant == "swin" else [256, 512, 1024, 2048]
    cfg['model']['neck'] = dict(type='FPN_CARAFE', in_channels=widths, out_channels=256, num_outs=5,
                                start_level=0 if variant == "swin" else 1, norm_cfg=GN)
    if variant == "resnext":
        cfg['model']['backbone'] = dict(cfg['model']['backbone'], type='ResNeXt', groups=32, base_width=4)
    cfg['model']['pretrained'] = None
    spec = _neck_spec(variant == "swin")
    if variant == "swin":
        sd = random_swin_state_dict(9, neck=spec, carafe_gain=fr.CARAFE_GAIN)
    else:
        sd = random_state_dict(50, seed=9, reference_init=False, residual_gain=0.5, neck=spec, carafe_gain=fr.CARAFE_GAIN,
                               **(dict(groups=32, base_width=4) if variant == "resnext" else {}))
    ck = tmp_path / "ck.pth"
    torch.save(dict(state_dict=sd), str(ck))
    m = init_detector(cfg, str(ck), device="cuda:0", precision=prec)
    key = "neck.upsample_modules.3.content_encoder.bias"
    assert torch.equal(m.state_dict()[key].cpu(), sd[key])
    img = torch.randn(1, 3, 256, 256, generator=torch.Generator().manual_seed(2)).to(dev)
    assert len(m.simple_test(img)) == 1
    u8 = (torch.rand(200, 260, 3, generator=torch.Generator().manual_seed(1)) * 255).to(torch.uint8).numpy()
    assert len(inference_detector(m, u8)) == 15


def _busy(dev):
    a = torch.randn(4096, 4096, device=dev)
    for _ in range(8):
        a = a @ a
        a = a / a.norm()
    return a


@pytest.mark.parametrize("fmt", FORMATS)
def test_side_stream_and_threads(dev, fmt):
    e = _engine(fmt, dev)
    x, _, r, _, logits = _launch_case(e, dev, 2, 15, 15, 30, 30, 5, 1, 2.0, seed=7)
    want = cf.carafe_add(e, x, logits, 5, 1, r).clone()
    torch.cuda.synchronize()
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _busy(dev)
        got = cf.carafe_add(e, x, logits, 5, 1, r)
    torch.cuda.current_stream().wait_stream(side)
    assert torch.equal(want, got)
    dets = [_det("r50", fmt, dev)[0] for _ in range(2)]
    img = torch.randn(2, 3, 128, 128, generator=torch.Generator().manual_seed(2)).to(dev)
    ref = [t.clone() for t in dets[0].forward_dense(img)[1]]
    torch.cuda.synchronize()
    res, errs = [None, None], []

    def work(i):
        try:
            with torch.cuda.device(dev):
                s = torch.cuda.Stream(device=dev)
                with torch.cuda.stream(s):
                    rr = [t.clone() for t in dets[i].forward_dense(img)[1]]
                s.synchronize()
                res[i] = rr
        except Exception as ex:                                          # noqa: BLE001
            errs.append(ex)

    th = [threading.Thread(target=work, args=(i,)) for i in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs
    for rr in res:
        for a, b in zip(ref, rr):
            if fmt == "fp32":
                assert torch.allclose(a, b, rtol=1e-5, atol=1e-5 * float(a.abs().max()))
            else:
                assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ the launch checker
@pytest.mark.parametrize("c", CARAFE_PARITY)
def test_carafe_parity_case_vs_fp64(dev, c):
    """the plans that only FPN_CARAFE's convolutions reach, launched against fp64 as tests/test_conv_plans_gpu.py launches
    PARITY"""
    from conv_plan_cases import planned, signature
    from orientedreppoints_b200.engine_tc import EngineTC, EngineTCSplit
    from test_conv_plans_gpu import Case, _check_values, _check_written_once
    case = Case(c, (EngineTCSplit if c[1] == "f16x3" else EngineTC)(dev), dev, seed=sum(c[3:7]) + len(c[-1]))
    plan = _check_written_once(case)
    assert signature(plan) == c[0] and plan == planned(c)
    _check_values(case, plan)


CHECKED = [("f16x3", 16, False), ("bf16", 16, False), ("f16x3", 4, True), ("bf16", 4, True), ("bf16", 1, False)]
# the workloads whose backbone and head plans tests/conv_plan_cases.PARITY pins (the benchmark's); at the others only the neck's
# plans are required to be pinned here
BENCH_WORKLOADS = CHECKED[:3]
NECK_LAYERS = ("lateral", "fpn", "up")


@pytest.mark.parametrize("prec,batch,test_scale", CHECKED, ids=["%s-x%d%s" % (p, n, "-960" if t else "") for p, n, t in CHECKED])
def test_every_launch_vs_fp64_r50_fpn_carafe(dev, monkeypatch, prec, batch, test_scale):
    """every convolution of R-50 FPN_CARAFE (GN, the default upsample_cfg) through the launch checker of
    tests/test_backbone_launches_gpu.py at the benchmark's inputs, every orp_carafe_add against the fp64 contract on the
    operands the engine holds, and every plan signature pinned"""
    import test_backbone_launches_gpu as tbl
    import test_production_launches_gpu as tpl
    t0 = time.time()
    name = "r50_fpn_carafe %s x%d%s" % (prec, batch, " at 960^2" if test_scale else "")
    spec = _neck_spec()
    sd = random_state_dict(50, seed=0, reference_init=False, residual_gain=0.5, neck=spec, carafe_gain=fr.CARAFE_GAIN)
    img, valid = tpl._inputs("r101", batch, test_scale, dev)
    det = OrientedRepPointsDetector(sd, 50, dev, prec, test_cfg=dict(score_thr=0.0), neck=spec)
    chk = tbl.BackboneChecker(det, name, monkeypatch)
    for kind, layers in (("lateral", det.neck.lat), ("fpn", det.neck.fpn)):
        for i, (L, _) in enumerate(layers):
            chk.names[id(L)] = "%s%d" % (kind, i)
    for j, (comp, enc) in enumerate(det.neck.up):
        chk.names[id(comp)], chk.names[id(enc)] = "up%d.compressor" % j, "up%d.encoder" % j
    carafes = []
    real = cf.carafe_add

    def checked(e, x, logits, k, g, residual):
        y = real(e, x, logits, k, g, residual)
        torch.cuda.synchronize()
        n = x.shape[0]
        for j in sorted({0, n - 1}):
            ref = _contract(_f(e, x), logits, k, g, _f(e, residual), j)
            err = _rel(_f(e, y[j:j + 1]).permute(0, 3, 1, 2), ref)
            assert err < TOL[e.name], "%s carafe %s: image %d rel err %.3e" % (name, tuple(x.shape), j, err)
        carafes.append(tuple(residual.shape[1:3]))
        return y
    monkeypatch.setattr(cf, "carafe_add", checked)
    if chk.split:
        det.eng.overflow_count()
    with torch.no_grad():
        det.forward_dense(img, valid)
    torch.cuda.synchronize()
    print(chk.summary(time.time() - t0))
    assert not chk.escaped, "%s: launches outside a checked call: %s" % (name, chk.escaped)
    assert chk.checked == chk.low and chk.checked > 0
    assert len(carafes) == 4
    if chk.split:
        assert det.eng.overflow_count() == 0, name
    monkeypatch.setattr(tbl, "PARITY", tbl.PARITY + CARAFE_PARITY)
    if (prec, batch, test_scale) not in BENCH_WORKLOADS:
        kept = [(s, l) for s, l in zip(chk.sigs, chk.layers) if l.startswith(NECK_LAYERS)]
        assert len(kept) == 18                                           # 5 laterals, 4 x (compressor, encoder), 5 fpn_convs
        chk.sigs, chk.layers = [s for s, _ in kept], [l for _, l in kept]
    tbl._signatures_pinned(chk)
    del det, chk
    torch.cuda.empty_cache()
