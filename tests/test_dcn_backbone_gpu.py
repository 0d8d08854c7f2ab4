"""GPU: ResNet backbones with deformable stages (dcn / stage_with_dcn) on every engine, against the fp64 graph of
tests/dcn_backbone_ref.py (deform_conv_ref, pinned to the reference's own DCN im2col kernels).

- every deformable conv2 launch of the backbone (stride 2, Cin = Cout = 64..512, folded-BN bias + ReLU, the engine's
  activation format out), DCN and DCNv2, alone, in f16x3, bf16 and fp32;
- the DCNv2 offset / mask split (orp_dcnv2_offset_mask) against an fp64 sigmoid, at a storage offset and on a side stream;
- the whole dense graph of R-50-DCN / R-101-DCN c3-c5 in f16x3 within 1e-4, and its detections;
- a captured deformable conv2 step bit-identical to the eager one, the captured dense graph within the GroupNorm replay
  tolerance; aug_test and the config-built detector on a DCN model."""
import numpy as np
import pytest
import torch

from dcn_backbone_ref import BATCHES, LAUNCHES_1024, forward_dense

pytestmark = pytest.mark.gpu

TOL = 1e-4             # north_star: "within 1e-4 fp32"
BF16_TOL = 1.5e-2      # the bf16 deformable tolerance of tests/test_f16x3_gpu.py (against fp64 on bf16-rounded operands)
F32_TOL = 2e-5         # fp32 CUDA-core FMAs over K = 9 * 512
C3_C5 = (False, True, True, True)
SPIN = 50_000_000      # torch.cuda._sleep cycles ahead of the inputs (tests/test_streams_gpu.py)


def _nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / (b.double().abs().max() + 1e-30))


def _engine(prec, cuda):
    from orientedreppoints_b200.detector import EngineF32
    from orientedreppoints_b200.engine_tc import EngineTC, EngineTCSplit
    return {"f16x3": EngineTCSplit, "bf16": EngineTC, "fp32": EngineF32}[prec](cuda)


def _to_engine(e, x_nhwc):
    if e.name == "f16x3":
        return e.from_float(x_nhwc)
    return x_nhwc.to(e.device, e.act_dtype).contiguous()


def _from_engine(e, y):
    return e.to_float(y) if e.name == "f16x3" else y.float()


def _launch_cases():
    out = []
    for n, tile in BATCHES:
        for planes, h, s in LAUNCHES_1024:
            for prec in ("f16x3", "bf16", "fp32"):
                if n == 16 and prec != "f16x3":
                    continue                       # the benchmark's batch runs f16x3
                out.append((prec, n, planes, h * tile // 1024, s))
    return out


@pytest.mark.parametrize("prec,n,planes,h,s", _launch_cases(),
                         ids=["%s-N%d-C%d-H%d-s%d" % c for c in _launch_cases()])
def test_backbone_deform_launch_vs_fp64(cuda, prec, n, planes, h, s):
    """one deformable conv2 as the engine runs it (folded-BN weight and bias, ReLU, activation format out), DCNv1 and DCNv2,
    offsets a few pixels off the grid and beyond the border, against deform_conv_ref in fp64 on the device"""
    from oracle import torch_reference as tr
    from orientedreppoints_b200.detector import ConvLayer
    e = _engine(prec, cuda)
    g = torch.Generator().manual_seed(planes + h + s + n)
    ho = (h - 1) // s + 1
    x = torch.relu(torch.randn(n, planes, h, h, generator=g))
    wt = torch.randn(planes, planes, 3, 3, generator=g) * (2.0 / (9 * planes)) ** 0.5
    b = torch.randn(planes, generator=g) * 0.1
    off = torch.randn(n, 18, ho, ho, generator=g) * 2.0
    m = torch.rand(n, 9, ho, ho, generator=g)
    L = ConvLayer(wt, b, s, 1, cuda)
    xr, wr = (x.bfloat16().double(), wt.bfloat16().double()) if prec == "bf16" else (x.double(), wt.double())
    xin = _to_engine(e, x.permute(0, 2, 3, 1).contiguous().to(cuda))
    for mask in (None, m):
        with torch.no_grad():
            ref = torch.relu(tr.deform_conv_ref(xr.to(cuda), off.double().to(cuda), wr.to(cuda), s, 1,
                                                mask=None if mask is None else mask.double().to(cuda))
                             + b.double().to(cuda).view(1, -1, 1, 1))
        y = e.deform_conv(xin, off.permute(0, 2, 3, 1).contiguous().to(cuda), L, relu=True,
                          mask=None if mask is None else mask.permute(0, 2, 3, 1).contiguous().to(cuda))
        assert tuple(y.shape[:3]) == (n, ho, ho)
        err = _rel(_nchw(_from_engine(e, y)), ref)
        print("%s N%d C%d H%d s%d %s: rel err %.2e" % (prec, n, planes, h, s, "DCNv2" if mask is not None else "DCN", err))
        assert err < {"f16x3": TOL, "bf16": BF16_TOL, "fp32": F32_TOL}[prec], ("DCNv2" if mask is not None else "DCN", err)
    if prec == "f16x3":
        assert e.overflow_count() == 0


def _offset_mask(om, n_pix, off, msk):
    from orientedreppoints_b200 import _lib
    _lib.check(_lib.lib().orp_dcnv2_offset_mask(_lib.ptr(om), n_pix, _lib.ptr(off), _lib.ptr(msk), _lib.current_stream_ptr()),
               "orp_dcnv2_offset_mask")


def test_offset_mask_split_vs_fp64(cuda):
    """channels 0..17 copied as they are, sigmoid(channels 18..26) within 2 ulp of the fp64 sigmoid, on views at an odd
    storage offset; on a side stream behind a spin, with the input written after the spin into a NaN buffer, the result is
    bit for bit the default stream's"""
    g = torch.Generator().manual_seed(0)
    n_pix = 2 * 37 * 53
    om = torch.randn(n_pix, 27, generator=g, dtype=torch.float64) * 8.0
    om[:40, 18:] = torch.tensor([0.0, -0.0, 1e-30, -1e-30, 15.0, -15.0, 30.0, -30.0, 88.0, -88.0, 103.0, -103.0, 200.0, -200.0,
                                 float("inf"), -float("inf"), 1e-7, -1e-7, 0.5, -0.5], dtype=torch.float64).repeat(18)[:360].view(40, 9)
    om = om.float()
    base = torch.full((n_pix * 27 + 3,), float("nan"), device=cuda)
    src = base[3:].view(n_pix, 27)
    src.copy_(om.to(cuda))
    obuf = torch.full((n_pix * 18 + 1,), float("nan"), device=cuda)
    mbuf = torch.full((n_pix * 9 + 5,), float("nan"), device=cuda)
    off, msk = obuf[1:].view(n_pix, 18), mbuf[5:].view(n_pix, 9)
    _offset_mask(src, n_pix, off, msk)
    torch.cuda.synchronize()
    assert torch.equal(off.cpu(), om[:, :18]) and bool(torch.isnan(obuf[:1]).all()) and bool(torch.isnan(mbuf[:5]).all())
    ref = torch.sigmoid(om[:, 18:].double())
    got = msk.cpu().double()
    ulp = torch.from_numpy(np.spacing(ref.float().abs().numpy())).double()
    worst = float(((got - ref).abs() / ulp).max())
    print("sigmoid max error %.2f ulp" % worst)
    assert worst <= 2.0
    # side stream
    side = torch.cuda.Stream(device=cuda)
    inp = torch.full_like(base, float("nan"))
    o2 = torch.full_like(obuf, float("nan"))
    m2 = torch.full_like(mbuf, float("nan"))
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(SPIN)
        inp[3:].copy_(base[3:])
        _offset_mask(inp[3:].view(n_pix, 27), n_pix, o2[1:].view(n_pix, 18), m2[5:].view(n_pix, 9))
    side.synchronize()
    assert torch.equal(o2[1:].cpu(), obuf[1:].cpu()) and torch.equal(m2[5:].cpu(), mbuf[5:].cpu())
    from orientedreppoints_b200 import _lib
    with pytest.raises(_lib.OrpError, match="dcnv2_offset_mask: bad arguments"):
        _offset_mask(src, -1, off, msk)
    _offset_mask(src, 0, off, msk)                                          # empty: a no-op


def _dcn_case(cuda, depth, kind, n, h, w, seed, prec="f16x3"):
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    from orientedreppoints_b200.weights import STAGE_BLOCKS, dcn_layout, random_state_dict
    dcn = dict(type=kind)
    # residual_gain 0.3 keeps the activations, and with them the offsets, at about 1 (offsets of 1-2 px rms in every stage).
    # At the 1.0 of the plain R-50 tests the activations grow to ~10 and the offsets with them; a difference of an offset
    # is then multiplied by the feature gradient at ~10 px in every deformable layer, and after 13 of them the fp64 graph
    # itself amplifies an fp32-rounding difference of its input beyond 1e-4 (the R-101 / 0.3 case stayed within it)
    sd = random_state_dict(depth, seed=0, reference_init=False, residual_gain=0.3, dcn=dcn, stage_with_dcn=C3_C5,
                           dcn_offset_scale=1.0)
    layout = dcn_layout(depth, dcn, C3_C5)
    det = OrientedRepPointsDetector(sd, depth, cuda, prec, test_cfg=dict(score_thr=0.02), dcn=layout)
    img = torch.randn(n, 3, h, w, generator=torch.Generator().manual_seed(seed)).to(cuda)
    outs, feats = det.forward_dense(img)
    torch.cuda.synchronize()
    if prec == "f16x3":
        assert det.eng.overflow_count() == 0
    sdg = {k: v.to(cuda).double() for k, v in sd.items()}
    with torch.no_grad():
        ref_outs, ref_feats = forward_dense(sdg, img.double(), layout, STAGE_BLOCKS[depth])
    errs = {}
    for lvl in range(5):
        errs["feat%d" % lvl] = _rel(_nchw(_from_engine(det.eng, feats[lvl])), ref_feats[lvl])
        for k, name in enumerate(("cls", "init", "refine")):
            a, b = _nchw(outs[lvl][k]), ref_outs[lvl][k]
            assert a.shape == b.shape
            errs["%s%d" % (name, lvl)] = float((a.double() - b).abs().max()) / max(1.0, float(b.abs().max()))
    return det, img, outs, ref_outs, errs


@pytest.mark.parametrize("depth,kind,n,size", [(50, 'DCN', 1, 1024), (50, 'DCNv2', 1, 1024), (50, 'DCN', 2, 512),
                                               (50, 'DCNv2', 2, 512), (101, 'DCNv2', 1, 512)])
def test_dense_graph_dcn_f16x3_vs_fp64(cuda, depth, kind, n, size):
    """R-50 / R-101 with DCN or DCNv2 in c3-c5: every FPN level and head output within 1e-4 of the fp64 graph"""
    _, _, _, _, errs = _dcn_case(cuda, depth, kind, n, size, size, 11)
    print("f16x3 R-%d-%s %dx%d^2 max rel err:" % (depth, kind, n, size), max(errs.values()), errs)
    for k, v in errs.items():
        assert v < TOL, (k, v)


def test_dcn_detections_f16x3_1024(cuda):
    """detections of R-50-DCNv2 c3-c5 at 1024^2 against the restated reference post-processing run on the fp64 graph's
    outputs, matched by content as in tests/test_f16x3_gpu.py::test_dense_graph_f16x3_1024_and_detections"""
    from oracle import torch_reference as tr
    det, img, outs, ref_outs, errs = _dcn_case(cuda, 50, 'DCNv2', 1, 1024, 1024, 5)
    assert max(errs.values()) < TOL, errs
    res = det.simple_test(img, [dict(scale_factor=1.0)], rescale=True, return_tensors=True)
    d, l = res[0][0].cpu(), res[0][1].cpu()
    rd, rl = tr.get_bboxes_single([o[0][0].float() for o in ref_outs], [o[2][0].float().cpu() for o in ref_outs], score_thr=0.02)
    assert d.shape[0] > 0 and rd.shape[0] > 0
    dist = torch.cdist(d[:, :26].double(), rd[:, :26].double(), p=float("inf"))
    dist = dist + (l[:, None] != rl[None, :]).double() * 1e6
    best, arg = dist.min(dim=1)
    matched = best < 1e-2
    frac, back = float(matched.float().mean()), float((dist.min(dim=0).values < 1e-2).float().mean())
    print("R-50-DCNv2 1024: %d detections (ref %d), %.4f / %.4f matched" % (d.shape[0], rd.shape[0], frac, back))
    assert frac > 0.98 and back > 0.98
    assert float((d[matched, 26] - rd[arg[matched], 26]).abs().max()) < 1e-4


@pytest.mark.parametrize("prec", ["f16x3", "bf16", "fp32"])
def test_dense_graph_dcn_every_engine(cuda, prec):
    """R-50-DCNv2 c3-c5 on each engine: f16x3 and fp32 within 1e-4 of the fp64 graph; bf16 FPN levels within the 0.06 of
    tests/test_dense_gpu.py::test_dense_graph_bf16_vs_f32_engine (bf16 activations through ~60 layers)"""
    _, _, _, _, errs = _dcn_case(cuda, 50, 'DCNv2', 2, 256, 320, 3, prec)
    print("%s R-50-DCNv2 max rel err:" % prec, max(errs.values()), errs)
    for k, v in errs.items():
        if prec != "bf16":
            assert v < TOL, (k, v)
        elif k.startswith("feat"):
            assert v < 0.06, (k, v)


def test_graph_replay_matches_eager(cuda):
    """CUDA-graph capture of the R-50-DCNv2 dense graph.  A deformable conv2 step (offset convolution, offset / mask split,
    deformable launch) captured alone replays to the eager pass's bits; the whole graph replays within the GroupNorm
    tolerance of tests/test_streams_gpu.py (its sums are fp64 atomics, the only order-dependent arithmetic of the graph)"""
    det, img, _, _, _ = _dcn_case(cuda, 50, 'DCNv2', 2, 512, 512, 7)
    eager, _ = det.forward_dense(img)
    eager = [[t.clone() for t in lvl] for lvl in eager]
    det.capture(img.shape)
    outs, _ = det.forward_dense_graph(img)
    torch.cuda.synchronize()
    for lvl in range(5):
        for k in range(3):
            assert _rel(outs[lvl][k], eager[lvl][k]) < 1e-5, (lvl, k)
    for li, b in ((1, 0), (3, 1)):
        blk = det.blocks[li][b]
        assert blk["dcn"] == 'DCNv2'
        planes, hin = 64 << li, (128 if b == 0 else 64) >> (li - 1)
        x = det.eng.from_float(torch.relu(torch.randn(2, hin, hin, planes, generator=torch.Generator().manual_seed(li))).to(cuda))
        want = det._conv2(x, blk).clone()
        side = torch.cuda.Stream(device=cuda)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            det._conv2(x, blk)                                           # warm-up off the capture
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            y = det._conv2(x, blk)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, want), (li, b)


def test_aug_test_and_config_model_with_dcn(cuda):
    """a config-built R-50-DCN c3-c5 detector (the backbone override of the README) runs simple_test and aug_test"""
    import importlib.util
    import os
    from orientedreppoints_b200.models import build_detector
    from orientedreppoints_b200.weights import random_state_dict
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("c", os.path.join(root, "configs", "dota", "orientedrepoints_r50_demo.py"))
    cfg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cfg)
    dcn = dict(type='DCNv2', deformable_groups=1, fallback_on_stride=False)
    model = dict(cfg.model, pretrained=None, backbone=dict(cfg.model["backbone"], dcn=dcn, stage_with_dcn=C3_C5))
    det = build_detector(model, test_cfg=dict(cfg.test_cfg, score_thr=0.02))
    det.load_state_dict(random_state_dict(50, seed=0, reference_init=False, dcn=dict(type='DCNv2'), stage_with_dcn=C3_C5,
                                          dcn_offset_scale=1.0), strict=True)
    det = det.to(cuda)
    assert det.engine().dcn == det.backbone.dcn_layout() and det.engine().dcn[1][0] == 'DCNv2'
    img = torch.randn(1, 3, 256, 256, generator=torch.Generator().manual_seed(3)).to(cuda)
    res = det(img, [dict(scale_factor=1.0)], return_loss=False, rescale=True)
    assert len(res) == 1 and len(res[0]) == 15 and sum(len(a) for a in res[0]) > 0
    metas = [[dict(img_shape=(256, 256, 3), scale_factor=1.0, flip=False)], [dict(img_shape=(256, 256, 3), scale_factor=1.0, flip=True)]]
    aug = det.aug_test([img, img.flip(-1)], metas, rescale=True)
    assert len(aug) == 15 and sum(len(a) for a in aug) > 0
