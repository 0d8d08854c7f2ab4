"""GPU: the dense path (backbone / FPN / head / DCN) against the PyTorch fp32 re-declaration of the
reference graph (oracle/torch_reference.py).  fp32 engine: tight tolerances (same arithmetic up to
summation order); bf16 tensor-core engine: tolerances stated per test."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


def _rel(a, b):
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


@pytest.fixture(scope="module")
def sd():
    from orientedreppoints_b200.weights import random_state_dict
    return random_state_dict(50, seed=0, reference_init=False)


def test_conv_and_dcn_f32_vs_torch(cuda):
    from oracle import torch_reference as tr
    from orientedreppoints_b200.detector import ConvLayer, EngineF32
    import torch.nn.functional as F
    e = EngineF32(cuda)
    g = torch.Generator().manual_seed(0)
    for (cin, cout, k, s, p, h, w) in [(64, 64, 3, 1, 1, 37, 53), (128, 256, 1, 2, 0, 40, 40), (256, 18, 1, 1, 0, 19, 23),
                                       (4, 64, 7, 2, 3, 96, 80), (256, 256, 3, 2, 1, 33, 31)]:
        x = torch.randn(2, cin, h, w, generator=g)
        wt = torch.randn(cout, cin, k, k, generator=g) * 0.05
        b = torch.randn(cout, generator=g)
        ref = F.conv2d(x.double(), wt.double(), b.double(), s, p).float()
        L = ConvLayer(wt, b, s, p, cuda)
        y = e.conv(x.permute(0, 2, 3, 1).contiguous().to(cuda), L)
        assert _rel(_nchw(y).cpu(), ref) < 1e-5, (cin, cout, k, s)
    # deformable conv incl. samples that leave the image
    x = torch.randn(2, 64, 21, 27, generator=g)
    off = torch.randn(2, 18, 21, 27, generator=g) * 3.0
    wt = torch.randn(32, 64, 3, 3, generator=g) * 0.05
    ref = tr.deform_conv_ref(x.double(), off.double(), wt.double()).float()
    L = ConvLayer(wt, None, 1, 1, cuda)
    y = e.deform_conv(x.permute(0, 2, 3, 1).contiguous().to(cuda), off.permute(0, 2, 3, 1).contiguous().to(cuda), L)
    assert _rel(_nchw(y).cpu(), ref) < 1e-5
    # DCNv2 (mask) surface
    m = torch.rand(2, 9, 21, 27, generator=g)
    ref = tr.deform_conv_ref(x.double(), off.double(), wt.double(), mask=m.double()).float()
    y = e.deform_conv(x.permute(0, 2, 3, 1).contiguous().to(cuda), off.permute(0, 2, 3, 1).contiguous().to(cuda), L,
                      mask=m.permute(0, 2, 3, 1).contiguous().to(cuda))
    assert _rel(_nchw(y).cpu(), ref) < 1e-5


def test_dense_graph_f32_vs_torch(cuda, sd):
    from oracle import torch_reference as tr
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    det = OrientedRepPointsDetector(sd, 50, cuda, "fp32")
    img = torch.randn(2, 3, 256, 320, generator=torch.Generator().manual_seed(1))
    outs, feats = det.forward_dense(img.to(cuda))
    # fp64 torch graph as the gold standard (torch's fp32 GPU convs silently use TF32)
    sdg = {k: v.to(cuda).double() for k, v in sd.items()}
    with torch.no_grad():
        ref_outs, ref_feats = tr.forward_dense(sdg, img.to(cuda).double())
    ref_feats = [f.float() for f in ref_feats]
    ref_outs = [[t.float() for t in o] for o in ref_outs]
    for lvl in range(5):
        assert _rel(_nchw(feats[lvl]), ref_feats[lvl]) < 2e-4, lvl
        for k, name in enumerate(("cls", "init", "refine")):
            a, b = _nchw(outs[lvl][k]), ref_outs[lvl][k]
            assert a.shape == b.shape
            assert float((a - b).abs().max()) < 2e-4 * max(1.0, float(b.abs().max())), (lvl, name)


def test_simple_test_matches_reference_pipeline(cuda, sd):
    """whole tile: detections (boxes, reppoints, scores, labels, ORDER) against the restated reference
    post-processing over the torch graph's outputs"""
    from oracle import torch_reference as tr
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    cfg = dict(score_thr=0.02)
    det = OrientedRepPointsDetector(sd, 50, cuda, "fp32", test_cfg=cfg)
    img = torch.randn(1, 3, 256, 256, generator=torch.Generator().manual_seed(2))
    from orientedreppoints_b200.core.get_bboxes import get_bboxes
    from orientedreppoints_b200.detector import STRIDES
    outs, _ = det.forward_dense(img.to(cuda))
    (dets, labels), = get_bboxes([o[0] for o in outs], [o[2] for o in outs], STRIDES, [dict(scale_factor=1.0)],
                                 det.test_cfg, rescale=True)
    # post-processing oracle on the SAME dense outputs (GN statistics use atomics: two forward passes differ
    # in the last bit); sigmoid evaluated by the same device routine, everything after it on the CPU oracle
    cls = [_nchw(o[0])[0] for o in outs]
    ref = [_nchw(o[2])[0].cpu() for o in outs]
    rd, rl = tr.get_bboxes_single(cls, ref, score_thr=0.02)
    assert dets.shape == rd.shape and dets.shape[0] > 10
    assert torch.equal(labels.cpu(), rl)                                    # index work: bit-exact
    assert float((dets.cpu() - rd).abs().max()) < 1e-3                      # coordinates in pixels (1e-4 * stride scale)
    assert torch.equal(dets[:, -1].cpu(), rd[:, -1])                        # scores


# ------------------------------------------------------------------------------- tensor-core engine
def _bf16_ref_conv(x, wt, b, s, p):
    """fp64 conv over the bf16-ROUNDED operands: what an exact accumulation of the tensor-core inputs gives"""
    import torch.nn.functional as F
    return F.conv2d(x.bfloat16().double(), wt.bfloat16().double(), None if b is None else b.double(), s, p)


@pytest.mark.parametrize("cin,cout,k,s,p,h,w,n", [
    (64, 64, 1, 1, 0, 32, 32, 1),        # one tile, one K block
    (64, 256, 1, 1, 0, 64, 64, 2),       # BN=256
    (256, 64, 3, 1, 1, 64, 64, 1),       # 3x3: TMA zero padding, 36 K blocks
    (128, 128, 3, 2, 1, 64, 64, 2),      # stride 2 through tensor-map element strides
    (512, 1024, 1, 2, 0, 32, 32, 2),     # 1x1 stride 2 (downsample), 4 N tiles
    (256, 256, 3, 1, 1, 37, 53, 2),      # ragged: partial tiles in W and H
    (256, 18, 1, 1, 0, 19, 23, 3),       # Cout 18 -> padded to 32, masked stores
    (256, 256, 3, 2, 1, 16, 16, 3),      # 8x8 output: tile spans 2 images
    (2048, 256, 3, 2, 1, 32, 32, 1),     # P6: K = 18432
])
def test_conv_tc_vs_exact(cuda, cin, cout, k, s, p, h, w, n):
    from orientedreppoints_b200.detector import ConvLayer
    from orientedreppoints_b200.engine_tc import EngineTC
    e = EngineTC(cuda)
    g = torch.Generator().manual_seed(cin + cout + k + h)
    x = torch.randn(n, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, k, k, generator=g) * (1.0 / (cin * k * k) ** 0.5)
    b = torch.randn(cout, generator=g)
    ref = _bf16_ref_conv(x, wt, b, s, p).float()
    L = ConvLayer(wt, b, s, p, cuda)
    xb = x.permute(0, 2, 3, 1).contiguous().to(cuda, torch.bfloat16)
    y32 = e.conv(xb, L, out_f32=True)
    assert _rel(_nchw(y32).cpu(), ref) < 2e-5, "fp32 accumulation of exact bf16 products"
    r = torch.randn(ref.shape, generator=g)
    yb = e.conv(xb, L, relu=True, residual=r.permute(0, 2, 3, 1).contiguous().to(cuda, torch.bfloat16))
    refb = torch.relu(ref + r.bfloat16().float())
    assert _rel(_nchw(yb.float()).cpu(), refb) < 6e-3          # one bf16 rounding of the output (2^-8)


def test_deform_conv_tc_vs_f32_engine(cuda):
    from oracle import torch_reference as tr
    from orientedreppoints_b200.detector import ConvLayer
    from orientedreppoints_b200.engine_tc import EngineTC
    e = EngineTC(cuda)
    g = torch.Generator().manual_seed(3)
    xs, offs, refs = [], [], []
    wt = torch.randn(256, 256, 3, 3, generator=g) * 0.02
    for (h, w) in [(40, 56), (20, 28), (10, 14), (5, 7), (3, 4)]:       # five "levels" in one launch
        x = torch.randn(2, 256, h, w, generator=g)
        off = torch.randn(2, 18, h, w, generator=g) * 2.5
        refs.append(tr.deform_conv_ref(x.bfloat16().double(), off.double(), wt.bfloat16().double()).float())
        xs.append(x.permute(0, 2, 3, 1).contiguous().to(cuda, torch.bfloat16))
        offs.append(off.permute(0, 2, 3, 1).contiguous().to(cuda))
    L = ConvLayer(wt, None, 1, 1, cuda)
    ys = e.deform_conv_multi(xs, offs, L)
    for y, ref in zip(ys, refs):
        # sampled values are rounded to bf16 before the MMA (2^-9 relative each), outputs to bf16
        assert _rel(_nchw(y.float()).cpu(), ref) < 1.5e-2


def test_dense_graph_bf16_vs_f32_engine(cuda, sd):
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    d32 = OrientedRepPointsDetector(sd, 50, cuda, "fp32")
    d16 = OrientedRepPointsDetector(sd, 50, cuda, "bf16")
    img = torch.randn(2, 3, 256, 320, generator=torch.Generator().manual_seed(1)).to(cuda)
    o32, f32 = d32.forward_dense(img)
    o16, f16 = d16.forward_dense(img)
    for lvl in range(5):
        assert _rel(f16[lvl].float(), f32[lvl]) < 0.06, lvl          # bf16 activations through ~60 layers
        for k in range(3):
            a, b = o16[lvl][k], o32[lvl][k]
            assert a.shape == b.shape and a.dtype == torch.float32
            assert float((a - b).abs().max()) < 0.08 * max(1.0, float(b.abs().max())), (lvl, k)


def test_fused_postprocess_equals_torch_mirror_and_oracle(cuda, sd):
    """orp_head_postprocess (one device pipeline) == the op-by-op mirror of get_bboxes/multiclass_rnms ==
    the restated reference pipeline on the CPU oracle: labels/order bit-exact, scores bit-exact, coordinates 1e-3 px"""
    from oracle import torch_reference as tr
    from orientedreppoints_b200.core.get_bboxes import get_bboxes, get_bboxes_fused
    from orientedreppoints_b200.detector import OrientedRepPointsDetector, STRIDES
    for thr, size, cap in ((0.02, 256, 2000), (0.0, 384, 300), (0.5, 256, 2000)):
        det = OrientedRepPointsDetector(sd, 50, cuda, "fp32", test_cfg=dict(score_thr=thr, max_per_img=cap))
        img = torch.randn(2, 3, size, size, generator=torch.Generator().manual_seed(5)).to(cuda)
        outs, _ = det.forward_dense(img)
        cls, ref = [o[0] for o in outs], [o[2] for o in outs]
        metas = [dict(scale_factor=1.0), dict(scale_factor=1.0)]
        mirror = get_bboxes(cls, ref, STRIDES, metas, det.test_cfg, rescale=True)
        dets, labels, counts = get_bboxes_fused(cls, ref, STRIDES, metas, det.test_cfg, rescale=True)
        counts = counts.tolist()
        for i in range(2):
            d, l = dets[i, :counts[i]], labels[i, :counts[i]]
            md, ml = mirror[i]
            assert d.shape == md.shape, (thr, i, d.shape, md.shape)
            assert torch.equal(l, ml)
            assert torch.equal(d[:, -1], md[:, -1])
            assert float((d - md).abs().max()) < 1e-3 if d.numel() else True
            assert bool((labels[i, counts[i]:] == -1).all())
        if thr == 0.02:
            rd, rl = tr.get_bboxes_single([c[0].permute(2, 0, 1) for c in cls], [r[0].permute(2, 0, 1).cpu() for r in ref],
                                          score_thr=thr, max_per_img=cap)
            assert torch.equal(labels[0, :counts[0]].cpu(), rl) and torch.equal(dets[0, :counts[0], -1].cpu(), rd[:, -1])


def test_stem_space_to_depth_form(cuda, sd):
    """default stem path (space-to-depth copy + 4x4 stride-1 conv through TMA) against the im2col GEMM (same bf16
    operands, different accumulation order) and against torch's conv2d on the bf16-rounded operands
    (resnet.py:495 conv1 + folded norm1 + ReLU)"""
    import torch.nn.functional as F
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    det = OrientedRepPointsDetector(sd, 50, cuda, "bf16")
    for (n, h, w) in ((2, 256, 320), (1, 250, 198), (3, 64, 66), (1, 1024, 1024)):
        img = torch.randn(n, 3, h, w, generator=torch.Generator().manual_seed(h)).to(cuda)
        a = det.eng.stem(img, det.stem)                       # s2d
        b = det.eng.stem(img, det.stem, mode="im2col")
        assert a.shape == b.shape
        diff = (a.float() - b.float()).abs()
        assert float(diff.max()) <= 2e-2 * max(1.0, float(b.float().abs().max())), float(diff.max())
        assert float((diff > 0).float().mean()) < 0.05        # only last-bit flips of the bf16 rounding
        wq = det.stem.w_raw.to(cuda).bfloat16().double().permute(0, 3, 1, 2)            # [64,3,7,7]
        ref = F.relu(F.conv2d(img.bfloat16().double(), wq, det.stem.bias.double().to(cuda), stride=2, padding=3))
        err = (a.double().permute(0, 3, 1, 2) - ref).abs().max()
        assert float(err) <= 1e-2 * max(1.0, float(ref.abs().max())), float(err)


def test_uint8_tiles_normalize_fused_into_stem(cuda, sd):
    """decoded uint8 HWC tiles: Normalize (mmdet/datasets/pipelines/transforms.py:Normalize -> mmcv.imnormalize,
    mean/std/to_rgb of configs/dota/orientedrepoints_r50_demo.py:72-73) fused into the stem input transform gives
    exactly what normalising first and feeding the float NCHW tensor gives"""
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    det = OrientedRepPointsDetector(sd, 50, cuda, "bf16", test_cfg=dict(score_thr=0.0))
    u8 = torch.randint(0, 256, (2, 128, 160, 3), generator=torch.Generator().manual_seed(5), dtype=torch.uint8).to(cuda)
    x = det.normalize(u8)
    assert x.shape == (2, 3, 128, 160) and x.dtype == torch.float32
    ref = ((u8.cpu().double().flip(-1) - torch.tensor([123.675, 116.28, 103.53], dtype=torch.float64))
           / torch.tensor([58.395, 57.12, 57.375], dtype=torch.float64)).permute(0, 3, 1, 2)
    assert float((x.cpu().double() - ref).abs().max()) < 1e-5
    a = det.eng.stem_u8(u8, det.stem, det.img_norm_cfg)
    b = det.eng.stem(x, det.stem)
    assert torch.equal(a, b)
    ra = det.simple_test(u8, return_tensors=True)
    rb = det.simple_test(x, return_tensors=True)
    for (da, la), (db, lb) in zip(ra, rb):
        assert torch.equal(da, db) and torch.equal(la, lb)
    # fp32 engine takes the same tiles (normalised by torch ops on the device)
    d32 = OrientedRepPointsDetector(sd, 50, cuda, "fp32")
    o_u8, _ = d32.forward_dense(u8)
    o_f, _ = d32.forward_dense(x)
    assert torch.allclose(o_u8[0][0], o_f[0][0], rtol=1e-4, atol=1e-4)      # fp32 GroupNorm statistics use atomics: not bit-reproducible


def test_r101_graph_bf16_vs_f32_engine(cuda):
    """BASELINE.json configs[3] backbone: same code path with STAGE_BLOCKS[101] = (3, 4, 23, 3)"""
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    from orientedreppoints_b200.weights import random_state_dict
    sd101 = random_state_dict(101, seed=3, reference_init=False)
    assert "backbone.layer3.22.conv3.weight" in sd101
    d32 = OrientedRepPointsDetector(sd101, 101, cuda, "fp32")
    d16 = OrientedRepPointsDetector(sd101, 101, cuda, "bf16")
    img = torch.randn(1, 3, 192, 256, generator=torch.Generator().manual_seed(1)).to(cuda)
    o32, f32 = d32.forward_dense(img)
    o16, f16 = d16.forward_dense(img)
    for lvl in range(5):
        assert _rel(f16[lvl].float(), f32[lvl]) < 0.08, lvl
        for k in range(3):
            a, b = o16[lvl][k], o32[lvl][k]
            assert float((a - b).abs().max()) < 0.1 * max(1.0, float(b.abs().max())), (lvl, k)
