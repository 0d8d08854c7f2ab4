"""GPU: Swin-T backbone (SURVEY 8 row a2) - component kernels against torch on identical bf16 inputs (tight),
whole backbone / detector against the fp32 torch re-declaration of the reference graph (bf16 tolerance)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def swin_sd():
    from orientedreppoints_b200.swin import random_swin_state_dict
    return random_swin_state_dict(0)


def _rel(a, b):
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def test_layernorm_and_gathers(cuda, swin_sd):
    from orientedreppoints_b200 import _lib
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    det = OrientedRepPointsDetector(swin_sd, "swin_tiny", cuda, "bf16")
    sw = det.swin
    g = torch.Generator().manual_seed(0)
    for c in (96, 192, 1536):
        x = torch.randn(2, 9, 11, c, generator=g).to(cuda).bfloat16()
        ln = type("L", (), {})()
        ln.gamma = torch.rand(c, generator=g).to(cuda) + 0.5
        ln.beta = torch.randn(c, generator=g).to(cuda)
        y = sw._ln(x, ln, 14, 14)
        ref = F.layer_norm(x.float(), (c,), ln.gamma, ln.beta, 1e-5)
        assert _rel(y[:, :9, :11].float(), ref) < 8e-3                      # bf16 output rounding
        assert float(y[:, 9:].abs().max()) == 0 and float(y[:, :, 11:].abs().max()) == 0
    x = torch.randn(2, 9, 11, 96, generator=g).to(cuda).bfloat16()
    y = torch.empty((2, 5, 6, 384), dtype=torch.bfloat16, device=cuda)
    _lib.check(sw.lib.orp_patch_merge_gather_bf16(_lib.ptr(x), 2, 9, 11, 96, _lib.ptr(y), _lib.current_stream_ptr()), "merge")
    xp = F.pad(x, (0, 0, 0, 1, 0, 1))
    ref = torch.cat([xp[:, 0::2, 0::2], xp[:, 1::2, 0::2], xp[:, 0::2, 1::2], xp[:, 1::2, 1::2]], -1)
    assert torch.equal(y, ref)
    assert torch.equal(sw.subsample2(x), x[:, ::2, ::2].contiguous())
    img = torch.randn(2, 3, 37, 50, generator=g).to(cuda)
    rows = torch.empty((2, 10, 13, 64), dtype=torch.bfloat16, device=cuda)
    _lib.check(sw.lib.orp_patch_embed_rows_bf16(_lib.ptr(img), 2, 37, 50, _lib.ptr(rows), _lib.current_stream_ptr()), "embed")
    ip = F.pad(img, (0, 2, 0, 3))
    ref = ip.unfold(2, 4, 4).unfold(3, 4, 4).permute(0, 2, 3, 1, 4, 5).reshape(2, 10, 13, 48).bfloat16()
    assert torch.equal(rows[..., :48], ref) and float(rows[..., 48:].abs().max()) == 0


@pytest.mark.parametrize("h,w,heads,shift", [(14, 14, 3, 0), (14, 21, 3, 3), (10, 13, 6, 3), (7, 7, 24, 3), (19, 9, 12, 0)])
def test_window_attention_vs_torch(cuda, h, w, heads, shift):
    from oracle import torch_swin as ts
    from orientedreppoints_b200 import _lib
    c = heads * 32
    hp, wp = (h + 6) // 7 * 7, (w + 6) // 7 * 7
    g = torch.Generator().manual_seed(h * w + heads)
    qkv = torch.randn(2, hp, wp, 3 * c, generator=g).to(cuda).bfloat16()
    table = (torch.randn(169, heads, generator=g) * 0.5).to(cuda)
    out = torch.empty((2, h, w, c), dtype=torch.bfloat16, device=cuda)
    _lib.check(_lib.lib().orp_window_attention_bf16(_lib.ptr(qkv), 2, h, w, hp, wp, c, heads, shift, _lib.ptr(table),
                                                    float(32 ** -0.5), _lib.ptr(out), _lib.current_stream_ptr()), "attn")
    x = qkv.float()
    sx = torch.roll(x, shifts=(-shift, -shift), dims=(1, 2)) if shift else x
    xw = ts.window_partition(sx, 7).view(-1, 49, 3 * c)
    q, k, v = xw.reshape(-1, 49, 3, heads, 32).permute(2, 0, 3, 1, 4)
    mask = ts.shift_mask(hp, wp, shift, cuda) if shift else None
    aw = ts.attention_core(q, k, v, table, heads, mask).view(-1, 7, 7, c)
    sx = ts.window_reverse(aw, 7, hp, wp)
    ref = (torch.roll(sx, shifts=(shift, shift), dims=(1, 2)) if shift else sx)[:, :h, :w]
    assert _rel(out.float(), ref) < 6e-3                                     # one bf16 rounding of the output


def test_swin_backbone_and_detector_vs_torch(cuda, swin_sd):
    from oracle import torch_reference as tr
    from oracle import torch_swin as ts
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    det = OrientedRepPointsDetector(swin_sd, "swin_tiny", cuda, "bf16", test_cfg=dict(score_thr=0.02))
    img = torch.randn(2, 3, 250, 198, generator=torch.Generator().manual_seed(3)).to(cuda)
    sdg = {k: v.to(cuda) for k, v in swin_sd.items()}
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    with torch.no_grad():
        ref_feats = ts.swin_forward(sdg, img)
        ref_fpn = ts.swin_fpn(sdg, ref_feats)
        ref_outs = [tr.head_single(sdg, f)[:3] for f in ref_fpn]
    feats = det.swin.forward(img)
    for a, b in zip(feats, ref_feats):
        assert a.shape == b.permute(0, 2, 3, 1).shape
        assert _rel(a.float().permute(0, 3, 1, 2), b) < 0.05
    outs, fpn = det.forward_dense(img)
    for lvl in range(5):
        assert _rel(fpn[lvl].float().permute(0, 3, 1, 2), ref_fpn[lvl]) < 0.08, lvl
        for k in range(3):
            a, b = outs[lvl][k].permute(0, 3, 1, 2), ref_outs[lvl][k]
            assert a.shape == b.shape
            assert float((a - b).abs().max()) < 0.1 * max(1.0, float(b.abs().max())), (lvl, k)
    res = det.simple_test(img)
    assert len(res) == 2 and len(res[0]) == 15


def test_swin_f16x3_kernels_and_backbone_vs_fp64(cuda, swin_sd):
    """Swin-T in the parity arithmetic (f16x3 Linear layers on the wgmma kernels, LayerNorm / window attention / gathers on split fp16
    tokens): component kernels vs torch in fp64, whole backbone + FPN + head vs the fp64 evaluation of the reference graph
    (oracle/torch_swin.py, pinned to the reference's own SwinTransformer), tolerance = north_star's 1e-4"""
    from oracle import torch_reference as tr
    from oracle import torch_swin as ts
    from orientedreppoints_b200 import _lib
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    det = OrientedRepPointsDetector(swin_sd, "swin_tiny", cuda, "f16x3", test_cfg=dict(score_thr=0.02))
    e, sw = det.eng, det.swin
    g = torch.Generator().manual_seed(1)
    # LayerNorm into a padded grid
    x = torch.randn(2, 9, 11, 192, generator=g)
    ln = type("L", (), {})()
    ln.gamma = torch.rand(192, generator=g).to(cuda) + 0.5
    ln.beta = torch.randn(192, generator=g).to(cuda)
    y = e.to_float(sw._ln(e.from_float(x), ln, 14, 14))
    ref = F.layer_norm(x.double().to(cuda), (192,), ln.gamma.double(), ln.beta.double(), 1e-5)
    assert _rel(y[:, :9, :11].double(), ref) < 2e-6 and float(y[:, 9:].abs().max()) == 0
    # merge gather / subsample are pure moves of (hi, lo) pairs
    xs = e.from_float(x)
    gth = e.alloc(2, 5, 6, 768)
    _lib.check(sw.lib.orp_patch_merge_gather_f16x3(_lib.ptr(xs), 2, 9, 11, 192, _lib.ptr(gth), _lib.current_stream_ptr()), "merge")
    xp = F.pad(e.to_float(xs), (0, 0, 0, 1, 0, 1))
    assert torch.equal(e.to_float(gth), torch.cat([xp[:, 0::2, 0::2], xp[:, 1::2, 0::2], xp[:, 0::2, 1::2], xp[:, 1::2, 1::2]], -1))
    assert torch.equal(e.to_float(sw.subsample2(xs)), e.to_float(xs)[:, ::2, ::2].contiguous())
    # window attention with shift, padding and the region mask
    h, w, heads, shift = 10, 13, 6, 3
    c, hp, wp = heads * 32, 14, 14
    qkv = torch.randn(2, hp, wp, 3 * c, generator=g)
    table = (torch.randn(169, heads, generator=g) * 0.5).to(cuda)
    out = e.to_float(sw._attention(e.from_float(qkv), 2, h, w, c, heads, shift, table))
    xq = qkv.double().to(cuda)
    sx = torch.roll(xq, shifts=(-shift, -shift), dims=(1, 2))
    xw = ts.window_partition(sx, 7).view(-1, 49, 3 * c)
    q, k, v = xw.reshape(-1, 49, 3, heads, 32).permute(2, 0, 3, 1, 4)
    aw = ts.attention_core(q, k, v, table.double(), heads, ts.shift_mask(hp, wp, shift, cuda).double()).view(-1, 7, 7, c)
    ref = torch.roll(ts.window_reverse(aw, 7, hp, wp), shifts=(shift, shift), dims=(1, 2))[:, :h, :w]
    assert _rel(out.double(), ref) < 5e-6
    # whole graph
    img = torch.randn(2, 3, 250, 198, generator=torch.Generator().manual_seed(3)).to(cuda)
    sdg = {k2: v2.to(cuda).double() for k2, v2 in swin_sd.items()}
    with torch.no_grad():
        ref_feats = ts.swin_forward(sdg, img.double())
        ref_fpn = ts.swin_fpn(sdg, ref_feats)
        ref_outs = [tr.head_single(sdg, f)[:3] for f in ref_fpn]
    feats = sw.forward(img)
    worst = 0.0
    for a, b in zip(feats, ref_feats):
        worst = max(worst, _rel(e.to_float(a).permute(0, 3, 1, 2).double(), b))
    outs, fpn = det.forward_dense(img)
    for lvl in range(5):
        worst = max(worst, _rel(e.to_float(fpn[lvl]).permute(0, 3, 1, 2).double(), ref_fpn[lvl]))
        for k in range(3):
            a, b = outs[lvl][k].permute(0, 3, 1, 2).double(), ref_outs[lvl][k]
            worst = max(worst, float((a - b).abs().max()) / max(1.0, float(b.abs().max())))
    print("Swin-T f16x3 vs fp64 graph: max rel err %.2e" % worst)
    assert worst < 1e-4
    assert e.overflow_count() == 0
    res = det.simple_test(img)
    assert len(res) == 2 and len(res[0]) == 15


@pytest.mark.parametrize("precision", ["bf16", "f16x3"])
def test_swin_uint8_tiles_equal_normalized_float_input(cuda, swin_sd, precision):
    """decoded uint8 HWC tiles through the fused Normalize + patch gather == the pipeline's Normalize / ImageToTensor done with
    torch ops followed by the float entry point: identical bits (same two fp32 roundings per pixel)"""
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    det = OrientedRepPointsDetector(swin_sd, "swin_tiny", cuda, precision, test_cfg=dict(score_thr=0.02))
    u8 = torch.randint(0, 256, (2, 122, 95, 3), generator=torch.Generator().manual_seed(5), dtype=torch.uint8).to(cuda)
    fa = det.swin.forward(u8, det.img_norm_cfg)
    fb = det.swin.forward(det.normalize(u8))
    for a, b in zip(fa, fb):
        assert torch.equal(det.eng.to_float(a), det.eng.to_float(b))
