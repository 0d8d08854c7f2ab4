"""GPU: the Swin backbones beyond Swin-T/w7 (Swin-S/B/L, 7x7 and 12x12 windows) in both tensor-core formats.  The 12x12
window attention (orp_window_attention12_*) and the wide LayerNorm (orp_layernorm_wide_*) against fp64 and their refusals;
whole backbone + FPN + head graphs against the fp64 oracle (f16x3) and torch (bf16); uint8 input; a config-built model
through init_detector / inference_detector / aug_test; every convolution launch of a Swin-B/w12 8 x 1024^2 step against fp64;
the new entry points on a side stream."""
import os

import pytest
import torch
import torch.nn.functional as F

from orientedreppoints_b200 import _lib

pytestmark = pytest.mark.gpu

ORP_EINVAL = -1
FMTS = ["bf16", "f16x3"]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rel(a, b):
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def _engine(prec, dev):
    from orientedreppoints_b200.engine_tc import EngineTC, EngineTCSplit
    return EngineTCSplit(dev) if prec == "f16x3" else EngineTC(dev)


def _attention_ref(x64, h, w, heads, shift, table64, ws, scale=None):
    """fp64 (shifted) window attention of qkv [B,Hp,Wp,3C] (tests/swin_arch_ref.py), at the original positions"""
    import swin_arch_ref as sr
    return sr.window_attention(x64, h, w, heads, shift, table64, ws, scale)


def _run_attention12(e, x32, b, h, w, heads, shift, table, scale):
    c = heads * 32
    hp, wp = x32.shape[1], x32.shape[2]
    xin = e.from_float(x32)
    out = e.alloc(b, h, w, c)
    _lib.check(getattr(_lib.lib(), "orp_window_attention12_%s" % e.suffix)(
        _lib.ptr(xin), b, h, w, hp, wp, c, heads, shift, _lib.ptr(table), scale, _lib.ptr(out), _lib.current_stream_ptr()),
        "orp_window_attention12")
    return e.to_float(out), e.to_float(xin)


def _check_attention12(dev, prec, b, h, w, heads, shift, seed, scale=None):
    e = _engine(prec, dev)
    c, hp, wp = heads * 32, -(-h // 12) * 12, -(-w // 12) * 12
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(b, hp, wp, 3 * c, generator=g, device=dev)
    table = torch.randn(529, heads, generator=g, device=dev) * 0.5
    s = float(32 ** -0.5) if scale is None else scale
    out, held = _run_attention12(e, x, b, h, w, heads, shift, table, s)
    del x
    ref = _attention_ref(held.double(), h, w, heads, shift, table.double(), 12, scale)
    err = _rel(out.double(), ref)
    assert err < (5e-6 if prec == "f16x3" else 6e-3), (prec, b, h, w, heads, shift, err)
    if prec == "f16x3":
        assert e.overflow_count() == 0
    return err


# every stage of Swin-B (heads 4 / 8 / 16 / 32) for 8 tiles of 1024^2 and of 960^2 (the test pipeline's scale)
STAGES = [(t >> (2 + i), 4 << i) for t in (1024, 960) for i in range(4)]


@pytest.mark.parametrize("prec", FMTS)
@pytest.mark.parametrize("h,heads", STAGES, ids=["%dx%d-h%d" % (h, h, n) for h, n in STAGES])
@pytest.mark.parametrize("shift", [0, 6])
def test_attention12_stage_shapes_vs_fp64(cuda, prec, h, heads, shift):
    _check_attention12(cuda, prec, 8, h, h, heads, shift, seed=h * 100 + heads + shift)
    torch.cuda.empty_cache()


# odd and padded grids, grids smaller than one window, one window, heads 4..48, a qk_scale other than head_dim ** -0.5
EDGES = [(1, 12, 12, 4, 6, None), (1, 12, 12, 4, 0, None), (2, 5, 7, 8, 6, None), (2, 11, 3, 6, 0, None), (2, 13, 25, 16, 6, None),
         (1, 23, 11, 32, 0, None), (3, 30, 30, 48, 6, None), (1, 24, 36, 12, 6, None), (2, 1, 1, 4, 6, None), (1, 37, 49, 24, 6, 0.1)]


@pytest.mark.parametrize("prec", FMTS)
@pytest.mark.parametrize("b,h,w,heads,shift,scale", EDGES)
def test_attention12_edges_vs_fp64(cuda, prec, b, h, w, heads, shift, scale):
    _check_attention12(cuda, prec, b, h, w, heads, shift, seed=b * 1000 + h * 37 + w + heads, scale=scale)


@pytest.mark.parametrize("prec", FMTS)
@pytest.mark.parametrize("c", [1544, 2048, 3072])
def test_layernorm_wide_vs_fp64(cuda, prec, c):
    """into a padded grid (the interior written, the rest left as the caller zeroed it), as the PatchMerging norms run"""
    e = _engine(prec, cuda)
    g = torch.Generator().manual_seed(c)
    x = (torch.randn(2, 9, 11, c, generator=g) * 3 + 1).to(cuda)
    gamma = (torch.rand(c, generator=g) + 0.5).to(cuda)
    beta = torch.randn(c, generator=g).to(cuda)
    xin = e.from_float(x)
    y = e.alloc(2, 12, 13, c, zero=True)
    _lib.check(getattr(_lib.lib(), "orp_layernorm_wide_%s" % e.suffix)(_lib.ptr(xin), 2, 9, 11, c, _lib.ptr(gamma), _lib.ptr(beta),
                                                                        1e-5, 12, 13, _lib.ptr(y), _lib.current_stream_ptr()),
               "orp_layernorm_wide")
    yf = e.to_float(y)
    ref = F.layer_norm(e.to_float(xin).double(), (c,), gamma.double(), beta.double(), 1e-5)
    assert _rel(yf[:, :9, :11].double(), ref) < (2e-6 if prec == "f16x3" else 8e-3)
    assert float(yf[:, 9:].abs().max()) == 0 and float(yf[:, :, 11:].abs().max()) == 0


def test_invalid_launches_are_refused(cuda):
    lib, st = _lib.lib(), _lib.current_stream_ptr()
    big = torch.zeros(1 << 22, dtype=torch.float16, device=cuda)
    out = torch.full((1 << 22,), 7.0, dtype=torch.float16, device=cuda)
    gamma = torch.ones(4096, device=cuda)
    table = torch.zeros(529 * 48, device=cuda)
    p, o, gp, tp = _lib.ptr(big), _lib.ptr(out), _lib.ptr(gamma), _lib.ptr(table)
    scale = 32 ** -0.5
    for fmt in FMTS:
        ln = getattr(lib, "orp_layernorm_wide_%s" % fmt)
        assert ln(p, 1, 2, 2, 1536, gp, gp, 1e-5, 2, 2, o, st) == ORP_EINVAL          # C <= 1536: orp_layernorm_*
        assert ln(p, 1, 2, 2, 3080, gp, gp, 1e-5, 2, 2, o, st) == ORP_EINVAL          # C > 3072
        assert ln(p, 1, 2, 2, 2052, gp, gp, 1e-5, 2, 2, o, st) == ORP_EINVAL          # C % 8
        assert ln(p, 1, 2, 2, 2048, gp, gp, 1e-5, 1, 2, o, st) == ORP_EINVAL          # Hp < H
        assert ln(p, 1, 2, 2, 2048, gp, gp, 1e-5, 2, 1, o, st) == ORP_EINVAL          # Wp < W
        at = getattr(lib, "orp_window_attention12_%s" % fmt)
        assert at(p, 1, 12, 12, 12, 12, 128, 4, 0, tp, scale, o, st) == 0
        torch.cuda.synchronize()
        out.fill_(7.0)
        assert at(p, 1, 12, 12, 12, 12, 128, 3, 0, tp, scale, o, st) == ORP_EINVAL   # heads * 32 != C
        assert at(p, 1, 12, 12, 12, 12, 128, 4, 12, tp, scale, o, st) == ORP_EINVAL  # shift >= 12
        assert at(p, 1, 12, 12, 12, 12, 128, 4, -1, tp, scale, o, st) == ORP_EINVAL  # shift < 0
        assert at(p, 1, 12, 13, 12, 13, 128, 4, 0, tp, scale, o, st) == ORP_EINVAL   # Wp % 12
        assert at(p, 1, 13, 12, 13, 12, 128, 4, 0, tp, scale, o, st) == ORP_EINVAL   # Hp % 12
        assert at(p, 1, 7, 7, 7, 7, 128, 4, 0, tp, scale, o, st) == ORP_EINVAL       # a 7x7 grid: orp_window_attention_*
    torch.cuda.synchronize()
    assert bool((out == 7.0).all()), "a refused call wrote its output"


# ------------------------------------------------------------------------------------------------ whole graphs
GRAPHS = ["swin_small", "swin_base", "swin_base_w12", "swin_large_w12"]


def _detector(name, prec, dev, **kw):
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    from orientedreppoints_b200.swin import ARCHS, random_swin_state_dict
    sd = random_swin_state_dict(0, arch=ARCHS[name])
    return sd, OrientedRepPointsDetector(sd, name, dev, prec, test_cfg=dict(score_thr=0.02), **kw)


@pytest.mark.parametrize("name", GRAPHS)
def test_f16x3_graph_vs_fp64(cuda, name):
    """backbone + FPN + head in f16x3 against the fp64 evaluation of the reference graph (tests/swin_arch_ref.py, pinned to the
    reference's own module for these architectures by tests/test_swin_variants_cpu.py), within north_star's 1e-4"""
    import swin_arch_ref as ts
    from oracle import torch_reference as tr
    from orientedreppoints_b200.swin import ARCHS
    sd, det = _detector(name, "f16x3", cuda)
    e = det.eng
    e.overflow_count()
    img = torch.randn(2, 3, 250, 198, generator=torch.Generator().manual_seed(3)).to(cuda)
    sdg = {k: v.to(cuda).double() for k, v in sd.items()}
    with torch.no_grad():
        ref_feats = ts.swin_forward(sdg, img.double(), arch=ARCHS[name])
        ref_fpn = ts.swin_fpn(sdg, ref_feats)
        ref_outs = [tr.head_single(sdg, f)[:3] for f in ref_fpn]
    worst = 0.0
    for a, b in zip(det.swin.forward(img), ref_feats):
        assert a.shape[:3] == (b.shape[0], b.shape[2], b.shape[3])
        worst = max(worst, _rel(e.to_float(a).permute(0, 3, 1, 2).double(), b))
    outs, fpn = det.forward_dense(img)
    for lvl in range(5):
        worst = max(worst, _rel(e.to_float(fpn[lvl]).permute(0, 3, 1, 2).double(), ref_fpn[lvl]))
        for k in range(3):
            a, b = outs[lvl][k].permute(0, 3, 1, 2).double(), ref_outs[lvl][k]
            worst = max(worst, float((a - b).abs().max()) / max(1.0, float(b.abs().max())))
    print("%s f16x3 vs fp64 graph: max rel err %.2e" % (name, worst))
    assert worst < 1e-4
    assert e.overflow_count() == 0
    res = det.simple_test(img)
    assert len(res) == 2 and len(res[0]) == 15


@pytest.mark.parametrize("name", GRAPHS)
def test_bf16_graph_vs_torch(cuda, name):
    """bf16 against the fp32 torch evaluation of the reference graph, with the tolerances of the Swin-T bf16 test"""
    import swin_arch_ref as ts
    from oracle import torch_reference as tr
    from orientedreppoints_b200.swin import ARCHS
    sd, det = _detector(name, "bf16", cuda)
    img = torch.randn(2, 3, 250, 198, generator=torch.Generator().manual_seed(3)).to(cuda)
    sdg = {k: v.to(cuda) for k, v in sd.items()}
    tf32 = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            ref_feats = ts.swin_forward(sdg, img, arch=ARCHS[name])
            ref_fpn = ts.swin_fpn(sdg, ref_feats)
            ref_outs = [tr.head_single(sdg, f)[:3] for f in ref_fpn]
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    for a, b in zip(det.swin.forward(img), ref_feats):
        assert _rel(a.float().permute(0, 3, 1, 2), b) < 0.05
    outs, fpn = det.forward_dense(img)
    for lvl in range(5):
        assert _rel(fpn[lvl].float().permute(0, 3, 1, 2), ref_fpn[lvl]) < 0.08, lvl
        for k in range(3):
            a, b = outs[lvl][k].permute(0, 3, 1, 2), ref_outs[lvl][k]
            assert float((a - b).abs().max()) < 0.1 * max(1.0, float(b.abs().max())), (lvl, k)


@pytest.mark.parametrize("prec", FMTS)
def test_uint8_tiles_equal_normalized_float_input(cuda, prec):
    _, det = _detector("swin_base_w12", prec, cuda)
    u8 = torch.randint(0, 256, (2, 122, 95, 3), generator=torch.Generator().manual_seed(5), dtype=torch.uint8).to(cuda)
    fa = det.swin.forward(u8, det.img_norm_cfg)
    fb = det.swin.forward(det.normalize(u8))
    for a, b in zip(fa, fb):
        assert torch.equal(det.eng.to_float(a), det.eng.to_float(b))


def test_config_built_swin_b_w12(cuda):
    """the Swin-T config with backbone and neck overridden to Swin-B / window 12: init_detector, inference_detector, aug_test"""
    import numpy as np
    from orientedreppoints_b200.apis import Config, inference_detector, init_detector
    cfg = Config.fromfile(os.path.join(ROOT, "configs", "dota", "orientedrepoints_swin_tiny_demo.py"))
    cfg['model']['backbone'].update(embed_dim=128, depths=[2, 2, 18, 2], num_heads=[4, 8, 16, 32], window_size=12)
    cfg['model']['neck'].update(in_channels=[256, 512, 1024])
    cfg['test_cfg'] = dict(cfg['test_cfg'], score_thr=0.02)
    model = init_detector(cfg, None, device=cuda)
    assert model.backbone.arch.window == 12 and model.engine().swin.arch.embed == 128
    img = np.random.RandomState(0).randint(0, 256, (300, 410, 3)).astype(np.uint8)
    res = inference_detector(model, img)
    assert len(res) == 15 and all(a.ndim == 2 and a.shape[1] == 27 for a in res)
    x = torch.randn(1, 3, 256, 256, generator=torch.Generator().manual_seed(3)).to(cuda)
    metas = [[dict(img_shape=(256, 256, 3), scale_factor=1.0, flip=False)], [dict(img_shape=(256, 256, 3), scale_factor=1.0, flip=True)]]
    aug = model.aug_test([x, x.flip(-1)], metas, rescale=True)
    assert len(aug) == 15


def test_every_conv_launch_of_swin_b_w12_step_vs_fp64(cuda, monkeypatch):
    """one eager forward_dense of 8 uint8 tiles of 1024^2 through Swin-B / window 12 in f16x3, every tensor-core launch checked
    against fp64 at its production shape by the checker of tests/test_production_launches_gpu.py"""
    import time
    import test_production_launches_gpu as tpl

    def names(det):
        out = {id(det.swin.embed): "patch_embed"}
        for i, stage in enumerate(det.swin.blocks):
            for j, blk in enumerate(stage):
                for k in ("qkv", "proj", "fc1", "fc2"):
                    out[id(blk[k])] = "stage%d.%d.%s" % (i, j, k)
        for i, m in enumerate(det.swin.merges):
            out[id(m["red"])] = "merge%d" % i
        for i, (L, _) in enumerate(det.lat):
            out[id(L)] = "lateral%d" % i
        for i, (L, _) in enumerate(det.fpn):
            out[id(L)] = "fpn%d" % i
        for i, ((lc, _), (lr, _)) in enumerate(zip(det.cls_convs, det.reg_convs)):
            out[id(lc)], out[id(lr)] = "cls_convs%d" % i, "reg_convs%d" % i
        for k in ("cls_dcn", "cls_out", "init_conv", "init_out", "ref_dcn", "ref_out"):
            out[id(getattr(det, k))] = k
        return out
    monkeypatch.setattr(tpl, "_layer_names", names)
    t0 = time.time()
    _, det = _detector("swin_base_w12", "f16x3", cuda)
    img = torch.randint(0, 256, (8, 1024, 1024, 3), generator=torch.Generator().manual_seed(1000), dtype=torch.uint8).to(cuda)
    chk = tpl.LaunchChecker(det, "swin_base_w12 f16x3 x8")
    det.eng.overflow_count()
    with torch.no_grad():
        det.forward_dense(img)
    torch.cuda.synchronize()
    line = chk.summary(time.time() - t0)
    print(line)
    assert not chk.escaped and chk.checked == chk.low and chk.checked > 100, line
    del det, chk
    torch.cuda.empty_cache()


def test_new_entry_points_on_a_side_stream(cuda):
    """each entry point of orp_b200_swin.h launched on a PyTorch side stream (behind a long kernel on it) gives the bits of
    the default-stream launch"""
    lib = _lib.lib()
    g = torch.Generator(device=cuda).manual_seed(9)
    for prec in FMTS:
        e = _engine(prec, cuda)
        qkv = e.from_float(torch.randn(2, 24, 36, 3 * 256, generator=g, device=cuda))
        table = torch.randn(529, 8, generator=g, device=cuda)
        x = e.from_float(torch.randn(2, 9, 11, 2048, generator=g, device=cuda))
        gamma, beta = torch.rand(2048, generator=g, device=cuda) + 0.5, torch.randn(2048, generator=g, device=cuda)

        def run():
            a = e.alloc(2, 20, 30, 256)
            _lib.check(getattr(lib, "orp_window_attention12_%s" % prec)(_lib.ptr(qkv), 2, 20, 30, 24, 36, 256, 8, 6, _lib.ptr(table),
                                                                         0.17, _lib.ptr(a), _lib.current_stream_ptr()), "attn12")
            y = e.alloc(2, 9, 11, 2048)
            _lib.check(getattr(lib, "orp_layernorm_wide_%s" % prec)(_lib.ptr(x), 2, 9, 11, 2048, _lib.ptr(gamma), _lib.ptr(beta),
                                                                     1e-5, 9, 11, _lib.ptr(y), _lib.current_stream_ptr()), "ln")
            return a, y
        ref = run()
        torch.cuda.synchronize()
        side = torch.cuda.Stream(cuda)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            big = torch.randn(4096, 4096, device=cuda)
            for _ in range(8):
                big = big @ big * 1e-3                                     # keeps the side stream busy before the launches
            got = run()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        for a, b in zip(got, ref):
            assert torch.equal(a, b), prec
