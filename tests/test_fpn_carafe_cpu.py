"""FPN_CARAFE without a GPU: the fp64 restatement (tests/fpn_carafe_ref.py) against the reference's own FPN_CARAFE and
CARAFEPack (tests/golden/fpn_carafe_ref.npz), the carafe semantics element by element, the config-built trees and keys, the
init, unchanged draws without the option, every refusal, the engine's state-dict check and the header bindings."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

from orientedreppoints_b200 import _lib
from orientedreppoints_b200.carafe_fpn import check_neck
from orientedreppoints_b200.models import FPN_CARAFE, build_detector
from orientedreppoints_b200.swin import random_swin_state_dict
from orientedreppoints_b200.weights import fpn_carafe_keys, fpn_carafe_spec, random_state_dict
import fpn_carafe_ref as fr

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = np.load(os.path.join(HERE, "golden", "fpn_carafe_ref.npz"))
TAGS = [c["tag"] for c in fr.CASES]
# the FPN_CARAFE convolutions (channel_compressor, the content_encoder's fp32 output of 100 channels, the biased laterals and
# fpn_convs, the GN ones at the 960^2 test scale and at one tile) reach plan signatures no case of tests/conv_plan_cases.PARITY
# pins: R-50 FPN_CARAFE (GN or no norm, the default upsample_cfg) at 16 x 1024^2, 1 x 1024^2 and 4 x 960^2.  Their cases, in
# PARITY's format, at the shape of the first layer that reaches each
CARAFE_PARITY = [
    # f16x3 x16 1024 comp0
    (('f16x3', 0, 'split', 64, 1, 1, 0, 0, 0, 1, 1, 0, 3, 0, 1, 0, 0, 1, 0, 0), 'f16x3', 'conv', 256, 64, 1, 1, 1, 0, 0, 0, 0, [(16, 64, 64)]),
    # f16x3 x16 1024 enc0
    (('f16x3', 0, 'f32', 128, 0, 0, 0, 0, 0, 0, 1, 0, 5, 0, 1, 0, 0, 1, 1, 0), 'f16x3', 'conv', 64, 100, 3, 1, 1, 0, 1, 0, 0, [(16, 64, 64)]),
    # f16x3 x16 1024 enc1
    (('f16x3', 0, 'f32', 128, 0, 0, 0, 0, 0, 0, 1, 0, 5, 0, 1, 0, 0, 0, 1, 0), 'f16x3', 'conv', 64, 100, 3, 1, 1, 0, 1, 0, 0, [(16, 32, 32)]),
    # f16x3 x16 1024 enc2, enc3; x1 1024 enc0..3; x4 960 enc1..3
    (('f16x3', 0, 'f32', 64, 0, 0, 0, 0, 0, 0, 1, 0, 6, 0, 1, 0, 0, 0, 1, 0), 'f16x3', 'conv', 64, 100, 3, 1, 1, 0, 1, 0, 0, [(16, 16, 16)]),
    # f16x3 x4 960 enc0
    (('f16x3', 0, 'f32', 64, 0, 0, 0, 0, 0, 0, 1, 0, 6, 0, 1, 0, 0, 1, 1, 0), 'f16x3', 'conv', 64, 100, 3, 1, 1, 0, 1, 0, 0, [(4, 60, 60)]),
    # bf16 x16 1024 enc0
    (('bf16', 0, 'f32', 128, 0, 0, 0, 0, 0, 0, 1, 0, 5, 0, 1, 0, 0, 1, 1, 0), 'bf16', 'conv', 64, 100, 3, 1, 1, 0, 1, 0, 0, [(16, 64, 64)]),
    # bf16 x16 1024 comp1..3; x1 1024 comp0..3; x4 960 comp0..3
    (('bf16', 0, 'bf16', 64, 1, 0, 0, 0, 1, 0, 2, 0, 6, 0, 1, 0, 0, 0, 0, 0), 'bf16', 'conv', 256, 64, 1, 1, 1, 0, 0, 0, 0, [(16, 32, 32)]),
    # bf16 x16 1024 enc1
    (('bf16', 0, 'f32', 128, 0, 0, 0, 0, 0, 0, 1, 0, 5, 0, 1, 0, 0, 0, 1, 0), 'bf16', 'conv', 64, 100, 3, 1, 1, 0, 1, 0, 0, [(16, 32, 32)]),
    # bf16 x16 1024 enc2, enc3; x1 1024 enc0..3; x4 960 enc1..3
    (('bf16', 0, 'f32', 64, 0, 0, 0, 0, 1, 0, 1, 0, 6, 0, 1, 0, 0, 0, 1, 0), 'bf16', 'conv', 64, 100, 3, 1, 1, 0, 1, 0, 0, [(16, 16, 16)]),
    # bf16 x4 960 GN lat1, fpn1
    (('bf16', 0, 'bf16', 128, 1, 0, 0, 0, 0, 0, 1, 1, 5, 0, 0, 0, 0, 1, 0, 0), 'bf16', 'conv', 1024, 256, 1, 1, 0, 0, 0, 0, 1, [(4, 60, 60)]),
    # bf16 x4 960 and x1 1024: lat3, lat4, fpn3, fpn4 (split-K)
    (('bf16', 0, 'f32', 64, 0, 0, 0, 0, 0, 0, 1, 0, 6, 0, 0, 1, 0, 0, 0, 0), 'bf16', 'conv', 256, 256, 3, 2, 0, 0, 0, 0, 1, [(4, 15, 15)]),
    # bf16 x4 960 enc0
    (('bf16', 0, 'f32', 64, 0, 0, 0, 0, 1, 0, 1, 0, 6, 0, 1, 0, 0, 1, 1, 0), 'bf16', 'conv', 64, 100, 3, 1, 1, 0, 1, 0, 0, [(4, 60, 60)]),
    # bf16 x4 960 biased lat1, fpn1
    (('bf16', 0, 'bf16', 128, 1, 0, 0, 0, 0, 0, 1, 0, 5, 0, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 1024, 256, 1, 1, 1, 0, 0, 0, 0, [(4, 60, 60)]),
    # bf16 x1 1024 GN lat0
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 0, 0, 0, 2, 1, 3, 0, 0, 0, 0, 0, 0, 0), 'bf16', 'conv', 512, 256, 1, 1, 0, 0, 0, 0, 1, [(1, 128, 128)]),
    # bf16 x1 1024 biased lat0
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 0, 0, 0, 2, 0, 3, 0, 1, 0, 0, 0, 0, 0), 'bf16', 'conv', 512, 256, 1, 1, 1, 0, 0, 0, 0, [(1, 128, 128)]),
]
GN = dict(type='GN', num_groups=32, requires_grad=True)
HEAD = dict(type='OrientedRepPointsHead', num_classes=16, in_channels=256, feat_channels=256, point_feat_channels=256,
            stacked_convs=3, num_points=9, gradient_mul=0.3, point_strides=[8, 16, 32, 64, 128], point_base_scale=2, norm_cfg=GN)
R50 = dict(type='ResNet', depth=50, num_stages=4, out_indices=(0, 1, 2, 3), frozen_stages=1, style='pytorch')
SWIN_T = dict(type='SwinTransformer', embed_dim=96, depths=[2, 2, 6, 2], num_heads=[3, 6, 12, 24], window_size=7, out_indices=(1, 2, 3))


def case(tag):
    return next(c for c in fr.CASES if c["tag"] == tag)


def neck(in_channels=(256, 512, 1024, 2048), start_level=1, **kw):
    return dict(type='FPN_CARAFE', in_channels=list(in_channels), out_channels=256, num_outs=5, start_level=start_level, **kw)


@pytest.mark.parametrize("tag", TAGS)
def test_restatement_vs_reference(tag):
    c = case(tag)
    sd = {k: v.double() for k, v in fr.weights(c).items()}
    with torch.no_grad():
        levels = fr.neck(sd, fr.spec_of(c), fr.inputs(c))
    sizes = fr.level_sizes(*c["hw"])
    for i, lv in enumerate(levels):
        assert tuple(lv.shape[2:]) == sizes[i]
        g = torch.from_numpy(GOLD["%s/level%d" % (tag, i)]).double()
        a = lv[:, :fr.OUT_CHANNELS]
        assert a.shape == g.shape
        assert float((a - g).abs().max()) <= 1e-6 * max(1.0, float(g.abs().max())), (tag, i)


def test_carafe_semantics_elementwise():
    """the logit index ((g k^2 + t) 4 + (oy % 2) 2 + ox % 2) at (oy / 2, ox / 2), the softmax over all k^2 taps, the border
    taps skipped without renormalising, channel c in group c / (C / G)"""
    g = torch.Generator().manual_seed(0)
    n, c, h, w, k, grp = 1, 8, 3, 4, 3, 2
    x = torch.randn((n, c, h, w), generator=g, dtype=torch.float64)
    logits = 2 * torch.randn((n, k * k * grp * 4, h, w), generator=g, dtype=torch.float64)
    got = fr.carafe(x, logits, k, grp)
    r = (k - 1) // 2
    for ch in range(c):
        gi = ch // (c // grp)
        for oy in range(2 * h):
            for ox in range(2 * w):
                lg = torch.stack([logits[0, (gi * k * k + t) * 4 + (oy % 2) * 2 + ox % 2, oy // 2, ox // 2] for t in range(k * k)])
                wt = torch.softmax(lg, 0)
                want = 0.0
                for t in range(k * k):
                    iy, ix = oy // 2 + t // k - r, ox // 2 + t % k - r
                    if 0 <= iy < h and 0 <= ix < w:
                        want += float(wt[t] * x[0, ch, iy, ix])
                assert abs(float(got[0, ch, oy, ox]) - want) < 1e-12
    ones = fr.carafe(torch.ones((1, 8, 3, 3), dtype=torch.float64), torch.zeros((1, 9 * 4, 3, 3), dtype=torch.float64), 3, 1)
    assert float(ones[0, 0, 0, 0]) == pytest.approx(4 / 9) and float(ones[0, 0, 2, 2]) == pytest.approx(1.0)


@pytest.mark.parametrize("tag", TAGS)
def test_config_tree_keys_equal_the_reference(tag):
    c = case(tag)
    cfg = fr.neck_cfg(c)
    cfg.pop("type")
    m = FPN_CARAFE(**cfg)
    ref = dict(zip(["neck." + k for k in GOLD["%s/keys" % tag]], [tuple(int(d) for d in s.split(",")) for s in GOLD["%s/shapes" % tag]]))
    ours = {"neck." + k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert list(ours) == list(ref)
    assert ours == ref == fpn_carafe_keys(m.spec)


@pytest.mark.parametrize("backbone", ["r50", "x50", "swin"])
def test_detector_builds_and_inits_like_the_reference(backbone):
    if backbone == "swin":
        bb, nk = SWIN_T, neck((192, 384, 768), 0, norm_cfg=GN)
    else:
        bb = R50 if backbone == "r50" else dict(R50, type='ResNeXt', groups=32, base_width=4)
        nk = neck(norm_cfg=GN)
    m = build_detector(dict(type='OrientedRepPointsDetector', backbone=bb, neck=nk, bbox_head=HEAD))
    sd = m.state_dict()
    assert {k: tuple(v.shape) for k, v in sd.items() if k.startswith("neck.")} == fpn_carafe_keys(m.neck.spec)
    if backbone == "swin":
        return                                                  # the Swin draw randomises its neck's norms and biases
    for j in range(4):
        w = sd["neck.upsample_modules.%d.content_encoder.weight" % j]
        assert 0.0008 < float(w.std()) < 0.0012 and float(sd["neck.upsample_modules.%d.content_encoder.bias" % j].abs().max()) == 0
        cw = sd["neck.upsample_modules.%d.channel_compressor.weight" % j]
        assert float(cw.abs().max()) <= math.sqrt(6.0 / (256 + 64))                 # xavier-uniform bound
    assert float(sd["neck.lateral_convs.3.gn.weight"].min()) == 1.0 and "neck.lateral_convs.3.conv.bias" not in sd


def test_draws_without_the_option_unchanged():
    def fp(sd):
        return sum(float(v.double().abs().sum()) * (i + 1) for i, (k, v) in enumerate(sorted(sd.items())))
    # fingerprints of the draws before FPN_CARAFE existed
    assert fp(random_state_dict(50, seed=0)) == pytest.approx(198209202.6039899, rel=1e-12)
    assert fp(random_state_dict(50, seed=5, reference_init=False)) == pytest.approx(225502612.1176003, rel=1e-12)
    assert fp(random_swin_state_dict(0)) == pytest.approx(88728404.41940056, rel=1e-12)
    spec = fpn_carafe_spec((512, 1024, 2048), 256, GN)
    a, b = random_state_dict(50, seed=0), random_state_dict(50, seed=0, neck=spec)
    assert all(torch.equal(a[k], b[k]) for k in a if k.startswith("backbone."))


def test_gain_spreads_the_logits():
    spec = fpn_carafe_spec((512, 1024, 2048), 256, GN)
    sd = random_state_dict(50, seed=0, reference_init=False, neck=spec, carafe_gain=3.0)
    x = torch.randn(1, 256, 16, 16, generator=torch.Generator().manual_seed(0))
    p = "neck.upsample_modules.0."
    comp = torch.nn.functional.conv2d(x, sd[p + "channel_compressor.weight"], sd[p + "channel_compressor.bias"])
    lg = torch.nn.functional.conv2d(comp, sd[p + "content_encoder.weight"], sd[p + "content_encoder.bias"], padding=1)
    assert float(lg.std()) > 2.0                                  # several units: a peaked softmax


@pytest.mark.parametrize("kw,exc,word", [
    (dict(upsample_cfg=dict(type='nearest')), NotImplementedError, "nearest"),
    (dict(upsample_cfg=dict(type='bilinear')), NotImplementedError, "bilinear"),
    (dict(upsample_cfg=dict(type='deconv', upsample_kernel=3)), ValueError, "deconv"),
    (dict(upsample_cfg=dict(type='pixel_shuffle', upsample_kernel=3)), ValueError, "pixel_shuffle"),
    (dict(upsample_cfg=None), ValueError, "slice_as"),
    (dict(upsample_cfg=dict(type=None)), ValueError, "slice_as"),
    (dict(upsample_cfg=dict(type='carafe', up_kernel=4)), ValueError, "up_kernel"),
    (dict(upsample_cfg=dict(type='carafe', up_kernel=9)), NotImplementedError, "up_kernel"),
    (dict(upsample_cfg=dict(type='carafe', up_group=3)), ValueError, "up_group"),
    (dict(upsample_cfg=dict(type='carafe', up_group=8)), NotImplementedError, "up_group"),
    (dict(upsample_cfg=dict(type='carafe', encoder_kernel=5)), NotImplementedError, "encoder_kernel"),
    (dict(upsample_cfg=dict(type='carafe', encoder_dilation=2)), NotImplementedError, "encoder_dilation"),
    (dict(upsample_cfg=dict(type='carafe', compressed_channels=12)), NotImplementedError, "compressed_channels"),
    (dict(upsample_cfg=dict(type='carafe', scale=2)), ValueError, "scale"),
    (dict(norm_cfg=dict(type='BN')), NotImplementedError, "norm_cfg"),
    (dict(norm_cfg=dict(type='GN', num_groups=16)), NotImplementedError, "norm_cfg"),
    (dict(act_cfg=dict(type='LeakyReLU')), NotImplementedError, "act_cfg"),
    (dict(act_cfg=dict(type='ReLU'), order=('act', 'conv', 'norm')), NotImplementedError, "order"),
    (dict(order=('norm', 'conv', 'act')), ValueError, "order"),
    (dict(end_level=3), NotImplementedError, "end_level"),
    (dict(num_outs=6), NotImplementedError, "num_outs"),
    (dict(start_level=0), NotImplementedError, "start_level"),
    (dict(num_outs=2), ValueError, "num_outs"),
    (dict(out_channels=128), NotImplementedError, "out_channels"),
])
def test_refusals(kw, exc, word):
    cfg = neck(norm_cfg=GN)
    cfg.update(kw)
    cfg.pop("type")
    with pytest.raises(exc, match=word):
        FPN_CARAFE(**cfg)


def test_accepted_forms():
    base = neck()
    base.pop("type")
    m = FPN_CARAFE(**dict(base, order=('act', 'conv', 'norm')))           # the same graph without an activation
    assert m.spec == FPN_CARAFE(**base).spec
    for k in (1, 3, 5, 7):
        for g in (1, 2, 4):
            FPN_CARAFE(**dict(base, upsample_cfg=dict(type='carafe', up_kernel=k, up_group=g, encoder_kernel=1,
                                                      compressed_channels=8)))


def test_detector_level_refusals():
    with pytest.raises(ValueError, match="in_channels"):
        build_detector(dict(type='OrientedRepPointsDetector', backbone=SWIN_T, neck=neck((96, 192, 384, 768), 1), bbox_head=HEAD))
    with pytest.raises(ValueError, match="in_channels"):
        build_detector(dict(type='OrientedRepPointsDetector', backbone=R50, neck=neck((256, 512, 1024, 1024)), bbox_head=HEAD))
    with pytest.raises(ValueError, match="in_channels"):
        build_detector(dict(type='OrientedRepPointsDetector', backbone=R50, neck=neck(norm_cfg=GN),
                            bbox_head=dict(HEAD, in_channels=128)))
    hr = dict(type='HRNet', extra=dict(
        stage1=dict(num_modules=1, num_branches=1, block='BOTTLENECK', num_blocks=(4,), num_channels=(64,)),
        stage2=dict(num_modules=1, num_branches=2, block='BASIC', num_blocks=(4, 4), num_channels=(18, 36)),
        stage3=dict(num_modules=4, num_branches=3, block='BASIC', num_blocks=(4, 4, 4), num_channels=(18, 36, 72)),
        stage4=dict(num_modules=3, num_branches=4, block='BASIC', num_blocks=(4, 4, 4, 4), num_channels=(18, 36, 72, 144))))
    with pytest.raises(NotImplementedError, match="FPN_CARAFE"):
        build_detector(dict(type='OrientedRepPointsDetector', backbone=hr, neck=neck((18, 36, 72, 144)), bbox_head=HEAD))


def test_engine_checks_the_state_dict():
    spec = fpn_carafe_spec((512, 1024, 2048), 256, None, dict(type='ReLU'))
    sd = {k: torch.zeros(s) for k, s in fpn_carafe_keys(spec).items()}
    check_neck(sd, spec)
    for bad, word in ((lambda d: d.pop("neck.fpn_convs.2.conv.bias"), "missing"),
                      (lambda d: d.__setitem__("neck.fpn_convs.2.gn.weight", torch.ones(256)), "unexpected"),
                      (lambda d: d.__setitem__("neck.upsample_modules.1.content_encoder.weight", torch.zeros(36, 64, 3, 3)),
                       "wrong shape")):
        d = dict(sd)
        bad(d)
        with pytest.raises(ValueError, match=word):
            check_neck(d, spec)


def test_carafe_parity_case_plans():
    from conv_plan_cases import PARITY, planned, signature
    for c in CARAFE_PARITY:
        assert signature(planned(c)) == c[0] and c[0] not in {p[0] for p in PARITY}


def test_header_symbols_bound_with_arity():
    with open(os.path.join(ROOT, "include", "orp_b200_carafe.h")) as f:
        src = f.read()
    decl = dict(re.findall(r"^int (orp_\w+)\(([^;]*)\);", src, re.M | re.S))
    assert set(decl) == set(_lib.CARAFE_SIGNATURES) == {"orp_carafe_add_bf16", "orp_carafe_add_f16x3", "orp_carafe_add_f32"}
    lib = _lib.lib()
    for name, args in decl.items():
        assert len(args.split(",")) == len(_lib.CARAFE_SIGNATURES[name][1]), name
        assert isinstance(getattr(lib, name), ctypes._CFuncPtr)
    for other in ("orp_b200.h", "orp_b200_dcnv2.h", "orp_b200_swin.h", "orp_b200_group.h", "orp_b200_hrnet.h", "orp_b200_attention.h",
                  "orp_b200_context.h"):
        with open(os.path.join(ROOT, "include", other)) as f:
            assert not any(name in f.read() for name in decl), other
