"""Generalized attention in ResNet backbones, without a GPU: the fp64 restatement (tests/gen_attention_ref.py) against the
reference's own GeneralizedAttention / ResNet (tests/golden/gen_attention_ref.npz), the config-built parameter trees and the
reference's initialisation, unchanged draws without attention, the refusals, the launch planner and the header bindings."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from orientedreppoints_b200 import _lib
from orientedreppoints_b200.models import build_backbone, build_detector
from orientedreppoints_b200.weights import (STAGE_BLOCKS, gen_attention_keys, gen_attention_layout, gen_attention_spec,
                                            random_state_dict)
import gen_attention_ref as gr

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = np.load(os.path.join(HERE, "golden", "gen_attention_ref.npz"))
PUB = dict(gr.PUBLISHED)


def _cfg(t, s, heads, mag=1, emb=-1):
    return dict(spatial_range=-1, num_heads=heads, kv_stride=s, attention_type=t, position_magnitude=mag, position_embedding_dim=emb)


@pytest.mark.parametrize("tag", sorted({k[:-5] for k in GOLD.files if k.endswith("_meta") and k.startswith("t")}))
def test_block_restatement_vs_reference(tag):
    tcode, s, heads, planes, h, w, mag, emb, seed = [int(v) for v in GOLD[tag + "_meta"]]
    t = format(tcode, "04b")
    li = (64, 128, 256, 512).index(planes)
    stages = [[], [], [], []]
    stages[li] = [0]
    c = _cfg(t, s, heads, mag, emb)
    sd = random_state_dict(50, seed=seed, reference_init=False, gen_attention=c, stage_with_gen_attention=stages,
                           gen_attention_gamma=0.7)
    blk = {k: v.double() for k, v in gr.block_params(sd, "backbone.layer%d.0" % (li + 1)).items()}
    torch.manual_seed(0)
    x = torch.randn(2, planes, h, w, generator=torch.Generator().manual_seed(seed + 100), dtype=torch.float64)
    y = gr.block(gen_attention_spec(c, planes), blk, x)
    ref = torch.from_numpy(GOLD[tag + "_y"]).double()                  # the first channels (all heads feed each through proj_conv)
    assert ref.shape == (2, 32, h, w)
    y, x = y[:, :32], x[:, :32]
    assert (y - x).abs().max() > 0.1                                   # the block acts
    assert torch.allclose(y, ref, rtol=1e-6, atol=1e-6), float((y - ref).abs().max())


@pytest.mark.parametrize("tag", ["r50_1111", "r50_0010"])
def test_backbone_restatement_vs_reference(tag):
    tcode, seed, h, w = [int(v) for v in GOLD[tag + "_meta"]]
    c = _cfg(format(tcode, "04b"), 2, 8)
    sd = {k: v.double() for k, v in random_state_dict(50, seed=seed, reference_init=False, residual_gain=0.5, gen_attention=c,
                                                       stage_with_gen_attention=gr.PUBLISHED_STAGES, gen_attention_gamma=0.7).items()}
    img = torch.randn(1, 3, h, w, generator=torch.Generator().manual_seed(seed + 10), dtype=torch.float64)
    feats = gr.backbone(sd, img, None, gen_attention_layout(50, c, gr.PUBLISHED_STAGES))
    for l in (2, 3):
        ref = torch.from_numpy(GOLD["%s_c%d" % (tag, l + 2)]).double()  # the first 64 channels
        got = feats[l][:, :ref.shape[1]]
        assert ref.shape[1] == 64 and got.shape == ref.shape
        assert torch.allclose(got, ref, rtol=1e-5, atol=1e-5 * float(ref.abs().max())), (l, float((got - ref).abs().max()))


def _detector_cfg(t, stages=gr.PUBLISHED_STAGES, dcn=None, **extra):
    bb = dict(type='ResNet', depth=50, num_stages=4, out_indices=(0, 1, 2, 3), frozen_stages=1, style='pytorch',
              gen_attention=dict(PUB, attention_type=t, **extra), stage_with_gen_attention=stages)
    if dcn:
        bb.update(dcn=dict(type='DCN', deformable_groups=1, fallback_on_stride=False), stage_with_dcn=(False, True, True, True))
    return dict(type='OrientedRepPointsDetector', backbone=bb,
                neck=dict(type='FPN', in_channels=[256, 512, 1024, 2048], out_channels=256, start_level=1, add_extra_convs=True,
                          num_outs=5, norm_cfg=dict(type='GN', num_groups=32, requires_grad=True)),
                bbox_head=dict(type='OrientedRepPointsHead', num_classes=16, in_channels=256, feat_channels=256,
                               point_feat_channels=256, stacked_convs=3, num_points=9, gradient_mul=0.3, point_strides=[8, 16, 32, 64, 128],
                               point_base_scale=2, norm_cfg=dict(type='GN', num_groups=32, requires_grad=True)))


@pytest.mark.parametrize("t", ["1111", "0010", "1000", "0001", "0101", "0000"])
@pytest.mark.parametrize("dcn", [False, True])
def test_config_tree_keys_and_init(t, dcn):
    m = build_detector(_detector_cfg(t, dcn=dcn))
    sd = m.state_dict()
    att = sorted(k for k in sd if ".gen_attention_block." in k)
    spec3, spec4 = gen_attention_spec(dict(PUB, attention_type=t), 256), gen_attention_spec(dict(PUB, attention_type=t), 512)
    want = sorted("backbone.layer3.%d.gen_attention_block.%s" % (b, k) for b in range(6) for k in gen_attention_keys(spec3)) + \
        sorted("backbone.layer4.%d.gen_attention_block.%s" % (b, k) for b in range(3) for k in gen_attention_keys(spec4))
    assert att == sorted(want)
    for k in att:                                                       # the reference's shapes (generalized_attention.py:60-109)
        assert tuple(sd[k].shape) == gen_attention_keys(spec3 if ".layer3." in k else spec4)[k.split(".gen_attention_block.")[1]]
    # the reference's init: kaiming fan_out convs with zero bias, appr / geom bias within +-1/sqrt(2d), gamma 0
    for k in att:
        v = sd[k]
        d = 32 if ".layer3." in k else 64
        if k.endswith("gamma") or k.endswith("proj_conv.bias"):
            assert torch.count_nonzero(v) == 0
        elif k.endswith("_bias"):
            assert v.abs().max() <= 1 / (2 * d) ** 0.5 and v.std() > 0.25 / (2 * d) ** 0.5
        elif "conv.weight" in k:
            assert abs(float(v.std()) - (2.0 / v.shape[0]) ** 0.5) < 0.05 * (2.0 / v.shape[0]) ** 0.5
        else:                                                           # appr_geom_fc: kaiming_uniform(a=1)
            assert v.abs().max() <= (3.0 / v.shape[1]) ** 0.5
    assert m.backbone.gen_attention_layout() == gen_attention_layout(50, dict(PUB, attention_type=t), gr.PUBLISHED_STAGES)


def test_draws_without_attention_unchanged():
    a = random_state_dict(50, seed=3, reference_init=False)
    for extra in (dict(gen_attention=None), dict(gen_attention=dict(PUB), stage_with_gen_attention=((), (), (), ()))):
        b = random_state_dict(50, seed=3, reference_init=False, **extra)
        assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)


def test_index_past_the_stage_builds_nothing():
    bb = build_backbone(dict(type='ResNet', depth=50, gen_attention=dict(PUB), stage_with_gen_attention=[[], [5, 9], [], [0, 2, 7]]))
    lay = bb.gen_attention_layout()
    assert [sum(sp is not None for sp in s) for s in lay] == [0, 0, 0, 2]          # layer2 has blocks 0-3, layer4 0-2
    assert lay[3][0] is not None and lay[3][1] is None and lay[3][2] is not None
    sd = random_state_dict(50, gen_attention=dict(PUB), stage_with_gen_attention=[[], [5, 9], [], [0, 2, 7]])
    assert sorted({k.split(".gen_attention_block")[0] for k in sd if "gen_attention_block" in k}) == \
        ["backbone.layer4.0", "backbone.layer4.2"]


@pytest.mark.parametrize("extra, exc, word", [
    (dict(spatial_range=4), NotImplementedError, "spatial_range"),
    (dict(q_stride=2), NotImplementedError, "q_stride"),
    (dict(kv_stride=4), NotImplementedError, "kv_stride"),
    (dict(num_heads=6), NotImplementedError, "num_heads"),
    (dict(num_heads=2), NotImplementedError, "num_heads"),                       # head dimension 128 at c4
    (dict(attention_type='0100'), NotImplementedError, "attention_type"),
    (dict(attention_type='1110'), NotImplementedError, "attention_type"),
    (dict(attention_type='11'), ValueError, "attention_type"),
    (dict(attention_type='1121'), ValueError, "attention_type"),
    (dict(position_embedding_dim=66), ValueError, "position_embedding_dim"),
    (dict(no_such=1), TypeError, "no_such"),
])
def test_refusals(extra, exc, word):
    with pytest.raises(exc, match=word):
        build_backbone(dict(type='ResNet', depth=50, gen_attention=dict(PUB, **extra), stage_with_gen_attention=gr.PUBLISHED_STAGES))


def test_resnext_refuses_attention():
    with pytest.raises(NotImplementedError, match=r"resnext\.py:196-216"):
        build_backbone(dict(type='ResNeXt', depth=50, groups=32, base_width=4, gen_attention=dict(PUB),
                            stage_with_gen_attention=gr.PUBLISHED_STAGES))
    build_backbone(dict(type='ResNeXt', depth=50, groups=32, base_width=4, gen_attention=dict(PUB)))   # selects no block: fine


def test_engine_checks_layout_against_state_dict():
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    lay = gen_attention_layout(50, dict(PUB), gr.PUBLISHED_STAGES)
    plain = random_state_dict(50)
    with pytest.raises(ValueError, match="gen_attention_block"):
        OrientedRepPointsDetector(plain, 50, "cpu", "fp32", gen_attention=lay)       # layout names blocks the weights lack
    sd = random_state_dict(50, gen_attention=dict(PUB), stage_with_gen_attention=gr.PUBLISHED_STAGES)
    with pytest.raises(ValueError, match="gen_attention_block"):
        OrientedRepPointsDetector(sd, 50, "cpu", "fp32")                             # weights hold blocks the layout lacks
    other = gen_attention_layout(50, dict(PUB, attention_type='0010'), gr.PUBLISHED_STAGES)
    with pytest.raises(ValueError, match="attention_type 0010"):
        OrientedRepPointsDetector(sd, 50, "cpu", "fp32", gen_attention=other)


# every attention launch of R-50 with the published c4-c5 layout at the tile sizes the test pipeline produces
LAUNCHES = [(1024, 64, 256, 32), (1024, 32, 512, 64), (960, 60, 256, 32), (960, 30, 512, 64)]


@pytest.mark.parametrize("fmt", ["bf16", "f16x3", "fp32"])
@pytest.mark.parametrize("tile, h, c, d", LAUNCHES)
def test_planner_published_launches(fmt, tile, h, c, d):
    hk = -(-h // 2)
    for n in (1, 16):
        p = _lib.gen_attention_plan_for(fmt, n, h, h, c, 8, 2)
        assert p["head_dim"] == d and p["grid_x"] == -(-h * h // 64) and p["grid_y"] == 8 and p["grid_z"] == n
        assert p["rx"] == p["ry"] == h + 2 * (hk - 1) and p["content"] == 1 and p["position"] == 1
        assert p["threads"] == (64 if fmt == "fp32" else 128) and p["smem_bytes"] <= 227 * 1024
        s = _lib.gen_attention_plan_for(fmt, n, 1, 1, c, 8, 2, position=False, Hk=hk, Wk=hk, ld_q=c, ld_kv=2 * c)  # '0010'
        assert s["grid_x"] == 1 and s["position"] == 0 and s["rx"] == 0


@pytest.mark.parametrize("kw", [dict(C=256, heads=2), dict(C=192, heads=8), dict(kv_stride=3), dict(Hk=31),
                                dict(ld_q=260), dict(ld_kv=128), dict(H=4000, W=4000)])
def test_planner_refusals(kw):
    args = dict(N=2, H=64, W=64, C=256, heads=8, kv_stride=2)
    args.update({k: kw[k] for k in ("C", "heads", "kv_stride", "H", "W") if k in kw})
    extra = {k: kw[k] for k in ("Hk", "ld_q", "ld_kv") if k in kw}
    with pytest.raises(_lib.OrpError):
        _lib.gen_attention_plan_for("f16x3", args["N"], args["H"], args["W"], args["C"], args["heads"], args["kv_stride"], **extra)


def test_header_symbols_bound_with_arity():
    with open(os.path.join(ROOT, "include", "orp_b200_attention.h")) as f:
        src = f.read()
    decl = dict(re.findall(r"^int (orp_\w+)\(([^;]*)\);", src, re.M | re.S))
    assert set(decl) == set(_lib.ATTENTION_SIGNATURES)
    for name, args in decl.items():
        assert len(args.split(",")) == len(_lib.ATTENTION_SIGNATURES[name][1]), name
        lib = _lib.lib()
        assert isinstance(getattr(lib, name), ctypes._CFuncPtr)
    for other in ("orp_b200.h", "orp_b200_dcnv2.h", "orp_b200_swin.h", "orp_b200_group.h", "orp_b200_hrnet.h"):
        with open(os.path.join(ROOT, "include", other)) as f:
            text = f.read()
        assert not any(name in text for name in decl), other
    assert len(_lib.GenAttentionArgs._fields_) == 17 and len(_lib.GenAttentionPlan._fields_) == 11
