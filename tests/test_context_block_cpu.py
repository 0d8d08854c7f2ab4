"""Global context blocks in ResNet / ResNeXt backbones, without a GPU: the fp64 restatement (tests/context_block_ref.py) against
the reference's own ContextBlock / ResNet / ResNeXt (tests/golden/context_block_ref.npz), the config-built parameter trees
against the reference's, the reference's initialisation, unchanged draws without context blocks, the errors and the one kept
refusal, the engine's layout check, the pool planner and the header bindings."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

from orientedreppoints_b200 import _lib
from orientedreppoints_b200.models import build_backbone, build_detector
from orientedreppoints_b200.weights import STAGE_BLOCKS, gcb_keys, gcb_layout, gcb_spec, random_state_dict
import context_block_ref as cr

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = np.load(os.path.join(HERE, "golden", "context_block_ref.npz"))
POOLS = ("att", "avg")
FUSIONS = (("channel_add",), ("channel_mul",), ("channel_add", "channel_mul"))
C3_C5 = (False, True, True, True)
GA_CFG = dict(spatial_range=-1, num_heads=8, kv_stride=2, attention_type='1111')
GA_STAGES = [[], [], [0, 1, 2, 3, 4, 5], [0, 1, 2]]
# conv3 + bn3 without the residual and the ReLU (the input of a context block) reaches one plan signature no case of
# tests/conv_plan_cases.PARITY pins: R-50-GCB's layer2 c3 in bf16 at 16 x 1024^2.  Its case, in PARITY's format
GCB_PARITY = [
    # r50-gcb bf16 layer2.0.c3, layer2.1.c3, layer2.2.c3, layer2.3.c3
    (('bf16', 0, 'bf16', 256, 1, 0, 0, 0, 1, 0, 2, 0, 5, 0, 1, 0, 0, 1, 0, 0), 'bf16', 'conv', 128, 512, 1, 1, 1, 0, 0, 0, 0, [(2, 67, 67)]),
]
# the golden backbones: tag -> (gcb, dcn type or None, gen_attention)
BACKBONES = {"r50_r16": (dict(ratio=1. / 16.), None, False),
             "r50_avg_r4": (dict(ratio=1. / 4., pooling_type='avg', fusion_types=('channel_add', 'channel_mul')), None, False),
             "x50_32x4d_r16": (dict(ratio=1. / 16.), None, False),
             "r50_dcnv2_r16": (dict(ratio=1. / 16.), 'DCNv2', False),
             "r50_ga_r16": (dict(ratio=1. / 16.), None, True)}


def _keys(tag):
    return {k.split(":")[0]: tuple(int(d) for d in k.split(":")[1].split("x")) for k in GOLD[tag + "_keys"]}


def backbone_case(tag):
    """(state dict, gcb layout, depth, groups, dcn layout, attention layout) of a golden backbone, drawn as the generator draws
    it (gcb_gain 1, residual_gain 0.5)"""
    from orientedreppoints_b200.weights import dcn_layout, gen_attention_layout
    gcb, dcn, ga = BACKBONES[tag]
    depth, groups, bw, seed = [int(v) for v in GOLD[tag + "_meta"][:4]]
    extra = dict(dcn=dict(type=dcn), stage_with_dcn=C3_C5, dcn_offset_scale=0.5) if dcn else {}
    if ga:
        extra.update(gen_attention=GA_CFG, stage_with_gen_attention=GA_STAGES, gen_attention_gamma=0.7)
    sd = random_state_dict(depth, seed=seed, reference_init=False, residual_gain=0.5, groups=groups, base_width=bw, gcb=gcb,
                           stage_with_gcb=C3_C5, gcb_gain=1.0, **extra)
    return (sd, gcb_layout(depth, gcb, C3_C5), depth, groups, dcn_layout(50, dict(type=dcn), C3_C5) if dcn else None,
            gen_attention_layout(50, GA_CFG, GA_STAGES) if ga else None)


@pytest.mark.parametrize("tag", sorted(k[:-5] for k in GOLD.files if k.endswith("_meta") and k[:3] in ("att", "avg")))
def test_block_restatement_vs_reference(tag):
    pool, fus, r, c, h, w, seed = [int(v) for v in GOLD[tag + "_meta"]]
    cfg = dict(ratio=1. / r, pooling_type=POOLS[pool], fusion_types=FUSIONS[fus])
    li = (256, 512, 1024, 2048).index(c)
    stages = [False] * 4
    stages[li] = True
    sd = random_state_dict(50, seed=seed, reference_init=False, gcb=cfg, stage_with_gcb=stages, gcb_gain=1.0)
    p = {k: v.double() for k, v in cr.block_params(sd, "backbone.layer%d.0" % (li + 1)).items()}
    assert {k: tuple(v.shape) for k, v in p.items()} == _keys(tag) == gcb_keys(gcb_spec(cfg, c))
    x = torch.randn(2, c, h, w, generator=torch.Generator().manual_seed(seed + 100), dtype=torch.float64)
    y = cr.block(gcb_spec(cfg, c), p, x)[:, :32]
    ref = torch.from_numpy(GOLD[tag + "_y"]).double()
    assert (y - x[:, :32]).abs().max() > 0.1                            # the block acts
    assert torch.allclose(y, ref, rtol=1e-6, atol=1e-6), float((y - ref).abs().max())


@pytest.mark.parametrize("tag", sorted(BACKBONES))
def test_backbone_restatement_vs_reference(tag):
    sd, lay, depth, groups, dl, gal = backbone_case(tag)
    h, w = [int(v) for v in GOLD[tag + "_meta"][4:]]
    seed = int(GOLD[tag + "_meta"][3])
    sd = {k: v.double() for k, v in sd.items()}
    img = torch.randn(1, 3, h, w, generator=torch.Generator().manual_seed(seed + 10), dtype=torch.float64)
    feats = cr.backbone(sd, img, lay, depth, groups, dl, gal)
    for l in (1, 2, 3):
        ref = torch.from_numpy(GOLD["%s_c%d" % (tag, l + 2)]).double()
        got = feats[l][:, :ref.shape[1]]
        assert got.shape == ref.shape
        assert torch.allclose(got, ref, rtol=1e-5, atol=1e-5 * float(ref.abs().max())), (l, float((got - ref).abs().max()))


def _detector_cfg(gcb, stages=C3_C5, backbone_type='ResNet', **extra):
    bb = dict(type=backbone_type, depth=50, num_stages=4, out_indices=(0, 1, 2, 3), frozen_stages=1, style='pytorch', gcb=gcb,
              stage_with_gcb=stages, **extra)
    return dict(type='OrientedRepPointsDetector', backbone=bb,
                neck=dict(type='FPN', in_channels=[256, 512, 1024, 2048], out_channels=256, start_level=1, add_extra_convs=True,
                          num_outs=5, norm_cfg=dict(type='GN', num_groups=32, requires_grad=True)),
                bbox_head=dict(type='OrientedRepPointsHead', num_classes=16, in_channels=256, feat_channels=256,
                               point_feat_channels=256, stacked_convs=3, num_points=9, gradient_mul=0.3, point_strides=[8, 16, 32, 64, 128],
                               point_base_scale=2, norm_cfg=dict(type='GN', num_groups=32, requires_grad=True)))


@pytest.mark.parametrize("pool", POOLS)
@pytest.mark.parametrize("fus", FUSIONS)
@pytest.mark.parametrize("backbone_type, extra", [("ResNet", {}), ("ResNeXt", dict(groups=32, base_width=4))])
def test_config_tree_keys_and_init(pool, fus, backbone_type, extra):
    gcb = dict(ratio=1. / 16., pooling_type=pool, fusion_types=list(fus))
    m = build_detector(_detector_cfg(gcb, backbone_type=backbone_type, **extra))
    sd = m.state_dict()
    got = {k: tuple(v.shape) for k, v in sd.items() if ".context_block." in k}
    want = {}
    for li in (1, 2, 3):
        spec = gcb_spec(gcb, 256 << li)
        for b in range(STAGE_BLOCKS[50][li]):
            want.update({"backbone.layer%d.%d.context_block.%s" % (li + 1, b, k): s for k, s in gcb_keys(spec).items()})
    assert got == want
    # the reference's tree for each combination: the golden block keys of the same pooling and fusions
    tag = next(k[:-5] for k in GOLD.files if k.endswith("_meta") and k[:3] == pool and
               tuple(GOLD[k][:2]) == (POOLS.index(pool), FUSIONS.index(fus)))
    ref = {k for k in _keys(tag)}
    assert {k.split(".context_block.")[1] for k in got} == ref
    # the reference's init: every conv kaiming fan_out (conv_mask and the last conv included) with zero bias, LayerNorm 1 / 0
    for k in got:
        v = sd[k]
        if k.endswith(".1.weight"):
            assert torch.equal(v, torch.ones_like(v))
        elif k.endswith("bias"):
            assert torch.count_nonzero(v) == 0
        elif v.shape[0] > 1 and v.numel() > 1000:
            assert abs(float(v.std()) - math.sqrt(2.0 / v.shape[0])) < 0.1 * math.sqrt(2.0 / v.shape[0]), k
        else:                                                           # conv_mask [1, C, 1, 1]: fan_out 1, std sqrt(2)
            assert abs(float(v.std()) - math.sqrt(2.0 / v.shape[0])) < 0.15 * math.sqrt(2.0), k
    assert m.backbone.gcb_layout() == gcb_layout(50, gcb, C3_C5)
    if backbone_type == "ResNeXt":
        assert tuple(sd["backbone.layer2.0.conv2.weight"].shape) == (256, 8, 3, 3)


@pytest.mark.parametrize("tag", sorted(BACKBONES))
def test_backbone_keys_equal_the_reference(tag):
    gcb, dcn, ga = BACKBONES[tag]
    depth, groups, bw = [int(v) for v in GOLD[tag + "_meta"][:3]]
    extra = {}
    if groups > 1:
        extra = dict(groups=groups, base_width=bw)
    if dcn:
        extra.update(dcn=dict(type=dcn, deformable_groups=1, fallback_on_stride=False), stage_with_dcn=C3_C5)
    if ga:
        extra.update(gen_attention=GA_CFG, stage_with_gen_attention=GA_STAGES)
    bb = build_backbone(dict(type='ResNeXt' if groups > 1 else 'ResNet', depth=depth, gcb=gcb, stage_with_gcb=C3_C5, **extra))
    got = {k: tuple(v.shape) for k, v in bb.state_dict().items() if not k.endswith("num_batches_tracked")}
    assert got == _keys(tag)
    sd = backbone_case(tag)[0]
    assert {k[len("backbone."):]: tuple(v.shape) for k, v in sd.items() if k.startswith("backbone.")} == _keys(tag)


def test_reference_init_block_is_identity_relu():
    """zero_init_residual zeroes bn3, so x = 0, the context is 0 and add = the zero conv bias: the block gives relu(identity)"""
    sd = random_state_dict(50, gcb=dict(ratio=1. / 16.), stage_with_gcb=C3_C5)
    p = {k: v.double() for k, v in cr.block_params(sd, "backbone.layer3.0").items()}
    assert float(p['conv_mask.weight'].abs().max()) > 0 and float(p['channel_add_conv.3.weight'].abs().max()) > 0
    x = torch.zeros(1, 1024, 5, 6, dtype=torch.float64)
    assert torch.equal(cr.block(gcb_spec(dict(ratio=1. / 16.), 1024), p, x), x)


def test_draws_without_gcb_unchanged():
    a = random_state_dict(50, seed=3, reference_init=False)
    for extra in (dict(gcb=None), dict(gcb=None, stage_with_gcb=C3_C5), dict(gcb_gain=1.0)):
        b = random_state_dict(50, seed=3, reference_init=False, **extra)
        assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)


def test_gain_makes_every_term_act():
    sd = random_state_dict(50, seed=4, reference_init=False, gcb=dict(ratio=1. / 4., fusion_types=('channel_add', 'channel_mul')),
                           stage_with_gcb=C3_C5, gcb_gain=1.0)
    p = cr.block_params(sd, "backbone.layer2.1")
    for k in ("conv_mask.bias", "channel_add_conv.0.bias", "channel_mul_conv.1.bias", "channel_add_conv.3.bias"):
        assert float(p[k].abs().max()) > 0, k
    assert not torch.equal(p["channel_mul_conv.1.weight"], torch.ones_like(p["channel_mul_conv.1.weight"]))


@pytest.mark.parametrize("gcb, stages, exc, word", [
    (dict(ratio=1. / 16., pooling_type='max'), C3_C5, ValueError, "pooling_type"),
    (dict(ratio=1. / 16., fusion_types=()), C3_C5, ValueError, "fusion_types"),
    (dict(ratio=1. / 16., fusion_types=('channel_concat',)), C3_C5, ValueError, "fusion_types"),
    (dict(ratio=1. / 16., fusion_types='channel_add'), C3_C5, ValueError, "fusion_types"),
    (dict(ratio=1. / 1024.), C3_C5, ValueError, "ratio"),
    (dict(ratio=1. / 16.), (False, True, True), ValueError, "stage_with_gcb"),
    (dict(ratio=1. / 16., no_such=1), C3_C5, TypeError, "no_such"),
    (dict(pooling_type='att'), C3_C5, TypeError, "ratio"),
    (dict(ratio=2.0), C3_C5, NotImplementedError, "planes"),
    (dict(ratio=1. / 16.), (False, False, False, False), NotImplementedError, "no block.*stage_with_gcb"),
])
def test_errors(gcb, stages, exc, word):
    for kind in ('ResNet', 'ResNeXt'):
        with pytest.raises(exc, match=word):
            build_backbone(dict(type=kind, depth=50, gcb=gcb, stage_with_gcb=stages))
    if exc is not NotImplementedError or "planes" in word:
        with pytest.raises(exc, match=word):
            random_state_dict(50, gcb=gcb, stage_with_gcb=stages)


def test_combinations_build():
    """any dcn / gen_attention layout and any groups take a gcb"""
    dcn = dict(type='DCNv2', deformable_groups=1, fallback_on_stride=False)
    bb = build_backbone(dict(type='ResNet', depth=50, gcb=dict(ratio=1. / 16.), stage_with_gcb=C3_C5, dcn=dcn, stage_with_dcn=C3_C5,
                             gen_attention=GA_CFG, stage_with_gen_attention=GA_STAGES))
    assert hasattr(bb.layer3[0], 'context_block') and hasattr(bb.layer3[0], 'gen_attention_block') and bb.dcn_layout()[2][0] == 'DCNv2'
    x = build_backbone(dict(type='ResNeXt', depth=101, groups=64, base_width=4, gcb=dict(ratio=1. / 4.), stage_with_gcb=(True,) * 4))
    assert [sum(sp is not None for sp in s) for s in x.gcb_layout()] == list(STAGE_BLOCKS[101])


def test_engine_checks_layout_against_state_dict():
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    lay = gcb_layout(50, dict(ratio=1. / 16.), C3_C5)
    plain = random_state_dict(50)
    with pytest.raises(ValueError, match="context_block"):
        OrientedRepPointsDetector(plain, 50, "cpu", "fp32", gcb=lay)                # layout names blocks the weights lack
    sd = random_state_dict(50, gcb=dict(ratio=1. / 16.), stage_with_gcb=C3_C5)
    with pytest.raises(ValueError, match="context_block"):
        OrientedRepPointsDetector(sd, 50, "cpu", "fp32")                            # weights hold blocks the layout lacks
    other = gcb_layout(50, dict(ratio=1. / 4.), C3_C5)
    with pytest.raises(ValueError, match="128 planes"):
        OrientedRepPointsDetector(sd, 50, "cpu", "fp32", gcb=other)                 # wrong shapes
    extra = dict(sd, **{"backbone.layer2.0.context_block.channel_mul_conv.3.bias": torch.zeros(512)})
    with pytest.raises(ValueError, match="context_block"):
        OrientedRepPointsDetector(extra, 50, "cpu", "fp32", gcb=lay)                # an extra key
    with pytest.raises(ValueError, match="blocks of R-50"):
        OrientedRepPointsDetector(sd, 50, "cpu", "fp32", gcb=lay[:3])
    with pytest.raises(ValueError, match="ResNet / ResNeXt"):
        OrientedRepPointsDetector({}, "swin_tiny", "cpu", "fp32", gcb=lay)


# every pool launch of a ResNet at N = 1 / 16 on 1024^2 and 960^2 input: (tile, stage) -> map side
@pytest.mark.parametrize("fmt", ["bf16", "f16x3", "fp32"])
@pytest.mark.parametrize("tile", [1024, 960])
@pytest.mark.parametrize("stage", [0, 1, 2, 3])
def test_planner_every_stage(fmt, tile, stage):
    c, h = 256 << stage, tile // (4 << stage)
    for n in (1, 16):
        p = _lib.context_plan_for(fmt, n, h, h, c)
        assert p["grid_y"] == n and p["grid_x"] == p["chunks"] and p["threads"] == 256
        assert p["warps_per_slot"] * p["slots"] * 32 == p["threads"] and p["warps_per_slot"] * 256 >= c
        assert (p["chunks"] - 1) * p["pixels_per_chunk"] < h * h <= p["chunks"] * p["pixels_per_chunk"]     # every chunk holds pixels
        assert p["workspace_bytes"] == n * p["chunks"] * (c + 2) * 4
        assert n * p["chunks"] >= 132                                   # the grid covers the SMs
        assert n * p["chunks"] <= 528 + n
        assert p["pixels_per_chunk"] >= min(h * h, p["slots"] * 4)


@pytest.mark.parametrize("args", [(0, 8, 8, 256), (1, 0, 8, 256), (1, 8, 8, 12), (1, 8, 8, 4096), (70000, 8, 8, 256),
                                  (1, 65536, 65536, 256)])
def test_planner_refusals(args):
    with pytest.raises(_lib.OrpError):
        _lib.context_plan_for("f16x3", *args)
    with pytest.raises(KeyError):
        _lib.context_plan_for("fp16", 1, 8, 8, 256)


def test_gcb_parity_case_plans():
    from conv_plan_cases import PARITY, planned, signature
    for c in GCB_PARITY:
        assert signature(planned(c)) == c[0] and c[0] not in {p[0] for p in PARITY}


def test_header_symbols_bound_with_arity():
    with open(os.path.join(ROOT, "include", "orp_b200_context.h")) as f:
        src = f.read()
    decl = dict(re.findall(r"^int (orp_\w+)\(([^;]*)\);", src, re.M | re.S))
    assert set(decl) == set(_lib.CONTEXT_SIGNATURES)
    lib = _lib.lib()
    for name, args in decl.items():
        assert len(args.split(",")) == len(_lib.CONTEXT_SIGNATURES[name][1]), name
        assert isinstance(getattr(lib, name), ctypes._CFuncPtr)
    for other in ("orp_b200.h", "orp_b200_dcnv2.h", "orp_b200_swin.h", "orp_b200_group.h", "orp_b200_hrnet.h", "orp_b200_attention.h"):
        with open(os.path.join(ROOT, "include", other)) as f:
            text = f.read()
        assert not any(name in text for name in decl), other
        assert "orp_b200_context" not in text
    assert not set(decl) & set(_lib.SIGNATURES)
    assert len(_lib.ContextPlan._fields_) == 8 and len(_lib.ContextMlp._fields_) == 6
