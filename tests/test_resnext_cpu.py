"""CPU: the ResNeXt backbones (resnext.py) - parameter trees built from config dicts, their random draws, the refusals, the fp64
test graph against the reference's own module, the dry-run plans of every grouped tensor-core launch, and the bindings of
include/orp_b200_group.h."""
import os
import re

import numpy as np
import pytest
import torch

from orientedreppoints_b200 import _lib
from orientedreppoints_b200.models import build_backbone, build_detector
from orientedreppoints_b200.weights import STAGE_BLOCKS, block_width, random_state_dict
import resnext_ref as xr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg(depth, groups, base_width, **kw):
    return dict(type='ResNeXt', depth=depth, groups=groups, base_width=base_width, num_stages=4, out_indices=(0, 1, 2, 3),
                frozen_stages=1, norm_cfg=dict(type='BN', requires_grad=True), style='pytorch', **kw)


def _backbone_sd(sd):
    return {k[len("backbone."):]: v for k, v in sd.items() if k.startswith("backbone.")}


@pytest.mark.parametrize("depth,groups,base_width", [(d, g, b) for d in (50, 101, 152) for g, b in ((32, 4), (64, 4), (32, 8))] +
                         [(152, 1, 4)])
def test_config_built_tree_matches_random_state_dict(depth, groups, base_width):
    m = build_backbone(_cfg(depth, groups, base_width))
    for li, nblk in enumerate(STAGE_BLOCKS[depth]):
        layer = getattr(m, "layer%d" % (li + 1))
        assert len(layer) == nblk
        width = block_width(64 << li, groups, base_width)
        if groups > 1:
            assert width == (64 << li) * base_width * groups // 64
        for blk in layer:
            assert blk.conv1.out_channels == width and blk.conv2.groups == groups
            assert tuple(blk.conv2.weight.shape) == (width, width // groups, 3, 3)
            assert blk.conv3.in_channels == width and blk.conv3.out_channels == (256 << li)
    ref = _backbone_sd(random_state_dict(depth, seed=3, groups=groups, base_width=base_width))
    got = [k for k in m.state_dict() if not k.endswith("num_batches_tracked")]       # filled in by BatchNorm on load
    assert sorted(got) == sorted(ref)
    m.load_state_dict(ref, strict=True)
    for k in got:
        assert torch.equal(m.state_dict()[k], ref[k]), k


def test_groups_1_draws_are_the_resnet_draws():
    for depth in (50, 101):
        a, b = random_state_dict(depth, seed=5), random_state_dict(depth, seed=5, groups=1, base_width=8)
        assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    x = build_backbone(_cfg(50, 1, 4, dcn=dict(type='DCN'), stage_with_dcn=(False, True, True, True)))
    r = build_backbone(dict(type='ResNet', depth=50, dcn=dict(type='DCN'), stage_with_dcn=(False, True, True, True)))
    assert x.dcn_layout() == r.dcn_layout()
    assert {k: tuple(v.shape) for k, v in x.state_dict().items()} == {k: tuple(v.shape) for k, v in r.state_dict().items()}


def test_grouped_conv2_kaiming_fan_out():
    """kaiming_init fan_out = weight.shape[0] * 9 for the grouped conv2, as for any nn.Conv2d"""
    sd = random_state_dict(101, seed=1, groups=64, base_width=4)
    w = sd["backbone.layer3.5.conv2.weight"]
    assert tuple(w.shape) == (1024, 16, 3, 3)
    assert abs(float(w.std()) / (2.0 / (1024 * 9)) ** 0.5 - 1) < 0.02


def test_refusals():
    with pytest.raises(NotImplementedError, match="dcn"):
        build_backbone(_cfg(50, 32, 4, dcn=dict(type='DCN'), stage_with_dcn=(False, True, True, True)))
    with pytest.raises(NotImplementedError, match="dcn"):
        random_state_dict(50, groups=32, dcn=dict(type='DCN'), stage_with_dcn=(False, True, True, True))
    with pytest.raises(NotImplementedError, match="group widths"):
        build_backbone(_cfg(50, 32, 2))                       # width 2 * 32 = 64, but 2 channels per group
    with pytest.raises(NotImplementedError, match="multiple of 64"):
        build_backbone(_cfg(50, 12, 4))                       # width 48
    with pytest.raises(NotImplementedError, match="group widths"):
        random_state_dict(50, groups=2, base_width=64)       # layer4: 512 channels per group
    with pytest.raises(KeyError):
        build_backbone(_cfg(34, 32, 4))


def test_engine_refuses_state_dicts_that_contradict_the_model():
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    sd = random_state_dict(50, seed=0, groups=32, base_width=4)
    bad = dict(sd)
    bad["backbone.layer2.1.conv2.weight"] = torch.zeros(256, 4, 3, 3)        # 64 groups where the others have 32
    with pytest.raises(ValueError, match="groups"):
        OrientedRepPointsDetector(bad, 50, "cpu", "fp32")
    bad = dict(sd)
    p = "backbone.layer3.0."                                                   # stage 3 keeps stage 2's width and group width
    bad[p + "conv1.weight"], bad[p + "conv2.weight"] = torch.zeros(256, 512, 1, 1), torch.zeros(256, 8, 3, 3)
    bad[p + "conv3.weight"] = torch.zeros(1024, 256, 1, 1)
    with pytest.raises(ValueError, match="base_width"):
        OrientedRepPointsDetector(bad, 50, "cpu", "fp32")
    bad = dict(sd)
    bad["backbone.layer1.2.conv3.weight"] = torch.zeros(256, 64, 1, 1)       # conv3 not width wide
    with pytest.raises(ValueError, match="bottleneck"):
        OrientedRepPointsDetector(bad, 50, "cpu", "fp32")
    with pytest.raises(ValueError, match="depth"):
        OrientedRepPointsDetector(sd, 34, "cpu", "fp32")
    with pytest.raises(NotImplementedError, match="group"):
        OrientedRepPointsDetector(random_state_dict(50, groups=8, base_width=16), 50, "cpu", "fp32")   # 256 per group at layer4
    from orientedreppoints_b200.weights import dcn_layout
    with pytest.raises(NotImplementedError, match="grouped deformable"):
        OrientedRepPointsDetector(sd, 50, "cpu", "fp32", dcn=dcn_layout(50, dict(type='DCN'), (False, True, True, True)))


def test_detector_config_builds_resnext():
    from orientedreppoints_b200.apis import Config
    cfg = Config.fromfile(os.path.join(ROOT, "configs", "dota", "orientedrepoints_r50_demo.py"))
    cfg['model']['backbone'] = dict(type='ResNeXt', depth=101, groups=64, base_width=4, num_stages=4, out_indices=(0, 1, 2, 3),
                                    frozen_stages=1, norm_cfg=dict(type='BN', requires_grad=True), style='pytorch')
    model = build_detector(cfg['model'], test_cfg=cfg.get('test_cfg'))
    assert model.backbone.layer3[0].conv2.groups == 64
    ref = random_state_dict(101, seed=0, groups=64, base_width=4, num_classes=model.bbox_head.num_classes)
    for k, v in model.state_dict().items():
        if not k.endswith("num_batches_tracked"):
            assert torch.equal(v, ref[k]), k


@pytest.mark.parametrize("tag", ["x50_32x4d", "x101_64x4d", "x50_32x8d"])
def test_fp64_graph_matches_reference_module(tag):
    """tests/resnext_ref.py's fp64 backbone against the reference's own resnext.py (tests/golden/gen_golden_resnext.py)"""
    z = np.load(os.path.join(ROOT, "tests", "golden", "resnext_ref.npz"))
    depth, groups, base_width, seed, gain10, h, w = [int(v) for v in z[tag + "_meta"]]
    sd = random_state_dict(depth, seed=seed, reference_init=False, residual_gain=gain10 / 10, groups=groups, base_width=base_width)
    sdd = {k: v.double() for k, v in sd.items()}
    with torch.no_grad():
        outs = xr.backbone(sdd, torch.from_numpy(z[tag + "_img"]), depth, groups)
    for l, o in enumerate(outs):
        ref = z["%s_c%d" % (tag, l + 2)]
        assert o.shape == ref.shape
        assert np.abs(o.numpy() - ref).max() <= 1e-6 * max(1.0, float(np.abs(ref).max())), (tag, l)


PLAN_CASES = [(name, width, groups, h, stride, n, tile, split)
              for name, depth, groups, bw in xr.MODELS
              for (width, groups_, h, stride) in xr.group_launches(groups, bw)
              for n, tile in xr.BATCHES for split in (False, True)]


def test_plan_cases_cover_every_published_width():
    gws = {w // g for _, w, g, *_ in PLAN_CASES}
    assert gws == {4, 8, 16, 32, 64}


@pytest.mark.parametrize("name,width,groups,h,stride,n,tile,split", PLAN_CASES)
def test_group_plan(name, width, groups, h, stride, n, tile, split):
    h = h * tile // 1024
    p = _lib.tc_plan_group_for([(n, h, h)], width, groups, stride, split=split)
    ho = (h - 1) // stride + 1
    assert p["BN"] == 64 and p["n_tiles_n"] == width // 64 and p["Cout"] == width == p["Cout_padded"]
    assert p["ncat"] == 0 and p["res_mma"] == 0 and p["gn_fused"] == 0 and p["ksplit"] == 1 and p["deform"] == 0
    assert p["tma_epi"] == 1 and p["relu"] == 1 and p["bias"] == 1 and p["split"] == int(split)
    assert p["BW"][0] * p["BH"][0] * p["BI"][0] == 128
    mt = -(-ho // p["BW"][0]) * -(-ho // p["BH"][0]) * -(-n // p["BI"][0])
    assert p["num_tiles"] == mt * (width // 64)
    assert p["grid"] == min(132, p["num_tiles"]) - (min(132, p["num_tiles"]) % (width // 64) if p["b_resident"] else 0)
    # dynamic shared memory of the plan (dense_tc.cu: dyn_smem_bytes) beside the 4 KiB static budget, within the 227 KiB opt-in
    slab = 9 * (2 if split else 1) * 64 * 64 * 2
    stage = 16384 if p["b_resident"] else 16384 + 8192
    staging = p["epi_bufs"] * (32768 if p["epi_merge"] else 16384)
    smem = 1024 + 128 * 68 * 4 + p["stages"] * stage + (slab if p["b_resident"] else 0) + staging
    assert 2 <= p["stages"] <= 6 and smem + 4096 <= 227 * 1024, (p, smem)
    assert p["b_resident"] == (0 if split else int(p["grid"] >= width // 64))


def test_group_plan_refusals():
    ok = [(1, 64, 64)]
    _lib.tc_plan_group_for(ok, 256, 32, 1)
    for kw, match in ((dict(residual=1), "no residual"), (dict(residual=2), "no residual"), (dict(out_f32=True), "fp32 output"),
                      (dict(gn=True), "GroupNorm"), (dict(relu=2), "ReLU|16-bit")):
        with pytest.raises(_lib.OrpError, match=match if match != "ReLU|16-bit" else "16-bit"):
            _lib.tc_plan_group_for(ok, 256, 32, 1, **kw)
    with pytest.raises(_lib.OrpError, match="one 3x3"):
        _lib.tc_plan_group_for(ok * 2, 256, 32, 1)                       # several problems
    for width, groups in ((256, 128), (256, 2), (256, 3), (256, 0)):      # gw 2, 128, not dividing, no groups
        with pytest.raises(_lib.OrpError, match="group width"):
            _lib.tc_plan_group_for(ok, width, groups, 1)
    with pytest.raises(_lib.OrpError, match="multiple of 64"):
        _lib.tc_plan_group_for(ok, 96, 6, 1)                              # gw 16, width 96
    with pytest.raises(_lib.OrpError, match="bad arguments"):
        _lib.tc_plan_group_for(ok, 256, 32, 1, sms=0)


def _decls(header):
    src = open(os.path.join(ROOT, "include", header)).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return dict(re.findall(r"\b(orp_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", src))


def test_group_header_bindings_and_arity():
    decls = _decls("orp_b200_group.h")
    assert sorted(decls) == sorted(_lib.GROUP_SIGNATURES) == sorted(
        ["orp_group_conv2d_bf16", "orp_group_conv2d_f16x3", "orp_group_conv2d_f32", "orp_tc_plan_group_conv"])
    l = _lib.lib()
    for name, params in decls.items():
        assert hasattr(l, name), name
        assert len(_lib.GROUP_SIGNATURES[name][1]) == params.count(",") + 1, name
    assert not set(decls) & set(_decls("orp_b200.h"))
