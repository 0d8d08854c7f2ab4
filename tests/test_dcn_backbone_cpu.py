"""CPU: ResNet backbones with deformable stages (dcn / stage_with_dcn, mmdet/models/backbones/resnet.py:97-168, 365-424,
474-484): the parameter tree a config builds, the reference's initialisation, the shared-dict `fallback_on_stride` quirk,
the errors, the launch plans of the deformable backbone convolutions, and self-checks of the fp64 DCN graph
(tests/dcn_backbone_ref.py).  No kernel runs here."""
import importlib.util
import os

import pytest
import torch
import torch.nn as nn
from torch.nn.modules.utils import _pair

from dcn_backbone_ref import BATCHES, LAUNCHES_1024

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C3_C5 = (False, True, True, True)


def _cfg(depth):
    spec = importlib.util.spec_from_file_location("c%d" % depth, os.path.join(ROOT, "configs", "dota", "orientedrepoints_r%d_demo.py" % depth))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _build(depth, dcn, stages, **backbone):
    from orientedreppoints_b200.models import build_detector
    cfg = _cfg(depth)
    model = dict(cfg.model, pretrained=None, backbone=dict(cfg.model["backbone"], dcn=dcn, stage_with_dcn=stages, **backbone))
    return build_detector(model, test_cfg=cfg.test_cfg)


@pytest.mark.parametrize("depth,kind,stages", [
    (50, 'DCN', C3_C5), (50, 'DCNv2', C3_C5), (50, 'DCN', (True, False, False, True)), (50, 'DCNv2', (False, False, True, False)),
    (50, 'DCNv2', (True, True, True, True)), (101, 'DCN', C3_C5), (101, 'DCNv2', (False, False, True, True)),
])
def test_config_builds_the_deformable_tree(depth, kind, stages):
    from orientedreppoints_b200.ops import DeformConvPack, ModulatedDeformConvPack
    from orientedreppoints_b200.weights import STAGE_BLOCKS, dcn_layout, random_state_dict
    dcn = dict(type=kind, deformable_groups=1, fallback_on_stride=False)
    det = _build(depth, dcn, stages)
    cls = DeformConvPack if kind == 'DCN' else ModulatedDeformConvPack
    co = 18 if kind == 'DCN' else 27
    for li, nblk in enumerate(STAGE_BLOCKS[depth]):
        planes = 64 << li
        for b in range(nblk):
            c2 = getattr(det.backbone, "layer%d" % (li + 1))[b].conv2
            stride = 2 if (b == 0 and li > 0) else 1
            if stages[li]:
                assert type(c2) is cls and _pair(c2.stride) == (stride, stride) and _pair(c2.padding) == (1, 1)
                assert tuple(c2.weight.shape) == (planes, planes, 3, 3) and getattr(c2, "bias", None) is None
                assert tuple(c2.conv_offset.weight.shape) == (co, planes, 3, 3) and tuple(c2.conv_offset.bias.shape) == (co,)
                assert c2.conv_offset.stride == (stride, stride) and c2.conv_offset.padding == (1, 1)
            else:
                assert type(c2) is nn.Conv2d and c2.stride == (stride, stride)
    assert det.backbone.dcn_layout() == dcn_layout(depth, dict(type=kind, fallback_on_stride=False), stages)
    sd = {k: v for k, v in det.state_dict().items() if not k.endswith("num_batches_tracked")}
    ref = random_state_dict(depth, seed=0, reference_init=True, num_classes=16, dcn=dict(type=kind, fallback_on_stride=False),
                            stage_with_dcn=stages)
    assert sorted(sd) == sorted(ref)
    for k in ref:
        assert torch.equal(sd[k], ref[k]), k
    # the reference's init (resnet.py:474-484): DeformConv.reset_parameters' uniform bound, conv_offset all zero
    c2 = det.backbone.layer4[1].conv2 if stages[3] else det.backbone.layer3[1].conv2
    bound = 1.0 / (9 * c2.weight.shape[0]) ** 0.5
    wmax = float(c2.weight.detach().abs().max())
    assert 0.9 * bound < wmax <= bound
    assert float(c2.conv_offset.weight.abs().sum()) == 0 and float(c2.conv_offset.bias.abs().sum()) == 0


def test_plain_backbone_state_dict_unchanged():
    """no dcn: the same draws as before the deformable options existed (the goldens of the plain graph depend on them)"""
    from orientedreppoints_b200.weights import random_state_dict
    a = random_state_dict(50, seed=3, reference_init=False)
    b = random_state_dict(50, seed=3, reference_init=False, dcn=None, stage_with_dcn=C3_C5, dcn_offset_scale=1.0)
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    assert not any("conv_offset" in k for k in a)


def test_fallback_on_stride_pops_the_shared_dict():
    """resnet.py:146-147: every block pops fallback_on_stride from the ONE dict ResNet hands them, so with True only the
    first block built from it (layer2.0 for c3-c5) gets a plain conv"""
    from orientedreppoints_b200.ops import DeformConvPack
    from orientedreppoints_b200.weights import dcn_layout, random_state_dict
    dcn = dict(type='DCN', deformable_groups=1, fallback_on_stride=True)
    det = _build(50, dcn, C3_C5)
    assert 'fallback_on_stride' not in dcn                                  # popped from the caller's dict, as the reference does
    plain = [(li, b) for li, stage in enumerate(det.backbone.dcn_layout()) for b, k in enumerate(stage) if k is None and li > 0]
    assert plain == [(1, 0)]
    assert type(det.backbone.layer2[0].conv2) is nn.Conv2d and type(det.backbone.layer3[0].conv2) is DeformConvPack
    want = dcn_layout(50, dict(type='DCN', fallback_on_stride=True), C3_C5)
    assert det.backbone.dcn_layout() == want
    ref = random_state_dict(50, dcn=dict(type='DCN', fallback_on_stride=True), stage_with_dcn=C3_C5)
    assert sorted(k for k in det.state_dict() if not k.endswith("num_batches_tracked")) == sorted(ref)
    assert "backbone.layer2.0.conv2.conv_offset.weight" not in ref and "backbone.layer2.1.conv2.conv_offset.weight" in ref


def test_errors():
    with pytest.raises(NotImplementedError, match="deformable_groups"):
        _build(50, dict(type='DCN', deformable_groups=2), C3_C5)
    with pytest.raises(AssertionError, match="conv_cfg"):
        _build(50, dict(type='DCN'), C3_C5, conv_cfg=dict(type='Conv'))
    with pytest.raises(KeyError):
        _build(50, dict(type='DCNv3'), C3_C5)
    with pytest.raises(NotImplementedError):
        _build(50, None, C3_C5, gcb=dict(ratio=1. / 4.))


def test_engine_refuses_a_layout_that_does_not_match_the_weights():
    """the engine takes the deformable layers from the built module and checks them against the state dict"""
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    from orientedreppoints_b200.weights import dcn_layout, random_state_dict
    sd = random_state_dict(50, dcn=dict(type='DCN'), stage_with_dcn=C3_C5)
    v2 = dcn_layout(50, dict(type='DCNv2'), C3_C5)
    with pytest.raises(ValueError, match="DCNv2"):
        OrientedRepPointsDetector(sd, 50, "cpu", "fp32", dcn=v2)
    with pytest.raises(ValueError, match="conv_offset but dcn names a plain"):
        OrientedRepPointsDetector(sd, 50, "cpu", "fp32")
    with pytest.raises(ValueError, match="blocks of R-50"):
        OrientedRepPointsDetector(sd, 50, "cpu", "fp32", dcn=v2[:3])


def test_offset_mask_binding_matches_header():
    """the DCNv2 header's entry point is exported and bound with its declared arity"""
    import os
    import re
    from orientedreppoints_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(root, "include", "orp_b200_dcnv2.h")).read(), flags=re.S)
    decls = dict(re.findall(r"\b(orp_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", src))
    assert sorted(decls) == sorted(_lib.DCNV2_SIGNATURES)
    for name, params in decls.items():
        assert hasattr(_lib.lib(), name) and len(_lib.DCNV2_SIGNATURES[name][1]) == params.count(",") + 1


def _backbone_plans(split, n, tile):
    from orientedreppoints_b200 import _lib
    from orientedreppoints_b200.engine_tc import EngineTCSplit
    plans = []
    for planes, h, s in LAUNCHES_1024:
        h = h * tile // 1024
        cout_p = EngineTCSplit._pad_cout(planes) if split else (planes + 31) // 32 * 32
        dcn = _lib.tc_plan_for([(n, h, h)], planes, cout_p, 3, 3, planes, s, 1, bias=True, relu=1, deform=True, split=split)
        off = [_lib.tc_plan_for([(n, h, h)], co, 32, 3, 3, planes, s, 1, bias=True, out_f32=True, split=split) for co in (18, 27)]
        plans.append(((planes, h, s), dcn, off))
    return plans


@pytest.mark.parametrize("split", [1, 0], ids=["f16x3", "bf16"])
@pytest.mark.parametrize("n,tile", BATCHES)
def test_planner_takes_every_backbone_launch(split, n, tile):
    """every deformable conv2 of the backbone and its offset convolution plan (stride 2, Cin = Cout = 64..512, bias + ReLU,
    16-bit output); in f16x3, 256 and 512 channels run as N-tile pairs (every sample gathered once per M tile)"""
    for (planes, h, s), p, offs in _backbone_plans(split, n, tile):
        ho = (h + 2 - 3) // s + 1
        assert p["deform"] == 1 and p["bias"] == 1 and p["relu"] == 1 and p["out_f32"] == 0 and p["tma_epi"] == 1
        assert p["BW"][0] * p["BH"][0] * p["BI"][0] == 128 and p["BW"][0] * s <= 256
        assert p["num_tiles"] >= -(-n * ho * ho // 128) * p["n_tiles_n"]
        if split:
            assert p["dcat"] == 1 and p["n_pair"] == (2 if planes >= 256 and p["BN"] == 128 else 1)
        for o in offs:
            assert o["out_f32"] == 1 and o["deform"] == 0 and o["BN"] == 32


def test_fp64_dcn_graph_self_checks():
    """the fp64 DCN backbone: with all-zero offsets DCN is the plain backbone (to fp64 rounding: im2col GEMM against
    conv2d); with mask logits at +inf (mask 1) DCNv2 is bit for bit DCN with the same offsets"""
    from dcn_backbone_ref import backbone
    from oracle import torch_reference as tr
    from orientedreppoints_b200.weights import dcn_layout, random_state_dict
    img = torch.randn(1, 3, 64, 96, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    sd = {k: v.double() for k, v in random_state_dict(50, seed=2, reference_init=False, dcn=dict(type='DCN'),
                                                      stage_with_dcn=C3_C5).items()}
    with torch.no_grad():
        plain = tr.backbone(sd, img)
        dcn = backbone(sd, img, dcn_layout(50, dict(type='DCN'), C3_C5))
        for a, b in zip(dcn, plain):
            assert float((a - b).abs().max()) <= 1e-12 * float(b.abs().max())
        sd2 = {k: v.double() for k, v in random_state_dict(50, seed=2, reference_init=False, dcn=dict(type='DCNv2'),
                                                           stage_with_dcn=C3_C5, dcn_offset_scale=1.0).items()}
        sd1 = dict(sd2)
        for k in [k for k in sd2 if k.endswith("conv_offset.weight")]:
            b = k[:-len("weight")] + "bias"
            sd1[k], sd1[b] = sd2[k][:18], sd2[b][:18]
            sd2[b] = sd2[b].clone()
            sd2[b][18:] = float("inf")
        v1 = backbone(sd1, img, dcn_layout(50, dict(type='DCN'), C3_C5))
        v2 = backbone(sd2, img, dcn_layout(50, dict(type='DCNv2'), C3_C5))
        for a, b, p in zip(v2, v1, plain):
            assert torch.equal(a, b)
        assert any(float((a - p).abs().max()) > 1e-3 * float(p.abs().max()) for a, p in zip(v1[1:], plain[1:]))
