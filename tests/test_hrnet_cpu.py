"""CPU: the HRNet backbones with the HRFPN neck (hrnet.py, hrfpn.py) - parameter trees built from config dicts against the
reference's keys, the fp64 test graph and the engine's rewrites of it against the reference's own modules, the 3x3 stem in
space-to-depth form, the refusals, and the bindings of include/orp_b200_hrnet.h."""
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from orientedreppoints_b200 import _lib
from orientedreppoints_b200.hrnet import ARCHS, HRNetArch
from orientedreppoints_b200.models import build_backbone, build_detector, build_neck
from orientedreppoints_b200.weights import random_hrnet_state_dict
import hrnet_ref as hr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _shapes(m):
    return {k: list(v.shape) for k, v in m.state_dict().items()}


def _r50_cfg():
    from orientedreppoints_b200.apis import Config
    return Config.fromfile(os.path.join(ROOT, "configs", "dota", "orientedrepoints_r50_demo.py"))


def _hr_model_cfg(arch="hrnetv2p_w18", **neck):
    cfg = _r50_cfg()
    a = ARCHS[arch]
    cfg['model']['backbone'] = dict(type='HRNet', extra=a.extra())
    cfg['model']['neck'] = dict(dict(type='HRFPN', in_channels=list(a.out_widths), out_channels=256, stride=2), **neck)
    cfg['model']['pretrained'] = None
    return cfg


def _golden_keys(arch):
    """{"backbone": {key: shape}, "neck": {...}} of the reference's HRNet(arch) and HRFPN(256) (gen_golden_hrnet.py)"""
    z = np.load(os.path.join(GOLDEN, "hrnet_ref.npz"))
    out = {}
    for part in ("backbone", "neck"):
        shapes = [[int(d) for d in s.split(",") if d] for s in str(z["%s_shapes_%s" % (arch, part)]).split(";")]
        out[part] = dict(zip(str(z["keys_" + part]).split("\n"), shapes))
    return out


@pytest.mark.parametrize("arch", sorted(ARCHS))
def test_config_built_tree_has_the_reference_keys(arch):
    ref = _golden_keys(arch)
    a = ARCHS[arch]
    bb = build_backbone(dict(type='HRNet', extra=a.extra()))
    assert _shapes(bb) == ref["backbone"]
    # the reference's quirk: HRFPN's ConvModules never get norm_cfg, so they have a bias and no norm whatever it says
    nk = build_neck(dict(type='HRFPN', in_channels=list(a.out_widths), out_channels=256, stride=2, norm_cfg=dict(type='BN')))
    assert _shapes(nk) == ref["neck"]
    assert not any(".bn" in k or ".gn" in k for k in ref["neck"])
    sd = random_hrnet_state_dict(arch, seed=1)
    assert {k[9:]: list(v.shape) for k, v in sd.items() if k.startswith("backbone.")} == \
        {k: s for k, s in ref["backbone"].items() if not k.endswith("num_batches_tracked")}
    assert {k[5:]: list(v.shape) for k, v in sd.items() if k.startswith("neck.")} == ref["neck"]


def test_detector_config_builds_hrnet_and_loads_reference_keys():
    cfg = _hr_model_cfg("hrnetv2p_w32", pooling_type='MAX')
    model = build_detector(cfg['model'], test_cfg=cfg.get('test_cfg'))
    assert model.backbone.arch is not None and model.neck.pooling_type == 'MAX'
    ref = random_hrnet_state_dict("hrnetv2p_w32", seed=0, num_classes=model.bbox_head.num_classes)
    for k, v in model.state_dict().items():
        if not k.endswith("num_batches_tracked"):
            assert torch.equal(v, ref[k]), k
    model.load_state_dict(random_hrnet_state_dict("hrnetv2p_w32", seed=5, num_classes=model.bbox_head.num_classes,
                                                  reference_init=False), strict=False)


def test_reference_init():
    """kaiming fan_out on the backbone convs, constant-1 norms, caffe2_xavier (uniform +-sqrt(3 / fan_in)) on HRFPN"""
    sd = random_hrnet_state_dict("hrnetv2p_w48", seed=2)
    w = sd["backbone.stage4.0.branches.3.0.conv1.weight"]                     # [384, 384, 3, 3]
    assert abs(float(w.std()) / (2.0 / (384 * 9)) ** 0.5 - 1) < 0.02
    assert torch.equal(sd["backbone.stage3.1.fuse_layers.0.1.1.weight"], torch.ones(48))
    r = sd["neck.reduction_conv.conv.weight"]
    bound = (3.0 / 720) ** 0.5
    assert float(r.abs().max()) <= bound and float(r.abs().max()) > 0.99 * bound
    assert not sd["neck.reduction_conv.conv.bias"].any()
    z = random_hrnet_state_dict("hrnetv2p_w18", zero_init_residual=True)
    assert not z["backbone.stage2.0.branches.0.3.bn2.weight"].any() and not z["backbone.layer1.0.bn3.weight"].any()


def _golden_cases():
    z = np.load(os.path.join(GOLDEN, "hrnet_ref.npz"))
    return sorted({k[:-5] for k in z.files if k.endswith("_meta")})


@pytest.mark.parametrize("form", ["reference", "padded", "engine_order"])
@pytest.mark.parametrize("tag", _golden_cases())
def test_fp64_graph_matches_reference_modules(tag, form):
    """tests/hrnet_ref.py against the reference's own hrnet.py / hrfpn.py (tests/golden/gen_golden_hrnet.py), as written, with
    channel-padded weights, and in the engine's order of sums with HRFPN's reduction before the upsampling"""
    z = np.load(os.path.join(GOLDEN, "hrnet_ref.npz"))
    seed, gain10, h, w = [int(v) for v in z[tag + "_meta"]]
    arch = str(z[tag + "_arch"])
    sd = {k: v.double() for k, v in random_hrnet_state_dict(arch, seed=seed, reference_init=False, residual_gain=gain10 / 10,
                                                             feat=64).items()}
    img = torch.from_numpy(np.random.RandomState(seed + 10).standard_normal((1, 3, h, w)))
    with torch.no_grad():
        xs = hr.backbone(sd, img, arch, padded=form == "padded", engine_order=form == "engine_order")
        for l, x in enumerate(xs):
            ref = z["%s_y%d" % (tag, l)]
            assert x.shape == ref.shape
            assert np.abs(x.numpy() - ref).max() <= 1e-6 * max(1.0, float(np.abs(ref).max())), (l, form)
        for pooling in ("AVG", "MAX"):
            for l, f in enumerate(hr.hrfpn(sd, xs, pooling, engine_order=form == "engine_order")):
                ref = z["%s_%sp%d" % (tag, pooling + "_" if l else "", l)]
                assert f.shape == ref.shape
                assert np.abs(f.numpy() - ref).max() <= 1e-6 * max(1.0, float(np.abs(ref).max())), (pooling, l, form)


@pytest.mark.parametrize("h,w", [(64, 64), (96, 160), (30, 46)])
def test_3x3_stem_in_space_to_depth_form(h, w):
    """the HRNet conv1 weights in the s2d layout (EngineTC._s2d_weights), applied as a 4x4 stride-1 convolution to the s2d
    image (channel (dy * 2 + dx) * 3 + c of s2d pixel (i, j) = image (2i + dy - 4, 2j + dx - 4), 2 zero s2d pixels above /
    left), equal F.conv2d(3x3, stride 2, pad 1) in fp64"""
    from orientedreppoints_b200.detector import ConvLayer
    from orientedreppoints_b200.engine_tc import EngineTC
    g = torch.Generator().manual_seed(h + w)
    wt = torch.randn(64, 3, 3, 3, generator=g).double()                      # fp32 values: the layout is exact in fp64
    img = torch.randn(2, 3, h, w, generator=g, dtype=torch.float64)
    wp = EngineTC._s2d_weights(ConvLayer(wt.float(), None, 2, 1, "cpu")).double()   # [64, kh', kw', 16]
    hs, wsz = h // 2 + 3, w // 2 + 3
    pad = torch.zeros(2, 3, 2 * hs, 2 * wsz, dtype=torch.float64)
    pad[:, :, 4:4 + h, 4:4 + w] = img
    s2d = torch.zeros(2, 16, hs, wsz, dtype=torch.float64)
    for dy in range(2):
        for dx in range(2):
            s2d[:, (dy * 2 + dx) * 3:(dy * 2 + dx) * 3 + 3] = pad[:, :, dy::2, dx::2]
    got = F.conv2d(s2d, wp.permute(0, 3, 1, 2))[:, :, :(h + 1) // 2, :(w + 1) // 2]
    want = F.conv2d(img, wt, None, 2, 1)
    assert got.shape == want.shape
    assert float((got - want).abs().max()) < 1e-12


def test_refusals():
    a = ARCHS["hrnetv2p_w18"]
    for kw, match in ((dict(in_channels=1), "in_channels"), (dict(conv_cfg=dict(type='ConvWS')), "conv_cfg"),
                      (dict(norm_cfg=dict(type='GN', num_groups=2)), "norm_cfg")):
        with pytest.raises(NotImplementedError, match=match):
            build_backbone(dict(dict(type='HRNet', extra=a.extra()), **kw))
    bad = a.extra()
    bad['stage3'] = dict(bad['stage3'], block='BOTTLENECK')
    with pytest.raises(NotImplementedError, match="BOTTLENECK"):
        build_backbone(dict(type='HRNet', extra=bad))
    bad = a.extra()
    bad['stage2'] = dict(bad['stage2'], num_blocks=(4, 4, 4))
    with pytest.raises(ValueError, match="NUM_BRANCHES"):
        HRNetArch.from_extra(bad)
    bad = a.extra()
    bad['stage3'] = dict(bad['stage3'], num_branches=2, num_blocks=(4, 4), num_channels=(18, 36))
    with pytest.raises(NotImplementedError, match="num_branches"):
        HRNetArch.from_extra(bad)
    for kw, match in ((dict(stride=1), "stride"), (dict(num_outs=4), "num_outs")):
        with pytest.raises(NotImplementedError, match=match):
            build_neck(dict(dict(type='HRFPN', in_channels=list(a.out_widths), out_channels=256, stride=2), **kw))
    cfg = _hr_model_cfg()
    cfg['model']['neck'] = _r50_cfg()['model']['neck']
    with pytest.raises(NotImplementedError, match="HRNet with FPN|HRFPN"):
        build_detector(cfg['model'], test_cfg=cfg.get('test_cfg'))
    cfg = _r50_cfg()
    cfg['model']['neck'] = dict(type='HRFPN', in_channels=[256, 512, 1024, 2048], out_channels=256, stride=2)
    with pytest.raises(NotImplementedError, match="ResNet with HRFPN"):
        build_detector(cfg['model'], test_cfg=cfg.get('test_cfg'))
    cfg = _hr_model_cfg()
    cfg['model']['neck']['in_channels'] = [32, 64, 128, 256]
    with pytest.raises(ValueError, match="stage-4 widths"):
        build_detector(cfg['model'], test_cfg=cfg.get('test_cfg'))


def test_engine_refusals():
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    sd = random_hrnet_state_dict("hrnetv2p_w18", seed=0)
    det = OrientedRepPointsDetector(sd, "hrnetv2p_w18", "cpu", "fp32")
    assert det.hr_arch is ARCHS["hrnetv2p_w18"] and det.hrnet.conv2.cout == 64
    assert det.hrnet.stages[0][0][0][0][0][0].cout == 24                     # W18 branch 0: 18 channels carried as 24
    for shape in ((1, 3, 100, 128), (1, 3, 32, 64)):
        with pytest.raises(ValueError, match="multiples of 32"):
            det.extract_feat(torch.zeros(shape))
    bad = dict(sd)
    bad["backbone.stage3.0.branches.1.2.conv2.weight"] = torch.zeros(36, 40, 3, 3)
    with pytest.raises(ValueError, match="shape"):
        OrientedRepPointsDetector(bad, "hrnetv2p_w18", "cpu", "fp32")
    with pytest.raises(ValueError, match="shape"):
        OrientedRepPointsDetector(random_hrnet_state_dict("hrnetv2p_w32", seed=0), "hrnetv2p_w18", "cpu", "fp32")
    with pytest.raises(ValueError, match="pooling_type"):
        OrientedRepPointsDetector(sd, "hrnetv2p_w18", "cpu", "fp32", pooling_type='SUM')
    with pytest.raises(ValueError, match="dcn"):
        OrientedRepPointsDetector(sd, "hrnetv2p_w18", "cpu", "fp32", dcn=((None,),))


def _decls(header):
    src = open(os.path.join(ROOT, "include", header)).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return dict(re.findall(r"\b(orp_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", src))


def test_hrnet_header_bindings_and_arity():
    decls = _decls("orp_b200_hrnet.h")
    assert sorted(decls) == sorted(_lib.HRNET_SIGNATURES) == sorted(
        "orp_%s_%s" % (k, f) for k in ("hr_fuse", "hrfpn_reduce", "hrfpn_pool") for f in ("bf16", "f16x3", "f32"))
    l = _lib.lib()
    for name, params in decls.items():
        assert hasattr(l, name), name
        assert len(_lib.HRNET_SIGNATURES[name][1]) == params.count(",") + 1, name
    for other in ("orp_b200.h", "orp_b200_group.h", "orp_b200_swin.h", "orp_b200_dcnv2.h"):
        assert not set(decls) & set(_decls(other))
