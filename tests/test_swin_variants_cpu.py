"""CPU: the Swin backbones beyond Swin-T/w7 - Swin-T/S/B/L with 7x7 or 12x12 windows.  The config-built parameter containers
against the reference module's own keys and shapes, the arguments the library refuses, the parameterised fp64 oracle against
the reference module's outputs (tests/golden/gen_golden_swin_variants.py, tests/swin_arch_ref.py), the tensor-core planner on every Linear / FPN launch
of Swin-S/B/L, and the bindings of include/orp_b200_swin.h."""
import json
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
NAMES = ["swin_tiny", "swin_tiny_w12", "swin_small", "swin_small_w12", "swin_base", "swin_base_w12", "swin_large", "swin_large_w12"]


def _cfg_model(arch):
    """the model dict of configs/dota/orientedrepoints_swin_tiny_demo.py with backbone and neck set to `arch`"""
    import importlib.util
    spec = importlib.util.spec_from_file_location("cfg", os.path.join(ROOT, "configs", "dota", "orientedrepoints_swin_tiny_demo.py"))
    cfg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cfg)
    model = dict(cfg.model)
    model["backbone"] = dict(model["backbone"], embed_dim=arch.embed, depths=list(arch.depths), num_heads=list(arch.heads),
                             window_size=arch.window)
    model["neck"] = dict(model["neck"], in_channels=[arch.embed * 2, arch.embed * 4, arch.embed * 8])
    return model, cfg.test_cfg


@pytest.mark.parametrize("name", NAMES)
def test_config_built_container_has_the_reference_keys_and_shapes(name):
    from orientedreppoints_b200.models import build_detector
    from orientedreppoints_b200.swin import ARCHS, random_swin_state_dict
    ref = json.load(open(os.path.join(GOLDEN, "swin_var_keys.json")))[name]
    model, test_cfg = _cfg_model(ARCHS[name])
    det = build_detector(model, test_cfg=test_cfg)
    sd = {k: v for k, v in det.state_dict().items() if k.startswith(("backbone.", "neck."))}
    assert {k: list(v.shape) for k, v in sd.items()} == ref["params"]
    # the buffers the reference derives itself: one relative_position_index [w^2, w^2] per block
    w2 = ARCHS[name].window ** 2
    assert all(k.endswith("relative_position_index") and v == [w2, w2] for k, v in ref["buffers"].items())
    assert len(ref["buffers"]) == sum(ARCHS[name].depths)
    assert det.backbone.arch == ARCHS[name]
    # the initialisation draws random_swin_state_dict(0, arch), whose keys are the container's
    rs = random_swin_state_dict(0, arch=ARCHS[name])
    assert set(rs) == set(det.state_dict())
    assert all(torch.equal(det.state_dict()[k], v) for k, v in rs.items())


def test_swin_tiny_draws_are_unchanged():
    """random_swin_state_dict for Swin-T: the committed goldens swin_ref_c{0,1}.npz were made with these numbers"""
    from orientedreppoints_b200.swin import SWIN_T, random_swin_state_dict
    a, b = random_swin_state_dict(0), random_swin_state_dict(0, arch=SWIN_T)
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    assert tuple(a["backbone.layers.0.blocks.0.attn.relative_position_bias_table"].shape) == (169, 3)
    assert float(a["backbone.patch_embed.proj.weight"].sum()) == pytest.approx(-6.69655, abs=1e-4)


@pytest.mark.parametrize("arg,value", [
    ("depths", [2, 2, 6]), ("depths", [2, 2, 6, 2, 2]), ("depths", [2, 0, 6, 2]),
    ("embed_dim", 80), ("embed_dim", 224),
    ("num_heads", [3, 6, 12, 12]), ("num_heads", [6, 12, 24, 48]),
    ("window_size", 8), ("window_size", 14),
    ("qk_scale", "0.1"),
    ("mlp_ratio", 2.), ("qkv_bias", False), ("ape", True), ("patch_norm", False), ("out_indices", (0, 1, 2, 3)),
    ("patch_size", 2), ("in_chans", 4)])
def test_rejected_arguments_name_themselves(arg, value):
    from orientedreppoints_b200.models import SwinTransformer
    kw = dict(embed_dim=96, depths=[2, 2, 6, 2], num_heads=[3, 6, 12, 24], window_size=7, out_indices=(1, 2, 3))
    kw[arg] = value
    with pytest.raises(NotImplementedError, match=arg):
        SwinTransformer(**kw)


def test_qk_scale_reaches_the_container():
    from orientedreppoints_b200.models import SwinTransformer
    m = SwinTransformer(embed_dim=128, depths=[2, 2, 18, 2], num_heads=[4, 8, 16, 32], window_size=12, qk_scale=0.125,
                        out_indices=(1, 2, 3))
    assert m.arch.qk_scale == 0.125 and m.arch.window == 12


def test_engine_names():
    from orientedreppoints_b200.swin import ARCHS, SWIN_T, SwinArch, arch_of
    assert arch_of("swin_tiny") == SWIN_T == SwinArch(96, (2, 2, 6, 2), (3, 6, 12, 24), 7)
    assert arch_of(50) is None and arch_of(101) is None
    assert arch_of("swin_large_w12") == ARCHS["swin_large_w12"]
    with pytest.raises(ValueError):
        arch_of("swin_huge")
    with pytest.raises(NotImplementedError, match="window_size"):
        arch_of(SwinArch(96, (2, 2, 6, 2), (3, 6, 12, 24), 9))


@pytest.mark.parametrize("tag,name", [("s_w7", "swin_small"), ("b_w12", "swin_base_w12")])
def test_parameterised_oracle_equals_reference_module(tag, name):
    """the reference's own SwinTransformer + FPN in fp64 (window padding at every stage, stages smaller than one window)
    against the fp64 restatement of tests/swin_arch_ref.py"""
    import swin_arch_ref as ts
    from orientedreppoints_b200.swin import ARCHS, random_swin_state_dict
    g = np.load(os.path.join(GOLDEN, "swin_var_%s.npz" % tag))
    arch = ARCHS[name]
    sd = {k: v.double() for k, v in random_swin_state_dict(0, arch=arch).items()}
    img = torch.from_numpy(g["img"])
    with torch.no_grad():
        c = ts.swin_forward(sd, img, arch=arch)
        f = ts.swin_fpn(sd, c)
    for i, a in enumerate(c):
        ref = torch.from_numpy(g["stage%d" % i])
        assert a.shape == ref.shape and float((a - ref).abs().max()) < 1e-10 * max(1.0, float(ref.abs().max())), i
    for i, a in enumerate(f):
        ref = torch.from_numpy(g["fpn%d" % i])
        assert a.shape == ref.shape and float((a - ref).abs().max()) < 1e-10 * max(1.0, float(ref.abs().max())), i


def test_parameterised_oracle_is_the_swin_t_oracle():
    """with Swin-T's arguments tests/swin_arch_ref.py computes what oracle/torch_swin.py computes (pinned to the reference by
    tests/golden/swin_ref_c{0,1}.npz), on a grid that needs window padding"""
    import swin_arch_ref as sr
    from oracle import torch_swin as ts
    from orientedreppoints_b200.swin import SWIN_T, random_swin_state_dict
    sd = {k: v.double() for k, v in random_swin_state_dict(0).items()}
    img = torch.randn(1, 3, 70, 100, generator=torch.Generator().manual_seed(7), dtype=torch.float64)
    with torch.no_grad():
        a, b = sr.swin_forward(sd, img, SWIN_T), ts.swin_forward(sd, img)
    for x, y in zip(a, b):
        assert x.shape == y.shape and float((x - y).abs().max()) < 1e-12 * max(1.0, float(y.abs().max()))


def swin_linear_launches(arch, n, tile):
    """(name, (N, H, W), Cin, Cout, k, bias, relu, residual, gn) of every tensor-core launch of the backbone and FPN for n tiles of
    tile x tile: patch embed, per stage qkv on the window-padded grid, proj (+ shortcut), fc1 (+ GELU), fc2 (+ shortcut), the
    PatchMerging reduction, the FPN laterals and 3x3 convolutions (GroupNorm statistics in the epilogue)"""
    out = []
    h = (tile + 3) // 4
    out.append(("embed", (n, h, h), 64, arch.embed, 1, True, 0, 0, False))
    ws = arch.window
    for i in range(4):
        c = arch.embed << i
        hp = -(-h // ws) * ws
        out += [("qkv%d" % i, (n, hp, hp), c, 3 * c, 1, True, 0, 0, False), ("proj%d" % i, (n, h, h), c, c, 1, True, 0, 1, False),
                ("fc1_%d" % i, (n, h, h), c, 4 * c, 1, True, 2, 0, False), ("fc2_%d" % i, (n, h, h), 4 * c, c, 1, True, 0, 1, False)]
        if i < 3:
            h = (h + 1) // 2
            out.append(("red%d" % i, (n, h, h), 4 * c, 2 * c, 1, False, 0, 0, False))
    for i, s in enumerate((8, 16, 32)):
        hw = -(-tile // s)
        out += [("lat%d" % i, (n, hw, hw), arch.embed << (i + 1), 256, 1, False, 0, 0, True),
                ("fpn%d" % i, (n, hw, hw), 256, 256, 3, False, 0, 0, True)]
    return out


@pytest.mark.parametrize("split", [1, 0], ids=["f16x3", "bf16"])
@pytest.mark.parametrize("name", ["swin_small", "swin_small_w12", "swin_base", "swin_base_w12", "swin_large", "swin_large_w12"])
@pytest.mark.parametrize("tile", [1024, 960])
def test_planner_takes_every_linear_and_fpn_launch(split, name, tile):
    from orientedreppoints_b200 import _lib
    from orientedreppoints_b200.engine_tc import EngineTCSplit
    from orientedreppoints_b200.swin import ARCHS
    for lname, prob, cin, cout, k, bias, relu, residual, gn in swin_linear_launches(ARCHS[name], 8, tile):
        cout_p = EngineTCSplit._pad_cout(cout) if split else (cout + 31) // 32 * 32
        p = _lib.tc_plan_for([prob], cout, cout_p, k, k, cin, 1, k // 2, bias=bias, relu=relu, residual=residual, gn=gn,
                             split=split)
        n, h, w = prob
        assert p["Cout"] == cout and p["Cout_padded"] == cout_p and p["split"] == split, lname
        assert p["BN"] in (32, 64, 128, 256) and p["grid"] >= 1 and p["stages"] >= 2, lname
        m_tiles = -(-n * h * w // 128)
        assert p["num_tiles"] >= m_tiles and p["grid"] <= max(132, p["num_tiles"]), (lname, p)
        assert p["bias"] == int(bias) and p["relu"] == relu and p["gn_fused"] in (0, 1), lname


def test_bindings_match_header():
    """orp_b200_swin.h's entry points are exported and bound with their declared arity; orp_b200.h does not declare them"""
    from orientedreppoints_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "orp_b200_swin.h")).read(), flags=re.S)
    decls = dict(re.findall(r"\b(orp_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", src))
    assert sorted(decls) == sorted(_lib.SWIN_SIGNATURES) and len(decls) == 4
    for name, params in decls.items():
        assert hasattr(_lib.lib(), name) and len(_lib.SWIN_SIGNATURES[name][1]) == params.count(",") + 1
        assert name not in _lib.SIGNATURES
