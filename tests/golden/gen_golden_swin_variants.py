"""Golden vectors for the Swin backbones beyond Swin-T/w7 (SURVEY §8 a2): the reference's OWN
mmdet/models/backbones/swin_transformer.py::SwinTransformer and mmdet/models/necks/fpn.py::FPN(in_channels=[2E,4E,8E],
num_outs=5, GN), imported from the reference source tree with the stubs of gen_golden_swin.py and run on the CPU in float64
(eval mode: DropPath is the identity).

- swin_var_s_w7.npz, swin_var_b_w12.npz: Swin-S / window 7 and Swin-B / window 12 on one 60 x 76 image (tokens 15 x 19: every
  window grid is padded; the 1/16 and 1/32 stages are smaller than one window), weights random_swin_state_dict(0, arch=...)
  (not stored: a depth-18 backbone is tens of MB).  Outputs of the three backbone stages and the five FPN levels.
- swin_var_keys.json: the state-dict keys and shapes of backbone + neck for Swin-T/S/B/L at windows 7 and 12 (buffers the
  reference derives itself, relative_position_index, listed apart).

    python tests/golden/gen_golden_swin_variants.py     # needs the reference source tree
"""
import json
import os
import sys

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import gen_golden_dense as gd                                                        # noqa: E402
from orientedreppoints_b200.swin import ARCHS, random_swin_state_dict               # noqa: E402

CASES = {"s_w7": "swin_small", "b_w12": "swin_base_w12"}
IMG = (60, 76)


def install():
    """the stubs of gen_golden_swin.main (timm.models.layers, mmcv_custom, registries) -> (SwinTransformer, FPN)"""
    import importlib
    import types
    _, FPN, _ = gd.install_stubs()
    timm = gd._pkg("timm")
    tm = gd._pkg("timm.models")
    layers = types.ModuleType("timm.models.layers")

    class DropPath(nn.Module):
        def __init__(self, drop_prob=None):
            super().__init__()

        def forward(self, x):
            return x
    layers.DropPath = DropPath
    layers.to_2tuple = lambda v: v if isinstance(v, tuple) else (v, v)
    layers.trunc_normal_ = lambda *a, **k: None
    sys.modules["timm.models.layers"] = layers
    timm.models, tm.layers = tm, layers
    mc = types.ModuleType("mmcv_custom")
    mc.load_checkpoint = lambda *a, **k: None
    sys.modules["mmcv_custom"] = mc
    return importlib.import_module("mmdet.models.backbones.swin_transformer").SwinTransformer, FPN


def build(Swin, FPN, arch):
    m = nn.Module()
    m.backbone = Swin(embed_dim=arch.embed, depths=list(arch.depths), num_heads=list(arch.heads), window_size=arch.window,
                      mlp_ratio=4., qkv_bias=True, qk_scale=None, drop_rate=0., attn_drop_rate=0., drop_path_rate=0.2, ape=False,
                      patch_norm=True, out_indices=(1, 2, 3), use_checkpoint=False)
    m.neck = FPN(in_channels=[arch.embed * 2, arch.embed * 4, arch.embed * 8], out_channels=256, num_outs=5,
                 norm_cfg=dict(type='GN', num_groups=32, requires_grad=True))
    return m


def main():
    Swin, FPN = install()
    keys = {}
    for name in ("swin_tiny", "swin_tiny_w12", "swin_small", "swin_small_w12", "swin_base", "swin_base_w12", "swin_large",
                 "swin_large_w12"):
        m = build(Swin, FPN, ARCHS[name])
        bufs = set(k for k, _ in m.named_buffers())
        keys[name] = dict(params={k: list(v.shape) for k, v in m.state_dict().items() if k not in bufs},
                          buffers={k: list(v.shape) for k, v in m.state_dict().items() if k in bufs})
        print(name, len(keys[name]["params"]), len(keys[name]["buffers"]))
        del m
    with open(os.path.join(HERE, "swin_var_keys.json"), "w") as f:
        json.dump(keys, f, indent=0, sort_keys=True)
    for tag, name in CASES.items():
        arch = ARCHS[name]
        m = build(Swin, FPN, arch)
        sd = random_swin_state_dict(0, arch=arch)
        given = {k: v for k, v in sd.items() if k.startswith(("backbone.", "neck."))}
        own = m.state_dict()
        assert all(k.endswith(("relative_position_index", "attn_mask")) for k in own if k not in given)
        assert not [k for k in given if k not in own]
        m.load_state_dict(given, strict=False)
        m = m.double().eval()
        img = torch.randn(1, 3, *IMG, generator=torch.Generator().manual_seed(40), dtype=torch.float64)
        with torch.no_grad():
            c = m.backbone(img)
            fo = m.neck(c)
        out = {"img": img.numpy()}
        for i, t in enumerate(c):
            out["stage%d" % i] = t.numpy()
        for i, t in enumerate(fo):
            out["fpn%d" % i] = t.numpy()
        print(tag, [tuple(t.shape) for t in c], [tuple(t.shape) for t in fo])
        path = os.path.join(HERE, "swin_var_%s.npz" % tag)
        np.savez_compressed(path, **out)
        print("wrote", path, os.path.getsize(path))


if __name__ == "__main__":
    main()
