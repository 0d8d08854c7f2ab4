"""Golden vectors for the generalized attention block: the reference's OWN mmdet/ops/generalized_attention.py
(GeneralizedAttention) and mmdet/models/backbones/resnet.py, imported FROM the reference tree with
gen_golden_dense.install_stubs() (whose mmdet.ops then gets the real GeneralizedAttention) and executed on the CPU in float64
(torch.set_default_dtype: the reference builds its position embedding from default-dtype linspace / Tensor; .cuda() is a
no-op here).  Stored: the first Y_CHANNELS channels of every block output and the first C_CHANNELS of C4 / C5; every output
channel passes through proj_conv (and conv3) from all heads and positions, so a slice checks the whole attention.  Weights come from `orientedreppoints_b200.weights.random_state_dict` draws (gen_attention_gamma > 0, so the
blocks act), loaded strict=True with the reference's key names; inputs are regenerated from the seeds stored here.

    python tests/golden/gen_golden_gen_attention.py   # needs the reference source tree; writes tests/golden/gen_attention_ref.npz
"""
import importlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import gen_golden_dense                                                              # noqa: E402
from orientedreppoints_b200.weights import random_state_dict                        # noqa: E402

# block cases: (tag, attention_type, kv_stride, num_heads, planes (stage), H, W, position_magnitude, position_embedding_dim, seed)
BLOCKS = [("t1111_s2_even", "1111", 2, 8, 256, 12, 16, 1, -1, 1), ("t0010_s2_odd", "0010", 2, 8, 256, 9, 11, 1, -1, 2),
          ("t1000_s1_odd", "1000", 1, 8, 256, 7, 9, 1, -1, 3), ("t0101_s2_odd", "0101", 2, 4, 128, 11, 7, 1, -1, 4),
          ("t0001_s1_even", "0001", 1, 8, 512, 6, 8, 1, -1, 5), ("t0111_s2_even", "0111", 2, 16, 512, 8, 6, 2, 64, 6),
          ("t1111_s1_odd", "1111", 1, 8, 256, 5, 13, 1, 128, 7), ("t0010_s1_even", "0010", 1, 16, 512, 6, 6, 1, -1, 8)]
# backbone cases: (tag, attention_type, seed, H, W) on R-50 with the published c4-c5 layout
BACKBONES = [("r50_1111", "1111", 30, 64, 96), ("r50_0010", "0010", 31, 96, 64)]
STAGES = [[], [], [0, 1, 2, 3, 4, 5], [0, 1, 2]]
Y_CHANNELS, C_CHANNELS = 32, 64


def cfg(t, s, heads, mag=1, emb=-1):
    return dict(spatial_range=-1, num_heads=heads, kv_stride=s, attention_type=t, position_magnitude=mag,
                position_embedding_dim=emb)


def draw(*a, **k):
    """random_state_dict as the tests draw it (float32 tensors: the draws depend on the dtype)"""
    torch.set_default_dtype(torch.float32)
    try:
        return random_state_dict(*a, **k)
    finally:
        torch.set_default_dtype(torch.float64)


def main():
    torch.set_default_dtype(torch.float64)
    torch.Tensor.cuda = lambda self, *a, **k: self
    gen_golden_dense.install_stubs()
    GA = importlib.import_module("mmdet.ops.generalized_attention").GeneralizedAttention
    ops = sys.modules["mmdet.ops"]
    ops.GeneralizedAttention = GA
    resnet = importlib.import_module("mmdet.models.backbones.resnet")
    resnet.GeneralizedAttention = GA                                                  # bound from mmdet.ops at import time
    ResNet = resnet.ResNet
    out = {}
    for tag, t, s, heads, planes, h, w, mag, emb, seed in BLOCKS:
        c = cfg(t, s, heads, mag, emb)
        li = (64, 128, 256, 512).index(planes)
        stages = [[], [], [], []]
        stages[li] = [0]
        sd = draw(50, seed=seed, reference_init=False, gen_attention=c, stage_with_gen_attention=stages,
                               gen_attention_gamma=0.7)
        pre = "backbone.layer%d.0.gen_attention_block." % (li + 1)
        blk = {k[len(pre):]: v.double() for k, v in sd.items() if k.startswith(pre)}
        m = GA(planes, **c)
        res = m.load_state_dict(blk, strict=True)
        assert not res.missing_keys and not res.unexpected_keys
        m.eval()
        x = torch.randn(2, planes, h, w, generator=torch.Generator().manual_seed(seed + 100))
        with torch.no_grad():
            y = m(x)
        out[tag + "_meta"] = np.array([int(t, 2), s, heads, planes, h, w, mag, emb, seed], dtype=np.int64)
        out[tag + "_y"] = y[:, :Y_CHANNELS].numpy().astype(np.float32)
        print(tag, tuple(y.shape), float((y - x).abs().max()))
    for tag, t, seed, h, w in BACKBONES:
        c = cfg(t, 2, 8)
        sd = draw(50, seed=seed, reference_init=False, residual_gain=0.5, gen_attention=c,
                               stage_with_gen_attention=STAGES, gen_attention_gamma=0.7)
        bb = {k[len("backbone."):]: v.double() for k, v in sd.items() if k.startswith("backbone.")}
        model = ResNet(depth=50, num_stages=4, out_indices=(0, 1, 2, 3), frozen_stages=1, norm_cfg=dict(type='BN', requires_grad=True),
                       style='pytorch', gen_attention=c, stage_with_gen_attention=STAGES)
        res = model.load_state_dict(bb, strict=True)
        assert not res.missing_keys and not res.unexpected_keys
        model.eval()
        img = torch.randn(1, 3, h, w, generator=torch.Generator().manual_seed(seed + 10))
        with torch.no_grad():
            feats = model(img)
        out[tag + "_meta"] = np.array([int(t, 2), seed, h, w], dtype=np.int64)
        for l, f in enumerate(feats):
            if l >= 2:                                                                # C4, C5: the stages with attention
                out["%s_c%d" % (tag, l + 2)] = f[:, :C_CHANNELS].numpy().astype(np.float32)
        print(tag, [tuple(f.shape) for f in feats])
    np.savez_compressed(os.path.join(HERE, "gen_attention_ref.npz"), **out)
    print("wrote gen_attention_ref.npz")


if __name__ == "__main__":
    main()
