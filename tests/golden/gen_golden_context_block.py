"""Golden vectors for the global context block (GCB): the reference's OWN mmdet/ops/context_block.py (ContextBlock),
mmdet/models/backbones/resnet.py and resnext.py, imported FROM the reference tree with gen_golden_dense.install_stubs() (whose
mmdet.ops then gets the real ContextBlock, and whose conv registry gets a DCNv2 stand-in) and executed on the CPU in float64.
Stored: the first Y_CHANNELS channels of every block output (context_block(x), before the residual add) and the first
C_CHANNELS of C3 / C4 / C5 of every backbone; the context is pooled over all channels and the MLPs mix every channel, so a
slice checks the whole block.  Also stored: the reference's parameter names and shapes of every block and backbone, for the
CPU tests' tree comparison.  Weights come from `orientedreppoints_b200.weights.random_state_dict` draws (gcb_gain > 0, so
every term acts), loaded strict=True with the reference's key names; inputs are regenerated from the seeds stored here.

    python tests/golden/gen_golden_context_block.py   # needs the reference source tree; writes tests/golden/context_block_ref.npz
"""
import importlib
import os
import sys

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import gen_golden_dense                                                              # noqa: E402
from oracle import torch_reference as tr                                             # noqa: E402
from orientedreppoints_b200.weights import random_state_dict                        # noqa: E402

POOLS = ("att", "avg")
FUSIONS = (("channel_add",), ("channel_mul",), ("channel_add", "channel_mul"))
# block cases: (tag, pooling_type, fusion_types, ratio, channels (stage), H, W, seed): every (pooling x fusion) at ratio 1/16
# on an even map and at 1/4 on an odd one, the widths of the four stages in turn
BLOCKS = []
for _i, (_p, _f) in enumerate([(p, f) for p in POOLS for f in FUSIONS]):
    for _j, (_r, _hw) in enumerate(((1. / 16., (8, 12)), (1. / 4., (9, 7)))):
        _c = (256, 512, 1024, 2048)[(2 * _i + _j) % 4]
        BLOCKS.append(("%s_%s_r%d_%s" % (_p, "_".join(x.split("_")[1] for x in _f), round(1 / _r), "even" if _j == 0 else "odd"),
                       _p, _f, _r, _c, _hw[0], _hw[1], 10 + 2 * _i + _j))
C3_C5 = (False, True, True, True)
GA_STAGES = [[], [], [0, 1, 2, 3, 4, 5], [0, 1, 2]]
GA_CFG = dict(spatial_range=-1, num_heads=8, kv_stride=2, attention_type='1111')
# backbone cases: (tag, gcb, depth, groups, base_width, dcn type or None, gen_attention, seed, H, W)
BACKBONES = [("r50_r16", dict(ratio=1. / 16.), 50, 1, 4, None, False, 40, 64, 96),
             ("r50_avg_r4", dict(ratio=1. / 4., pooling_type='avg', fusion_types=('channel_add', 'channel_mul')), 50, 1, 4, None,
              False, 41, 96, 64),
             ("x50_32x4d_r16", dict(ratio=1. / 16.), 50, 32, 4, None, False, 42, 64, 64),
             ("r50_dcnv2_r16", dict(ratio=1. / 16.), 50, 1, 4, 'DCNv2', False, 43, 64, 96),
             ("r50_ga_r16", dict(ratio=1. / 16.), 50, 1, 4, None, True, 44, 96, 64)]
Y_CHANNELS, C_CHANNELS = 32, 64
GAIN, RESIDUAL_GAIN = 1.0, 0.5


def draw(*a, **k):
    """random_state_dict as the tests draw it (float32 tensors: the draws depend on the dtype)"""
    torch.set_default_dtype(torch.float32)
    try:
        return random_state_dict(*a, **k)
    finally:
        torch.set_default_dtype(torch.float64)


def backbone_draw(gcb, depth, groups, base_width, dcn, ga, seed):
    extra = dict(dcn=dict(type=dcn), stage_with_dcn=C3_C5, dcn_offset_scale=0.5) if dcn else {}
    if ga:
        extra.update(gen_attention=GA_CFG, stage_with_gen_attention=GA_STAGES, gen_attention_gamma=0.7)
    return draw(depth, seed=seed, reference_init=False, residual_gain=RESIDUAL_GAIN, groups=groups, base_width=base_width, gcb=gcb,
                stage_with_gcb=C3_C5, gcb_gain=GAIN, **extra)


class ModulatedDeformConvPack(nn.Module):
    """stand-in for mmdet/ops/dcn/deform_conv.py:ModulatedDeformConvPack (CUDA extension): the same parameters (weight, no
    bias, conv_offset 3x3 -> 27 with bias) and forward (offsets = channels 0..17, mask = sigmoid(18..26)), the sampling by
    oracle/torch_reference.py::deform_conv_ref"""

    def __init__(self, cin, cout, kernel_size, stride=1, padding=0, dilation=1, groups=1, deformable_groups=1, bias=False):
        super().__init__()
        assert kernel_size == 3 and dilation == 1 and groups == 1 and deformable_groups == 1 and not bias
        self.stride, self.padding = stride, padding
        self.weight = nn.Parameter(torch.empty(cout, cin, 3, 3))
        self.register_parameter('bias', None)
        self.conv_offset = nn.Conv2d(cin, 27, 3, stride, padding, bias=True)

    def forward(self, x):
        o1, o2, m = torch.chunk(self.conv_offset(x), 3, dim=1)
        return tr.deform_conv_ref(x, torch.cat((o1, o2), dim=1), self.weight, self.stride, self.padding, mask=torch.sigmoid(m))


def main():
    torch.set_default_dtype(torch.float64)
    torch.Tensor.cuda = lambda self, *a, **k: self
    gen_golden_dense.install_stubs()
    CB = importlib.import_module("mmdet.ops.context_block").ContextBlock
    GA = importlib.import_module("mmdet.ops.generalized_attention").GeneralizedAttention
    ops = sys.modules["mmdet.ops"]
    ops.ContextBlock, ops.GeneralizedAttention = CB, GA
    sys.modules["mmdet.ops.conv"].conv_cfg['DCNv2'] = ModulatedDeformConvPack
    resnet = importlib.import_module("mmdet.models.backbones.resnet")
    resnet.ContextBlock, resnet.GeneralizedAttention = CB, GA                         # bound from mmdet.ops at import time
    resnext = importlib.import_module("mmdet.models.backbones.resnext")
    out = {}
    for tag, pool, fus, ratio, c, h, w, seed in BLOCKS:
        cfg = dict(ratio=ratio, pooling_type=pool, fusion_types=fus)
        stages = [False] * 4
        li = (256, 512, 1024, 2048).index(c)
        stages[li] = True
        sd = draw(50, seed=seed, reference_init=False, gcb=cfg, stage_with_gcb=stages, gcb_gain=GAIN)
        pre = "backbone.layer%d.0.context_block." % (li + 1)
        blk = {k[len(pre):]: v.double() for k, v in sd.items() if k.startswith(pre)}
        m = CB(c, **cfg)
        res = m.load_state_dict(blk, strict=True)
        assert not res.missing_keys and not res.unexpected_keys
        m.eval()
        x = torch.randn(2, c, h, w, generator=torch.Generator().manual_seed(seed + 100))
        with torch.no_grad():
            y = m(x)
        out[tag + "_meta"] = np.array([POOLS.index(pool), FUSIONS.index(tuple(fus)), round(1 / ratio), c, h, w, seed], dtype=np.int64)
        out[tag + "_y"] = y[:, :Y_CHANNELS].numpy().astype(np.float32)
        out[tag + "_keys"] = np.array(["%s:%s" % (k, "x".join(str(d) for d in v.shape)) for k, v in m.state_dict().items()])
        print(tag, tuple(y.shape), float((y - x).abs().max()))
    for tag, gcb, depth, groups, bw, dcn, ga, seed, h, w in BACKBONES:
        sd = backbone_draw(gcb, depth, groups, bw, dcn, ga, seed)
        bb = {k[len("backbone."):]: v.double() for k, v in sd.items() if k.startswith("backbone.")}
        kw = dict(depth=depth, num_stages=4, out_indices=(0, 1, 2, 3), frozen_stages=1, norm_cfg=dict(type='BN', requires_grad=True),
                  style='pytorch', gcb=gcb, stage_with_gcb=C3_C5)
        if dcn:
            kw.update(dcn=dict(type=dcn, deformable_groups=1, fallback_on_stride=False), stage_with_dcn=C3_C5)
        if ga:
            kw.update(gen_attention=GA_CFG, stage_with_gen_attention=GA_STAGES)
        model = resnext.ResNeXt(groups=groups, base_width=bw, **kw) if groups > 1 else resnet.ResNet(**kw)
        res = model.load_state_dict(bb, strict=True)
        assert not res.missing_keys and not res.unexpected_keys
        model.eval()
        img = torch.randn(1, 3, h, w, generator=torch.Generator().manual_seed(seed + 10))
        with torch.no_grad():
            feats = model(img)
        out[tag + "_meta"] = np.array([depth, groups, bw, seed, h, w], dtype=np.int64)
        out[tag + "_keys"] = np.array(["%s:%s" % (k, "x".join(str(d) for d in v.shape)) for k, v in model.state_dict().items()
                                       if not k.endswith("num_batches_tracked")])
        for l, f in enumerate(feats):
            if l >= 1:                                                                # C3, C4, C5: the stages with context blocks
                out["%s_c%d" % (tag, l + 2)] = f[:, :C_CHANNELS].numpy().astype(np.float32)
        print(tag, [tuple(f.shape) for f in feats])
    np.savez_compressed(os.path.join(HERE, "context_block_ref.npz"), **out)
    print("wrote context_block_ref.npz")


if __name__ == "__main__":
    main()
