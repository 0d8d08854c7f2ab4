"""Swin-T backbone (mmdet/models/backbones/swin_transformer.py:449-631; cfg configs/dota/orientedrepoints_swin_tiny_demo.py:9-24:
embed_dim 96, depths [2,2,6,2], heads [3,6,12,24], window 7, mlp_ratio 4, qkv_bias, patch_norm, out_indices (1,2,3))
over the tensor-core engine: every Linear is a 1x1 convolution launch (csrc/dense_tc.cu), everything else is csrc/swin.cu.
Tokens are bf16 NHWC [B,H,W,C]; state-dict keys are the reference's (backbone.patch_embed.proj.weight, backbone.layers.i.blocks.j.
attn.qkv.weight, ..., backbone.layers.i.downsample.reduction.weight, backbone.norm{1,2,3}.weight)."""
import math

import torch

from . import _lib
from .detector import ConvLayer

DEPTHS = (2, 2, 6, 2)
HEADS = (3, 6, 12, 24)
EMBED = 96
WINDOW = 7


def random_swin_state_dict(seed=0, feat=256, num_classes=16):
    """trunc_normal(.02) linears, zero biases, unit LayerNorms (swin_transformer.py:571-579) - plus the FPN/head
    entries of weights.random_state_dict with the Swin neck shapes.  Biases/norms are randomised a little so that
    every term of the graph carries signal in the parity tests."""
    from .weights import random_state_dict
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def lin(name, cout, cin, bias=True):
        sd[name + ".weight"] = torch.empty(cout, cin).normal_(0, 0.02, generator=g).clamp_(-0.04, 0.04)
        if bias:
            sd[name + ".bias"] = torch.empty(cout).normal_(0, 0.02, generator=g)

    def ln(name, c):
        sd[name + ".weight"] = torch.empty(c).uniform_(0.8, 1.2, generator=g)
        sd[name + ".bias"] = torch.empty(c).normal_(0, 0.05, generator=g)

    sd["backbone.patch_embed.proj.weight"] = torch.empty(EMBED, 3, 4, 4).normal_(0, 0.1, generator=g)
    sd["backbone.patch_embed.proj.bias"] = torch.empty(EMBED).normal_(0, 0.02, generator=g)
    ln("backbone.patch_embed.norm", EMBED)
    for i, (depth, heads) in enumerate(zip(DEPTHS, HEADS)):
        c = EMBED << i
        for j in range(depth):
            p = "backbone.layers.%d.blocks.%d." % (i, j)
            ln(p + "norm1", c)
            lin(p + "attn.qkv", 3 * c, c)
            lin(p + "attn.proj", c, c)
            sd[p + "attn.relative_position_bias_table"] = torch.empty(169, heads).normal_(0, 0.2, generator=g)
            ln(p + "norm2", c)
            lin(p + "mlp.fc1", 4 * c, c)
            lin(p + "mlp.fc2", c, 4 * c)
        if i < 3:
            ln("backbone.layers.%d.downsample.norm" % i, 4 * c)
            lin("backbone.layers.%d.downsample.reduction" % i, 2 * c, 4 * c, bias=False)
    for i in (1, 2, 3):
        ln("backbone.norm%d" % i, EMBED << i)
    base = random_state_dict(50, seed=seed + 1, reference_init=False, num_classes=num_classes, feat=feat)
    for k, v in base.items():
        if k.startswith("bbox_head."):
            sd[k] = v
    for i, cin in enumerate((192, 384, 768)):
        sd["neck.lateral_convs.%d.conv.weight" % i] = torch.empty(feat, cin, 1, 1).normal_(0, 1.0 / math.sqrt(cin), generator=g)
        sd["neck.fpn_convs.%d.conv.weight" % i] = torch.empty(feat, feat, 3, 3).normal_(0, 1.0 / math.sqrt(feat * 9), generator=g)
        for kind in ("lateral_convs", "fpn_convs"):
            sd["neck.%s.%d.gn.weight" % (kind, i)] = torch.empty(feat).uniform_(0.5, 1.5, generator=g)
            sd["neck.%s.%d.gn.bias" % (kind, i)] = torch.empty(feat).normal_(0, 0.1, generator=g)
    return sd


class _LN:
    def __init__(self, sd, prefix, device):
        self.gamma = sd[prefix + ".weight"].to(device, torch.float32).contiguous()
        self.beta = sd[prefix + ".bias"].to(device, torch.float32).contiguous()


def _linear(sd, prefix, device):
    w = sd[prefix + ".weight"].float()
    b = sd.get(prefix + ".bias")
    return ConvLayer(w[:, :, None, None], None if b is None else b.float(), 1, 0, device)


class SwinTiny:
    def __init__(self, sd, device, engine):
        self.dev, self.e, self.lib = device, engine, _lib.lib()
        w = sd["backbone.patch_embed.proj.weight"].float()                    # [96,3,4,4] -> rows k = c*16 + kh*4 + kw, K 48 -> 64
        wk = torch.zeros(EMBED, 64)
        wk[:, :48] = w.reshape(EMBED, 48)
        self.embed = ConvLayer(wk[:, :, None, None], sd["backbone.patch_embed.proj.bias"].float(), 1, 0, device)
        self.embed_norm = _LN(sd, "backbone.patch_embed.norm", device)
        self.blocks, self.merges = [], []
        for i, (depth, heads) in enumerate(zip(DEPTHS, HEADS)):
            stage = []
            for j in range(depth):
                p = "backbone.layers.%d.blocks.%d." % (i, j)
                stage.append(dict(norm1=_LN(sd, p + "norm1", device), qkv=_linear(sd, p + "attn.qkv", device),
                                  proj=_linear(sd, p + "attn.proj", device),
                                  table=sd[p + "attn.relative_position_bias_table"].to(device, torch.float32).contiguous(),
                                  norm2=_LN(sd, p + "norm2", device), fc1=_linear(sd, p + "mlp.fc1", device),
                                  fc2=_linear(sd, p + "mlp.fc2", device), heads=heads, shift=0 if j % 2 == 0 else WINDOW // 2))
            self.blocks.append(stage)
            if i < 3:
                self.merges.append(dict(norm=_LN(sd, "backbone.layers.%d.downsample.norm" % i, device),
                                        red=_linear(sd, "backbone.layers.%d.downsample.reduction" % i, device)))
        self.out_norms = {i: _LN(sd, "backbone.norm%d" % i, device) for i in (1, 2, 3)}
        self._padded = {}

    # ------------------------------------------------------------------ primitive launches
    # (the engine decides the activation format: bf16 [B,H,W,C] or split fp16 [B,H,W,2,C]; `e.suffix` picks the entry points)
    def _fn(self, name):
        return getattr(self.lib, "orp_%s_%s" % (name, self.e.suffix))

    def _ln(self, x, norm, hp=None, wp=None):
        b, h, w, c = self.e.dims(x)
        hp, wp = hp or h, wp or w
        if (hp, wp) != (h, w):
            # F.pad zeros after norm1: the kernel writes the H x W interior only, so one zero-filled buffer per shape is
            # reused by every block of the stage (its consumer, the qkv projection, is stream-ordered before the next norm1)
            key = (b, h, w, hp, wp, c)
            y = self._padded.get(key)
            if y is None:
                y = self._padded[key] = self.e.alloc(b, hp, wp, c, zero=True)
        else:
            y = self.e.alloc(b, hp, wp, c)
        _lib.check(self._fn("layernorm")(_lib.ptr(x), b, h, w, c, _lib.ptr(norm.gamma), _lib.ptr(norm.beta), 1e-5, hp, wp,
                                         _lib.ptr(y), _lib.current_stream_ptr()), "orp_layernorm")
        return y

    def _attention(self, qkv, b, h, w, c, heads, shift, table):
        _, hp, wp, _ = self.e.dims(qkv)
        out = self.e.alloc(b, h, w, c)
        _lib.check(self._fn("window_attention")(_lib.ptr(qkv), b, h, w, hp, wp, c, heads, shift, _lib.ptr(table),
                                                float((c // heads) ** -0.5), _lib.ptr(out), _lib.current_stream_ptr()),
                   "orp_window_attention")
        return out

    def block(self, x, blk):
        e = self.e
        b, h, w, c = e.dims(x)
        hp = (h + WINDOW - 1) // WINDOW * WINDOW
        wp = (w + WINDOW - 1) // WINDOW * WINDOW
        t = self._ln(x, blk["norm1"], hp, wp)
        qkv = e.conv(t, blk["qkv"])                                                       # [B,Hp,Wp,3C], padded tokens -> bias
        a = self._attention(qkv, b, h, w, c, blk["heads"], blk["shift"], blk["table"])
        x = e.conv(a, blk["proj"], residual=x)                                            # x = shortcut + proj(attn)
        t = self._ln(x, blk["norm2"])
        hmid = e.conv(t, blk["fc1"], relu=2)                                              # fc1 + exact GELU
        return e.conv(hmid, blk["fc2"], residual=x)                                       # x = x + mlp(norm2(x))

    def merge(self, x, m):
        b, h, w, c = self.e.dims(x)
        ho, wo = (h + 1) // 2, (w + 1) // 2
        g = self.e.alloc(b, ho, wo, 4 * c)
        _lib.check(self._fn("patch_merge_gather")(_lib.ptr(x), b, h, w, c, _lib.ptr(g), _lib.current_stream_ptr()),
                   "orp_patch_merge_gather")
        return self.e.conv(self._ln(g, m["norm"]), m["red"])

    def forward(self, img, img_norm_cfg=None, valid_hw=None):
        """img: normalised float NCHW, or decoded uint8 HWC tiles [B,H,W,3] together with the pipeline's img_norm_cfg (Normalize +
        ImageToTensor are then fused into the patch gather; with valid_hw, device int32 [B,2] per-image extents, so is the Pad
        after Normalize: pixels outside enter as 0.0)"""
        if img.dtype == torch.uint8:
            import ctypes
            img = img.to(self.dev).contiguous()
            b, h, w, _ = img.shape
            mean = (ctypes.c_float * 3)(*[float(v) for v in img_norm_cfg["mean"]])
            stdinv = (ctypes.c_float * 3)(*[1.0 / float(v) for v in img_norm_cfg["std"]])      # rounded to fp32 as detector.normalize does
            ho, wo = (h + 3) // 4, (w + 3) // 4
            rows = self.e.alloc(b, ho, wo, 64)
            to_rgb = 1 if img_norm_cfg.get("to_rgb", True) else 0
            if valid_hw is None:
                _lib.check(self._fn("patch_embed_rows_u8")(_lib.ptr(img), b, h, w, mean, stdinv, to_rgb, _lib.ptr(rows),
                                                          _lib.current_stream_ptr()), "orp_patch_embed_rows_u8")
            else:
                from .engine_tc import _valid
                _lib.check(self._fn("patch_embed_rows_u8_padded")(_lib.ptr(img), b, h, w, mean, stdinv, to_rgb,
                                                                 _lib.ptr(_valid(valid_hw, b, img.device)), _lib.ptr(rows),
                                                                 _lib.current_stream_ptr()), "orp_patch_embed_rows_u8_padded")
        else:
            assert valid_hw is None, "valid_hw applies to uint8 images (float input is already normalised and padded)"
            img = img.to(self.dev, torch.float32).contiguous()
            b, _, h, w = img.shape
            ho, wo = (h + 3) // 4, (w + 3) // 4
            rows = self.e.alloc(b, ho, wo, 64)
            _lib.check(self._fn("patch_embed_rows")(_lib.ptr(img), b, h, w, _lib.ptr(rows), _lib.current_stream_ptr()),
                       "orp_patch_embed_rows")
        x = self._ln(self.e.conv(rows, self.embed), self.embed_norm)
        outs = []
        for i, stage in enumerate(self.blocks):
            for blk in stage:
                x = self.block(x, blk)
            if i in self.out_norms:
                outs.append(self._ln(x, self.out_norms[i]))
            if i < 3:
                x = self.merge(x, self.merges[i])
        return outs

    def subsample2(self, x):
        b, h, w, c = self.e.dims(x)
        y = self.e.alloc(b, (h - 1) // 2 + 1, (w - 1) // 2 + 1, c)
        _lib.check(self._fn("subsample2")(_lib.ptr(x), b, h, w, c, _lib.ptr(y), _lib.current_stream_ptr()), "orp_subsample2")
        return y
