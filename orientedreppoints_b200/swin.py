"""Swin backbones (mmdet/models/backbones/swin_transformer.py:449-631) over the tensor-core engines: every Linear is a 1x1
convolution launch (csrc/dense_tc.cu), everything else is csrc/swin.cu.  Built for any architecture with four stages, head
dimension 32, embed_dim a multiple of 32 up to 192 and window 7 or 12 - Swin-T/S/B/L as published - with the rest as
configs/dota/orientedrepoints_swin_tiny_demo.py:9-24 has it (mlp_ratio 4, qkv_bias, patch_norm, no ape, patch_size 4,
out_indices (1,2,3)).  Tokens are NHWC [B,H,W,C] in the engine's format; state-dict keys are the reference's
(backbone.patch_embed.proj.weight, backbone.layers.i.blocks.j.attn.qkv.weight, ..., backbone.layers.i.downsample.reduction.weight,
backbone.norm{1,2,3}.weight)."""
import math
from collections import namedtuple

import torch

from . import _lib
from .detector import ConvLayer

DEPTHS = (2, 2, 6, 2)
HEADS = (3, 6, 12, 24)
EMBED = 96
WINDOW = 7


class SwinArch(namedtuple("SwinArch", "embed depths heads window qk_scale")):
    """embed_dim, depths, num_heads, window_size and qk_scale (None: head_dim ** -0.5) of a Swin backbone"""
    __slots__ = ()

    def __new__(cls, embed=EMBED, depths=DEPTHS, heads=HEADS, window=WINDOW, qk_scale=None):
        return super().__new__(cls, int(embed), tuple(int(d) for d in depths), tuple(int(h) for h in heads), int(window),
                               None if qk_scale is None else float(qk_scale))

    @property
    def channels(self):
        return tuple(self.embed << i for i in range(4))


def _arch(embed, depths, heads):
    return {"": SwinArch(embed, depths, heads, 7), "_w12": SwinArch(embed, depths, heads, 12)}


# the published Swin-T/S/B/L (7: 224 pretraining, 12: 384 pretraining); "swin_tiny" is the backbone of
# configs/dota/orientedrepoints_swin_tiny_demo.py
ARCHS = {name + sfx: a for name, (e, d, h) in (("swin_tiny", (96, (2, 2, 6, 2), (3, 6, 12, 24))),
                                              ("swin_small", (96, (2, 2, 18, 2), (3, 6, 12, 24))),
                                              ("swin_base", (128, (2, 2, 18, 2), (4, 8, 16, 32))),
                                              ("swin_large", (192, (2, 2, 18, 2), (6, 12, 24, 48))))
         for sfx, a in _arch(e, d, h).items()}
SWIN_T = ARCHS["swin_tiny"]


def check_arch(embed_dim, depths, num_heads, window_size, qk_scale=None):
    """the SwinArch of these SwinTransformer arguments; NotImplementedError naming the argument the library cannot build"""
    depths, num_heads = tuple(depths), tuple(num_heads)
    if len(depths) != 4:
        raise NotImplementedError("liborp_b200 builds Swin backbones with four stages, not depths=%r" % (depths,))
    if any(int(d) != d or d < 1 for d in depths):
        raise NotImplementedError("liborp_b200 builds Swin stages of at least one block, not depths=%r" % (depths,))
    if int(embed_dim) != embed_dim or embed_dim <= 0 or embed_dim % 32 or embed_dim * 8 > 1536:
        raise NotImplementedError("liborp_b200 builds Swin backbones with embed_dim a multiple of 32 and at most 192 (every block "
                                  "LayerNorm <= 1536 channels), not embed_dim=%r" % (embed_dim,))
    if len(num_heads) != 4 or any(h <= 0 or (int(embed_dim) << i) != 32 * h for i, h in enumerate(num_heads)):
        raise NotImplementedError("liborp_b200 builds Swin attention with head dimension 32 at every stage (num_heads = "
                                  "embed_dim * 2**i / 32), not num_heads=%r for embed_dim=%r" % (num_heads, embed_dim))
    if window_size not in (7, 12):
        raise NotImplementedError("liborp_b200 builds Swin window attention over 7x7 or 12x12 windows, not window_size=%r"
                                  % (window_size,))
    if qk_scale is not None and not isinstance(qk_scale, (int, float)):
        raise NotImplementedError("qk_scale must be None or a float, not qk_scale=%r" % (qk_scale,))
    return SwinArch(embed_dim, depths, num_heads, window_size, qk_scale)


def arch_of(depth):
    """the SwinArch an engine's `depth` names ("swin_tiny", any key of ARCHS, or a SwinArch), None for a ResNet depth"""
    if isinstance(depth, SwinArch):
        return check_arch(depth.embed, depth.depths, depth.heads, depth.window, depth.qk_scale)
    if isinstance(depth, str) and depth.startswith("swin"):
        if depth not in ARCHS:
            raise ValueError("unknown Swin backbone %r: one of %s, or a swin.SwinArch" % (depth, ", ".join(sorted(ARCHS))))
        return ARCHS[depth]
    return None


def random_swin_state_dict(seed=0, feat=256, num_classes=16, arch=SWIN_T):
    """trunc_normal(.02) linears, zero biases, unit LayerNorms (swin_transformer.py:571-579) - plus the FPN/head
    entries of weights.random_state_dict with the Swin neck shapes (in_channels 2E, 4E, 8E).  Biases/norms are randomised a
    little so that every term of the graph carries signal in the parity tests.  The draws are in parameter order, so Swin-T's
    are those of every earlier version of this function."""
    from .weights import random_state_dict
    arch = arch_of(arch) if not isinstance(arch, str) else ARCHS[arch]
    embed, nb = arch.embed, (2 * arch.window - 1) ** 2
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def lin(name, cout, cin, bias=True):
        sd[name + ".weight"] = torch.empty(cout, cin).normal_(0, 0.02, generator=g).clamp_(-0.04, 0.04)
        if bias:
            sd[name + ".bias"] = torch.empty(cout).normal_(0, 0.02, generator=g)

    def ln(name, c):
        sd[name + ".weight"] = torch.empty(c).uniform_(0.8, 1.2, generator=g)
        sd[name + ".bias"] = torch.empty(c).normal_(0, 0.05, generator=g)

    sd["backbone.patch_embed.proj.weight"] = torch.empty(embed, 3, 4, 4).normal_(0, 0.1, generator=g)
    sd["backbone.patch_embed.proj.bias"] = torch.empty(embed).normal_(0, 0.02, generator=g)
    ln("backbone.patch_embed.norm", embed)
    for i, (depth, heads) in enumerate(zip(arch.depths, arch.heads)):
        c = embed << i
        for j in range(depth):
            p = "backbone.layers.%d.blocks.%d." % (i, j)
            ln(p + "norm1", c)
            lin(p + "attn.qkv", 3 * c, c)
            lin(p + "attn.proj", c, c)
            sd[p + "attn.relative_position_bias_table"] = torch.empty(nb, heads).normal_(0, 0.2, generator=g)
            ln(p + "norm2", c)
            lin(p + "mlp.fc1", 4 * c, c)
            lin(p + "mlp.fc2", c, 4 * c)
        if i < 3:
            ln("backbone.layers.%d.downsample.norm" % i, 4 * c)
            lin("backbone.layers.%d.downsample.reduction" % i, 2 * c, 4 * c, bias=False)
    for i in (1, 2, 3):
        ln("backbone.norm%d" % i, embed << i)
    base = random_state_dict(50, seed=seed + 1, reference_init=False, num_classes=num_classes, feat=feat)
    for k, v in base.items():
        if k.startswith("bbox_head."):
            sd[k] = v
    for i, cin in enumerate(arch.channels[1:]):
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


class Swin:
    """the backbone of one SwinArch; picks its attention (7x7 / 12x12 windows) and LayerNorm (<= 1536 / wider) entry points"""

    def __init__(self, sd, device, engine, arch=SWIN_T):
        self.dev, self.e, self.lib = device, engine, _lib.lib()
        self.arch = arch = arch_of(arch)
        embed, win = arch.embed, arch.window
        nb = (2 * win - 1) ** 2
        w = sd["backbone.patch_embed.proj.weight"].float()                    # [E,3,4,4] -> rows k = c*16 + kh*4 + kw, K 48 -> 64
        if tuple(w.shape) != (embed, 3, 4, 4):
            raise ValueError("backbone.patch_embed.proj.weight is %s; embed_dim %d needs [%d,3,4,4]" % (tuple(w.shape), embed, embed))
        wk = torch.zeros(embed, 64)
        wk[:, :48] = w.reshape(embed, 48)
        self.embed = ConvLayer(wk[:, :, None, None], sd["backbone.patch_embed.proj.bias"].float(), 1, 0, device)
        self.embed_norm = _LN(sd, "backbone.patch_embed.norm", device)
        self.blocks, self.merges = [], []
        for i, (depth, heads) in enumerate(zip(arch.depths, arch.heads)):
            stage = []
            for j in range(depth):
                p = "backbone.layers.%d.blocks.%d." % (i, j)
                table = sd[p + "attn.relative_position_bias_table"]
                if tuple(table.shape) != (nb, heads):
                    raise ValueError("%sattn.relative_position_bias_table is %s; window %d with %d heads needs [%d,%d]"
                                     % (p, tuple(table.shape), win, heads, nb, heads))
                stage.append(dict(norm1=_LN(sd, p + "norm1", device), qkv=_linear(sd, p + "attn.qkv", device),
                                  proj=_linear(sd, p + "attn.proj", device),
                                  table=table.to(device, torch.float32).contiguous(),
                                  norm2=_LN(sd, p + "norm2", device), fc1=_linear(sd, p + "mlp.fc1", device),
                                  fc2=_linear(sd, p + "mlp.fc2", device), heads=heads, shift=0 if j % 2 == 0 else win // 2))
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
        name = "layernorm" if c <= 1536 else "layernorm_wide"                 # the PatchMerging norms of Swin-B / L are wider
        _lib.check(self._fn(name)(_lib.ptr(x), b, h, w, c, _lib.ptr(norm.gamma), _lib.ptr(norm.beta), 1e-5, hp, wp,
                                  _lib.ptr(y), _lib.current_stream_ptr()), "orp_" + name)
        return y

    def _attention(self, qkv, b, h, w, c, heads, shift, table):
        _, hp, wp, _ = self.e.dims(qkv)
        out = self.e.alloc(b, h, w, c)
        name = "window_attention" if self.arch.window == 7 else "window_attention12"
        scale = float((c // heads) ** -0.5) if self.arch.qk_scale is None else self.arch.qk_scale     # WindowAttention :83
        _lib.check(self._fn(name)(_lib.ptr(qkv), b, h, w, hp, wp, c, heads, shift, _lib.ptr(table), scale, _lib.ptr(out),
                                  _lib.current_stream_ptr()), "orp_" + name)
        return out

    def block(self, x, blk):
        e = self.e
        b, h, w, c = e.dims(x)
        ws = self.arch.window
        hp = (h + ws - 1) // ws * ws
        wp = (w + ws - 1) // ws * ws
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
