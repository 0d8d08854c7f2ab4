"""fp64 evaluation of a Swin backbone of any architecture the library builds (test infrastructure): oracle/torch_swin.py's Swin-T
restatement (mmdet/models/backbones/swin_transformer.py:21-631) with embed_dim, depths, num_heads, window_size and qk_scale as
arguments.  Window partition / reverse, the shift mask, PatchMerging and the FPN are oracle/torch_swin.py's own functions (they
take any window and width); what is restated here is the part that reads Swin-T's constants: the attention core (relative
position bias table of (2 w - 1)^2 rows, qk_scale), the block (padding to multiples of the window) and the forward pass.
Pinned to the reference's own SwinTransformer + FPN for Swin-S/w7 and Swin-B/w12 by tests/golden/gen_golden_swin_variants.py
(tests/test_swin_variants_cpu.py); with Swin-T's arguments it is oracle/torch_swin.py's computation."""
import torch
import torch.nn.functional as F

from oracle import torch_swin as ts

SWIN_T = (96, (2, 2, 6, 2), (3, 6, 12, 24), 7, None)


def attention_core(q, k, v, table, heads, mask, qk_scale=None):
    """WindowAttention.forward (:122-154) after its qkv projection; the window side is sqrt(N) of the N tokens per window"""
    B_, _, N, hd = q.shape
    ws = int(round(N ** 0.5))
    q = q * (hd ** -0.5 if qk_scale is None else qk_scale)
    attn = q @ k.transpose(-2, -1)
    bias = table[ts.rel_index(ws).view(-1).to(table.device)].view(N, N, -1).permute(2, 0, 1).contiguous()
    attn = attn + bias.unsqueeze(0)
    if mask is not None:
        nW = mask.shape[0]
        attn = attn.view(B_ // nW, nW, heads, N, N) + mask.unsqueeze(1).unsqueeze(0)
        attn = attn.view(-1, heads, N, N)
    attn = attn.softmax(-1)
    return (attn @ v).transpose(1, 2).reshape(B_, N, heads * hd)


def window_attention(qkv, h, w, heads, shift, table, ws, qk_scale=None):
    """(shifted) window attention of a window-padded qkv [B,Hp,Wp,3C] (q | k | v, heads x head_dim), at the original
    positions [B,h,w,C]: roll, partition, attention_core with the region mask, reverse, roll back, crop"""
    b, hp, wp, c3 = qkv.shape
    c = c3 // 3
    sx = torch.roll(qkv, shifts=(-shift, -shift), dims=(1, 2)) if shift else qkv
    xw = ts.window_partition(sx, ws).view(-1, ws * ws, c3)
    q, k, v = xw.reshape(-1, ws * ws, 3, heads, c // heads).permute(2, 0, 3, 1, 4)
    mask = ts.shift_mask(hp, wp, shift, qkv.device, ws).to(qkv.dtype) if shift else None
    aw = attention_core(q, k, v, table, heads, mask, qk_scale).view(-1, ws, ws, c)
    sx = ts.window_reverse(aw, ws, hp, wp)
    return (torch.roll(sx, shifts=(shift, shift), dims=(1, 2)) if shift else sx)[:, :h, :w]


def block(x, H, W, sd, p, heads, shift, ws, qk_scale=None):
    """SwinTransformerBlock.forward (:199-256)"""
    B, L, C = x.shape
    shortcut = x
    t = F.layer_norm(x, (C,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], 1e-5).view(B, H, W, C)
    t = F.pad(t, (0, 0, 0, (ws - W % ws) % ws, 0, (ws - H % ws) % ws))
    qkv = F.linear(t, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"])
    a = window_attention(qkv, H, W, heads, shift, sd[p + "attn.relative_position_bias_table"], ws, qk_scale)
    a = F.linear(a.reshape(B, H * W, C), sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
    x = shortcut + a
    y = F.layer_norm(x, (C,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], 1e-5)
    y = F.linear(F.gelu(F.linear(y, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"])), sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])
    return x + y


def swin_forward(sd, img, arch=SWIN_T):
    """arch = (embed_dim, depths, num_heads, window_size[, qk_scale]) (a swin.SwinArch fits) -> [C@1/8 (2E), C@1/16 (4E),
    C@1/32 (8E)] in NCHW"""
    embed, depths, heads_, ws, qk_scale = (tuple(arch) + (None,))[:5]
    _, _, H, W = img.shape
    if W % 4:
        img = F.pad(img, (0, 4 - W % 4))
    if H % 4:
        img = F.pad(img, (0, 0, 0, 4 - H % 4))
    x = F.conv2d(img, sd["backbone.patch_embed.proj.weight"], sd["backbone.patch_embed.proj.bias"], stride=4)
    Wh, Ww = x.shape[2], x.shape[3]
    x = x.flatten(2).transpose(1, 2)
    x = F.layer_norm(x, (embed,), sd["backbone.patch_embed.norm.weight"], sd["backbone.patch_embed.norm.bias"], 1e-5)
    outs = []
    for i, (depth, heads) in enumerate(zip(depths, heads_)):
        for j in range(depth):
            x = block(x, Wh, Ww, sd, "backbone.layers.%d.blocks.%d." % (i, j), heads, 0 if j % 2 == 0 else ws // 2, ws, qk_scale)
        if i in (1, 2, 3):
            C = embed << i
            o = F.layer_norm(x, (C,), sd["backbone.norm%d.weight" % i], sd["backbone.norm%d.bias" % i], 1e-5)
            outs.append(o.view(-1, Wh, Ww, C).permute(0, 3, 1, 2).contiguous())
        if i < 3:
            x = ts.patch_merging(x, Wh, Ww, sd, "backbone.layers.%d.downsample." % i)
            Wh, Ww = (Wh + 1) // 2, (Ww + 1) // 2
    return outs


swin_fpn = ts.swin_fpn
