"""fp64 evaluation of ResNet backbones with generalized attention blocks (test infrastructure): the block of
mmdet/ops/generalized_attention.py restated from its formula (energy = Qc . K + Qp . (Px + Py), softmax over the keys, V,
proj_conv, gamma * out + x), materialised per image, and the ResNet of tests/dcn_backbone_ref.py with the block after
relu(bn2(conv2)) (resnet.py:216-217).  Checked against the reference's own module through tests/golden/gen_attention_ref.npz."""
import torch
import torch.nn.functional as F

from oracle import torch_reference as tr
from orientedreppoints_b200.gen_attention import position_table
from orientedreppoints_b200.weights import STAGE_BLOCKS
import dcn_backbone_ref as dr

# the published settings (mmdetection's empirical-attention configs) on R-50: c4-c5 blocks
PUBLISHED = dict(spatial_range=-1, num_heads=8, kv_stride=2)
PUBLISHED_STAGES = [[], [], [0, 1, 2, 3, 4, 5], [0, 1, 2]]


def qkv(blk, spec, x):
    """(Qc or None, Qp or None, K or None, V) of the block on x [N, C, H, W] as [N, heads, tokens, d]"""
    t, s, heads = spec['attention_type'], spec['kv_stride'], spec['num_heads']
    n, c, h, w = x.shape
    d = c // heads
    xk = x[:, :, ::s, ::s]

    def tok(y):
        return y.reshape(y.shape[0], heads, d, -1).transpose(2, 3)

    q = tok(F.conv2d(x, blk['query_conv.weight'])) if (t[0] or t[1]) else None
    k = tok(F.conv2d(xk, blk['key_conv.weight'])) if (t[0] or t[2]) else None
    v = tok(F.conv2d(xk, blk['value_conv.weight']))
    zero = torch.zeros(n, heads, h * w, d, dtype=x.dtype)
    qc = qp = None
    if t[0] or t[2]:
        qc = (q if t[0] else zero) + (blk['appr_bias'].reshape(1, heads, 1, d) if t[2] else 0)
    if t[1] or t[3]:
        qp = (q if t[1] else zero) + (blk['geom_bias'].reshape(1, heads, 1, d) if t[3] else 0)
    return qc, qp, k, v


def energy(spec, blk, qc, qp, k, h, w, hk, wk):
    """[N, heads, H W, Hk Wk] fp64"""
    heads = spec['num_heads']
    s = spec['kv_stride']
    ref = qc if qc is not None else qp
    n, _, _, d = ref.shape if ref is not None else (1, heads, h * w, 1)
    e = torch.zeros(n, heads, h * w, hk * wk, dtype=torch.float64)
    if qc is not None:
        e = e + qc @ k.transpose(2, 3)
    if qp is not None:
        px = position_table(spec, blk['appr_geom_fc_x.weight'], w, wk).reshape(-1, heads, d)     # [Rx, heads, d]
        py = position_table(spec, blk['appr_geom_fc_y.weight'], h, hk).reshape(-1, heads, d)
        qx, qy = torch.arange(w), torch.arange(h)
        ix = qx[:, None] - s * torch.arange(wk)[None, :] + s * (wk - 1)                         # [W, Wk] table rows
        iy = qy[:, None] - s * torch.arange(hk)[None, :] + s * (hk - 1)
        fx = px[ix].permute(2, 0, 1, 3)                                                         # [heads, W, Wk, d]
        fy = py[iy].permute(2, 0, 1, 3)
        q5 = qp.reshape(qp.shape[0], heads, h, w, d)
        ex = torch.einsum('nhyxd,hxkd->nhyxk', q5, fx)                                          # [N, heads, H, W, Wk]
        ey = torch.einsum('nhyxd,hykd->nhyxk', q5, fy)                                          # [N, heads, H, W, Hk]
        e = e + (ey[..., :, None] + ex[..., None, :]).reshape(qp.shape[0], heads, h * w, hk * wk)
    return e


def attention_core(spec, blk, x):
    """softmax(energy) V of the block on x, [N, C, H, W] before proj_conv (for '0010' alone: [N, C, 1, 1], the reference's
    one-row shortcut)"""
    t = spec['attention_type']
    n, c, h, w = x.shape
    s = spec['kv_stride']
    hk, wk = -(-h // s), -(-w // s)
    qc, qp, k, v = qkv(blk, spec, x)
    if t == (False, False, True, False):
        qc, h, w = qc[:, :, :1], 1, 1
    e = energy(spec, blk, qc, qp, k, h, w, hk, wk)
    o = torch.softmax(e, -1) @ v                                                                # [N, heads, H W, d]
    return o.transpose(2, 3).reshape(n, c, h, w)


def block(spec, blk, x):
    """gen_attention_block(x): gamma * proj_conv(attention) + x"""
    o = F.conv2d(attention_core(spec, blk, x), blk['proj_conv.weight'], blk['proj_conv.bias'])
    return blk['gamma'] * o + x


def block_params(sd, p):
    pre = p + '.gen_attention_block.'
    return {k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}


def backbone(sd, img, layout, ga_layout, depth=50):
    """C2..C5 of the ResNet with deformable conv2 per `layout` (None / 'DCN' / 'DCNv2') and attention per ga_layout"""
    x = F.relu(tr._bn(F.conv2d(img, sd["backbone.conv1.weight"], None, 2, 3), sd, "backbone.bn1"))
    x = F.max_pool2d(x, 3, 2, 1)
    outs = []
    for li, nblk in enumerate(STAGE_BLOCKS[depth]):
        for b in range(nblk):
            p = "backbone.layer%d.%d" % (li + 1, b)
            s = 2 if (b == 0 and li > 0) else 1
            o = F.relu(tr._bn(F.conv2d(x, sd[p + ".conv1.weight"]), sd, p + ".bn1"))
            o = F.relu(tr._bn(dr.conv2_ref(sd, p, o, s, layout[li][b] if layout else None), sd, p + ".bn2"))
            if ga_layout[li][b] is not None:
                o = block(ga_layout[li][b], block_params(sd, p), o)
            o = tr._bn(F.conv2d(o, sd[p + ".conv3.weight"]), sd, p + ".bn3")
            idt = tr._bn(F.conv2d(x, sd[p + ".downsample.0.weight"], None, s), sd, p + ".downsample.1") if b == 0 else x
            x = F.relu(o + idt)
        outs.append(x)
    return outs


def forward_dense(sd, img, layout, ga_layout, depth=50):
    """per level (cls_out, pts_init, pts_refine) in NCHW, and the FPN levels"""
    feats = tr.fpn(sd, backbone(sd, img, layout, ga_layout, depth))
    return [tr.head_single(sd, f)[:3] for f in feats], feats
