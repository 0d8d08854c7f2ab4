"""fp64 evaluation of ResNet / ResNeXt backbones with global context blocks (test infrastructure): the block of
mmdet/ops/context_block.py restated from its formula (softmax over all pixels of conv_mask(x) or the mean, then
channel_mul_conv / channel_add_conv: 1x1, LayerNorm over the P planes, ReLU, 1x1), and the bottleneck of resnet.py:203-239 with
the block on bn3(conv3(.)) before the residual add - with a grouped conv2 (resnext_ref), deformable conv2 (dcn_backbone_ref)
and attention blocks (gen_attention_ref) as the layouts say.  Checked against the reference's own modules through
tests/golden/context_block_ref.npz."""
import torch
import torch.nn.functional as F

from oracle import torch_reference as tr
from orientedreppoints_b200.weights import STAGE_BLOCKS
import dcn_backbone_ref as dr
import gen_attention_ref as gr

C3_C5 = (False, True, True, True)


def context(spec, p, x):
    """the pooled context [N, C] of x [N, C, H, W]: softmax-weighted ('att', conv_mask's bias included) or the mean"""
    n, c, h, w = x.shape
    if spec['pooling_type'] == 'avg':
        return x.mean((2, 3))
    logit = F.conv2d(x, p['conv_mask.weight'], p['conv_mask.bias']).reshape(n, h * w)
    return torch.einsum('nck,nk->nc', x.reshape(n, c, h * w), torch.softmax(logit, 1))


def mlp(p, f, ctx):
    """channel_{add,mul}_conv on ctx [N, C]: [N, C]"""
    t = ctx @ p[f + '_conv.0.weight'].flatten(1).t() + p[f + '_conv.0.bias']
    mean, var = t.mean(1, keepdim=True), t.var(1, unbiased=False, keepdim=True)
    t = (t - mean) / torch.sqrt(var + 1e-5) * p[f + '_conv.1.weight'].reshape(1, -1) + p[f + '_conv.1.bias'].reshape(1, -1)
    return F.relu(t) @ p[f + '_conv.3.weight'].flatten(1).t() + p[f + '_conv.3.bias']


def terms(spec, p, x):
    """(mul or None, add or None), fp [N, C]: sigmoid(channel_mul_conv(ctx)) and channel_add_conv(ctx)"""
    ctx = context(spec, p, x)
    mul = torch.sigmoid(mlp(p, 'channel_mul', ctx)) if 'channel_mul' in spec['fusion_types'] else None
    add = mlp(p, 'channel_add', ctx) if 'channel_add' in spec['fusion_types'] else None
    return mul, add


def block(spec, p, x):
    """context_block(x): x * mul + add, without the residual"""
    mul, add = terms(spec, p, x)
    out = x if mul is None else x * mul[:, :, None, None]
    return out if add is None else out + add[:, :, None, None]


def block_params(sd, p):
    pre = p + '.context_block.'
    return {k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}


def backbone(sd, img, gcb_layout, depth=50, groups=1, dcn_layout=None, ga_layout=None):
    """C2..C5 of the ResNet / ResNeXt with context blocks per gcb_layout"""
    x = F.relu(tr._bn(F.conv2d(img, sd["backbone.conv1.weight"], None, 2, 3), sd, "backbone.bn1"))
    x = F.max_pool2d(x, 3, 2, 1)
    outs = []
    for li, nblk in enumerate(STAGE_BLOCKS[depth]):
        for b in range(nblk):
            p = "backbone.layer%d.%d" % (li + 1, b)
            s = 2 if (b == 0 and li > 0) else 1
            o = F.relu(tr._bn(F.conv2d(x, sd[p + ".conv1.weight"]), sd, p + ".bn1"))
            if groups > 1:
                o = F.conv2d(o, sd[p + ".conv2.weight"], None, s, 1, groups=groups)
            else:
                o = dr.conv2_ref(sd, p, o, s, dcn_layout[li][b] if dcn_layout else None)
            o = F.relu(tr._bn(o, sd, p + ".bn2"))
            if ga_layout and ga_layout[li][b] is not None:
                o = gr.block(ga_layout[li][b], gr.block_params(sd, p), o)
            o = tr._bn(F.conv2d(o, sd[p + ".conv3.weight"]), sd, p + ".bn3")
            if gcb_layout[li][b] is not None:
                o = block(gcb_layout[li][b], block_params(sd, p), o)
            idt = tr._bn(F.conv2d(x, sd[p + ".downsample.0.weight"], None, s), sd, p + ".downsample.1") if b == 0 else x
            x = F.relu(o + idt)
        outs.append(x)
    return outs


def forward_dense(sd, img, gcb_layout, depth=50, groups=1, dcn_layout=None, ga_layout=None):
    """per level (cls_out, pts_init, pts_refine) in NCHW, and the FPN levels"""
    feats = tr.fpn(sd, backbone(sd, img, gcb_layout, depth, groups, dcn_layout, ga_layout))
    return [tr.head_single(sd, f)[:3] for f in feats], feats
