"""fp64 evaluation of the dense graph with deformable backbone layers (test infrastructure): the ResNet of
oracle/torch_reference.py with each block's conv2 as models.ResNet builds it for a dcn / stage_with_dcn configuration
(mmdet/models/backbones/resnet.py:146-168) - DeformConvPack (deform_conv.py:258-323) or ModulatedDeformConvPack
(:377-446): conv_offset, then deform_conv_ref, the fp64 deformable convolution pinned to the reference's own im2col
kernels.  FPN and head are oracle/torch_reference.py's."""
import torch
import torch.nn.functional as F

from oracle import torch_reference as tr

# the deformable conv2 launches of a ResNet with DCN in a stage, for 1024 x 1024 tiles: (planes = Cin = Cout, input H = W,
# stride).  The first block of layer2-4 has stride 2; input sizes halve for 512 x 512 tiles.
LAUNCHES_1024 = [(64, 256, 1), (128, 256, 2), (128, 128, 1), (256, 128, 2), (256, 64, 1), (512, 64, 2), (512, 32, 1)]
# the batches those launches run at: one 1024 tile, the benchmark's 16 tiles, two 512 tiles
BATCHES = [(1, 1024), (16, 1024), (2, 512)]


def conv2_ref(sd, p, x, stride, kind):
    """conv2 of block `p` (no norm): plain (kind None), DCN or DCNv2"""
    w = sd[p + ".conv2.weight"]
    if kind is None:
        return F.conv2d(x, w, None, stride, 1)
    om = F.conv2d(x, sd[p + ".conv2.conv_offset.weight"], sd[p + ".conv2.conv_offset.bias"], stride, 1)
    if kind == 'DCN':
        return tr.deform_conv_ref(x, om, w, stride, 1)
    o1, o2, m = torch.chunk(om, 3, dim=1)
    return tr.deform_conv_ref(x, torch.cat((o1, o2), dim=1), w, stride, 1, mask=torch.sigmoid(m))


def backbone(sd, img, layout, blocks=(3, 4, 6, 3)):
    """layout: per stage and block None / 'DCN' / 'DCNv2' (weights.dcn_layout)"""
    x = F.relu(tr._bn(F.conv2d(img, sd["backbone.conv1.weight"], None, 2, 3), sd, "backbone.bn1"))
    x = F.max_pool2d(x, 3, 2, 1)
    outs = []
    for li, nblk in enumerate(blocks):
        for b in range(nblk):
            p = "backbone.layer%d.%d" % (li + 1, b)
            s = 2 if (b == 0 and li > 0) else 1
            idt = x
            o = F.relu(tr._bn(F.conv2d(x, sd[p + ".conv1.weight"]), sd, p + ".bn1"))
            o = F.relu(tr._bn(conv2_ref(sd, p, o, s, layout[li][b]), sd, p + ".bn2"))
            o = tr._bn(F.conv2d(o, sd[p + ".conv3.weight"]), sd, p + ".bn3")
            if b == 0:
                idt = tr._bn(F.conv2d(x, sd[p + ".downsample.0.weight"], None, s), sd, p + ".downsample.1")
            x = F.relu(o + idt)
        outs.append(x)
    return outs


def forward_dense(sd, img, layout, blocks=(3, 4, 6, 3)):
    """per level (cls_out, pts_init, pts_refine) in NCHW, and the FPN levels"""
    feats = tr.fpn(sd, backbone(sd, img, layout, blocks))
    return [tr.head_single(sd, f)[:3] for f in feats], feats
