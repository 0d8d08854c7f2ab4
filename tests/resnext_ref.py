"""fp64 evaluation of the dense graph with a ResNeXt backbone (test infrastructure): the bottleneck of resnext.py:11-70 -
conv1 / conv2 `width` wide, conv2 = F.conv2d(..., groups=groups) - with oracle/torch_reference.py's FPN and head."""
import torch.nn.functional as F

from oracle import torch_reference as tr
from orientedreppoints_b200.weights import STAGE_BLOCKS, block_width

# the published models: (name, depth, groups, base_width)
MODELS = [("X-50-32x4d", 50, 32, 4), ("X-101-32x4d", 101, 32, 4), ("X-101-64x4d", 101, 64, 4), ("X-50-32x8d", 50, 32, 8),
          ("X-152-32x4d", 152, 32, 4), ("X-152-64x4d", 152, 64, 4), ("X-152-32x8d", 152, 32, 8)]
# the batches grouped launches are planned / tested at: one 1024 tile, the benchmark's 16 tiles, two 512 tiles
BATCHES = [(1, 1024), (16, 1024), (2, 512)]


def group_launches(groups, base_width, tile=1024):
    """the distinct grouped conv2 launches of a ResNeXt on tile x tile input: (width, groups, input H = W, stride).  The first
    block of layer2-4 has stride 2 on the previous stage's map"""
    out = []
    for li in range(4):
        width = block_width(64 << li, groups, base_width)
        h = tile // (4 << li)
        if li > 0:
            out.append((width, groups, 2 * h, 2))
        out.append((width, groups, h, 1))
    return out


def backbone(sd, img, depth, groups):
    x = F.relu(tr._bn(F.conv2d(img, sd["backbone.conv1.weight"], None, 2, 3), sd, "backbone.bn1"))
    x = F.max_pool2d(x, 3, 2, 1)
    outs = []
    for li, nblk in enumerate(STAGE_BLOCKS[depth]):
        for b in range(nblk):
            p = "backbone.layer%d.%d" % (li + 1, b)
            s = 2 if (b == 0 and li > 0) else 1
            idt = x
            o = F.relu(tr._bn(F.conv2d(x, sd[p + ".conv1.weight"]), sd, p + ".bn1"))
            o = F.relu(tr._bn(F.conv2d(o, sd[p + ".conv2.weight"], None, s, 1, groups=groups), sd, p + ".bn2"))
            o = tr._bn(F.conv2d(o, sd[p + ".conv3.weight"]), sd, p + ".bn3")
            if b == 0:
                idt = tr._bn(F.conv2d(x, sd[p + ".downsample.0.weight"], None, s), sd, p + ".downsample.1")
            x = F.relu(o + idt)
        outs.append(x)
    return outs


def forward_dense(sd, img, depth, groups):
    """per level (cls_out, pts_init, pts_refine) in NCHW, and the FPN levels"""
    feats = tr.fpn(sd, backbone(sd, img, depth, groups))
    return [tr.head_single(sd, f)[:3] for f in feats], feats
