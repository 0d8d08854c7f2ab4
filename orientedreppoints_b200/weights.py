"""State-dict layout and random initialisation of OrientedRepPointsDetector (R-50 / R-101 + FPN + head).

Key names follow the reference modules so published checkpoints load unchanged (SURVEY.md section 5):
  backbone.conv1.weight, backbone.bn1.*, backbone.layer{1..4}.{i}.conv{1,2,3}.weight / bn{1,2,3}.* /
  downsample.{0,1}.*            (mmdet/models/backbones/resnet.py:84-239, 345-515)
  neck.lateral_convs.{i}.{conv,gn}.*, neck.fpn_convs.{i}.{conv,gn}.*   (necks/fpn.py:88-128)
  bbox_head.{cls,reg}_convs.{i}.{conv,gn}.*, bbox_head.reppoints_*     (orientedreppoints_head.py:91-132)
Tensors are in the reference's layouts (conv weights [Cout, Cin, KH, KW]).
"""
import math

import torch

STAGE_BLOCKS = {50: (3, 4, 6, 3), 101: (3, 4, 23, 3)}


def _kaiming_fan_out(w, gen):
    # mmcv kaiming_init(mode='fan_out', nonlinearity='relu', distribution='normal') - resnet.py:443-454
    fan_out = w.shape[0] * w.shape[2] * w.shape[3]
    return w.normal_(0, math.sqrt(2.0 / fan_out), generator=gen)


def _xavier_uniform(w, gen):
    # fpn.py:132-135 xavier_init(distribution='uniform')
    fan_in = w.shape[1] * w.shape[2] * w.shape[3]
    fan_out = w.shape[0] * w.shape[2] * w.shape[3]
    a = math.sqrt(6.0 / (fan_in + fan_out))
    return w.uniform_(-a, a, generator=gen)


def dcn_layout(depth, dcn=None, stage_with_dcn=(False, False, False, False)):
    """what ResNet(depth, dcn=dcn, stage_with_dcn=...) builds as each block's conv2, per stage and block: None (nn.Conv2d),
    'DCN' or 'DCNv2'.  `fallback_on_stride` applies to the first block built from the dcn dict only (ResNet pops it from
    the dict all blocks share, resnet.py:146-147); `dcn` itself is left as it is."""
    fallback = bool(dcn.get('fallback_on_stride', False)) if dcn is not None else False
    layout = []
    for li, nblk in enumerate(STAGE_BLOCKS[depth]):
        stage = []
        for b in range(nblk):
            if dcn is None or not stage_with_dcn[li]:
                stage.append(None)
            else:
                stage.append(None if fallback else dcn['type'])
                fallback = False
        layout.append(tuple(stage))
    return tuple(layout)


def random_state_dict(depth=50, seed=0, reference_init=True, num_classes=16, feat=256, residual_gain=1.0, dcn=None,
                      stage_with_dcn=(False, False, False, False), dcn_offset_scale=0.0):
    """reference_init=True reproduces the reference's init_weights (incl. zero_init_residual and all-ones
    norm scales); False randomises norm parameters / running statistics so that every branch of the graph
    carries signal (used by the parity tests); residual_gain scales the randomised scale of every block's last norm
    (1.0 doubles the activation variance per block: fine for 16 blocks, ~1e5 after R-101's 33 - use 0.3 there).
    dcn / stage_with_dcn: the backbone's deformable conv2 layers as ResNet takes them (dcn_layout).  Their weights follow
    the reference (resnet.py:474-484): DeformConv.reset_parameters' uniform +-1/sqrt(9 planes) (kaiming_init skips a layer
    that is not an nn.Conv2d; with reference_init=False the kaiming draw of a plain conv2 instead) and an all-zero
    conv_offset.  dcn_offset_scale > 0 (tests only) draws conv_offset from N(0, scale^2 / fan_in) with N(0, scale^2) biases
    instead, so that the samples leave the grid by about `scale` pixels per unit of input and the DCNv2 mask logits vary;
    with zero offsets a deformable layer is a plain convolution."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    layout = dcn_layout(depth, dcn, stage_with_dcn)

    def conv(name, cout, cin, k, init, bias=False, std=0.01):
        w = torch.empty(cout, cin, k, k)
        if init == "kaiming":
            _kaiming_fan_out(w, g)
        elif init == "xavier":
            _xavier_uniform(w, g)
        else:
            w.normal_(0, std, generator=g)
        sd[name + ".weight"] = w
        if bias:
            sd[name + ".bias"] = torch.zeros(cout)

    def norm(name, c, running, zero_gamma=False):
        if reference_init:
            sd[name + ".weight"] = torch.zeros(c) if zero_gamma else torch.ones(c)
            sd[name + ".bias"] = torch.zeros(c)
            if running:
                sd[name + ".running_mean"] = torch.zeros(c)
                sd[name + ".running_var"] = torch.ones(c)
        else:
            sd[name + ".weight"] = torch.empty(c).uniform_(0.5, 1.5, generator=g) * (residual_gain if zero_gamma else 1.0)
            sd[name + ".bias"] = torch.empty(c).normal_(0, 0.1, generator=g)
            if running:
                sd[name + ".running_mean"] = torch.empty(c).normal_(0, 0.1, generator=g)
                sd[name + ".running_var"] = torch.empty(c).uniform_(0.5, 1.5, generator=g)

    # ---------------------------------------------------------------- backbone (resnet.py)
    conv("backbone.conv1", 64, 3, 7, "kaiming")
    norm("backbone.bn1", 64, True)
    inplanes = 64
    for li, (nblk, planes) in enumerate(zip(STAGE_BLOCKS[depth], (64, 128, 256, 512))):
        for b in range(nblk):
            p = "backbone.layer%d.%d" % (li + 1, b)
            conv(p + ".conv1", planes, inplanes, 1, "kaiming")
            norm(p + ".bn1", planes, True)
            kind = layout[li][b]
            if kind is None:
                conv(p + ".conv2", planes, planes, 3, "kaiming")
            else:
                if reference_init:
                    bound = 1.0 / math.sqrt(9 * planes)
                    sd[p + ".conv2.weight"] = torch.empty(planes, planes, 3, 3).uniform_(-bound, bound, generator=g)
                else:
                    conv(p + ".conv2", planes, planes, 3, "kaiming")
                co = 27 if kind == 'DCNv2' else 18
                w, bias = torch.zeros(co, planes, 3, 3), torch.zeros(co)
                if dcn_offset_scale > 0:
                    w.normal_(0, dcn_offset_scale / math.sqrt(9 * planes), generator=g)
                    bias.normal_(0, dcn_offset_scale, generator=g)
                sd[p + ".conv2.conv_offset.weight"], sd[p + ".conv2.conv_offset.bias"] = w, bias
            norm(p + ".bn2", planes, True)
            conv(p + ".conv3", planes * 4, planes, 1, "kaiming")
            norm(p + ".bn3", planes * 4, True, zero_gamma=True)           # zero_init_residual, resnet.py:486-491
            if b == 0:
                conv(p + ".downsample.0", planes * 4, inplanes, 1, "kaiming")
                norm(p + ".downsample.1", planes * 4, True)
            inplanes = planes * 4
    # ---------------------------------------------------------------- neck (fpn.py, start_level=1, 5 outs)
    for i, cin in enumerate((512, 1024, 2048)):
        conv("neck.lateral_convs.%d.conv" % i, feat, cin, 1, "xavier")
        norm("neck.lateral_convs.%d.gn" % i, feat, False)
        conv("neck.fpn_convs.%d.conv" % i, feat, feat, 3, "xavier")
        norm("neck.fpn_convs.%d.gn" % i, feat, False)
    conv("neck.fpn_convs.3.conv", feat, 2048, 3, "xavier")                 # extra_convs_on_inputs: on C5
    norm("neck.fpn_convs.3.gn", feat, False)
    conv("neck.fpn_convs.4.conv", feat, feat, 3, "xavier")
    norm("neck.fpn_convs.4.gn", feat, False)
    # ---------------------------------------------------------------- head (orientedreppoints_head.py:134-146)
    std = 0.01 if reference_init else 0.03
    for i in range(3):
        conv("bbox_head.cls_convs.%d.conv" % i, feat, feat, 3, "normal", std=std)
        norm("bbox_head.cls_convs.%d.gn" % i, feat, False)
        conv("bbox_head.reg_convs.%d.conv" % i, feat, feat, 3, "normal", std=std)
        norm("bbox_head.reg_convs.%d.gn" % i, feat, False)
    conv("bbox_head.reppoints_cls_conv", feat, feat, 3, "normal", std=std)                 # DeformConv, no bias
    conv("bbox_head.reppoints_cls_out", num_classes - 1, feat, 1, "normal", bias=True, std=std)
    sd["bbox_head.reppoints_cls_out.bias"].fill_(-math.log((1 - 0.01) / 0.01))            # bias_init_with_prob(0.01)
    conv("bbox_head.reppoints_pts_init_conv", feat, feat, 3, "normal", bias=True, std=std)
    conv("bbox_head.reppoints_pts_init_out", 18, feat, 1, "normal", bias=True, std=std)
    conv("bbox_head.reppoints_pts_refine_conv", feat, feat, 3, "normal", std=std)          # DeformConv, no bias
    conv("bbox_head.reppoints_pts_refine_out", 18, feat, 1, "normal", bias=True, std=std)
    if not reference_init:
        for k in list(sd):
            if k.endswith("_out.bias") or k.endswith("init_conv.bias"):
                sd[k] = sd[k] + torch.empty_like(sd[k]).normal_(0, 0.1, generator=g)
        # spread the predicted points so that the deformable sampling actually leaves the 3x3 grid
        sd["bbox_head.reppoints_pts_init_out.bias"] += torch.empty(18).uniform_(-1.5, 1.5, generator=g)
    return sd


def fold_bn(w, bn_w, bn_b, mean, var, eps=1e-5):
    """eval-mode BatchNorm folded into the preceding bias-free conv - the reference-sanctioned fold of
    tools/fuse_conv_bn.py:10-24.  Returns (w', b')."""
    factor = bn_w / torch.sqrt(var + eps)
    return w * factor.reshape(-1, 1, 1, 1), bn_b - mean * factor
