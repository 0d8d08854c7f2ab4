"""fp64 restatement of the FPN_CARAFE neck (mmdet/models/necks/fpn_carafe.py) and CARAFEPack (mmdet/ops/carafe/carafe.py)
on NCHW torch tensors, checked against the reference's own modules by tests/test_fpn_carafe_cpu.py.  TEST INFRASTRUCTURE."""
import torch
import torch.nn.functional as F


def carafe(x, logits, k, group):
    """CARAFEPack.kernel_normalizer + carafe with scale factor 2: x [N, C, H, W], the encoder's logits [N, k^2 * G * 4, H, W]
    -> [N, C, 2H, 2W].  Taps outside x contribute zero (unfold's padding): the softmax is not renormalised over them"""
    n, c, h, w = x.shape
    mask = F.softmax(F.pixel_shuffle(logits, 2).view(n, group, k * k, 2 * h, 2 * w), dim=2)
    cols = F.unfold(x, k, padding=(k - 1) // 2).view(n, c, k * k, h, w)
    cols = cols.repeat_interleave(2, dim=3).repeat_interleave(2, dim=4)              # the window of (oy / 2, ox / 2)
    return (cols.view(n, group, c // group, k * k, 2 * h, 2 * w) * mask.unsqueeze(2)).sum(3).view(n, c, 2 * h, 2 * w)


def carafe_add(x, logits, k, group, residual):
    """residual + carafe(x, ...) cut to the residual's extent (fpn_carafe.py tensor_add / slice_as)"""
    up = carafe(x, logits, k, group)
    return residual + up[:, :, :residual.shape[2], :residual.shape[3]]


def conv_module(x, sd, p, stride, pad, spec):
    """a ConvModule of the neck: conv (+ bias without a norm) (+ GroupNorm(32)) (+ ReLU)"""
    y = F.conv2d(x, sd[p + '.conv.weight'], sd.get(p + '.conv.bias'), stride, pad)
    if spec['norm'] == 'GN':
        y = F.group_norm(y, 32, sd[p + '.gn.weight'], sd[p + '.gn.bias'], 1e-5)
    return F.relu(y) if spec['relu'] else y


def upsample_logits(x, sd, j, spec):
    """CARAFEPack_j's channel_compressor + content_encoder on x"""
    p = 'neck.upsample_modules.%d.' % j
    comp = F.conv2d(x, sd[p + 'channel_compressor.weight'], sd[p + 'channel_compressor.bias'])
    return F.conv2d(comp, sd[p + 'content_encoder.weight'], sd[p + 'content_encoder.bias'], padding=(spec['encoder_kernel'] - 1) // 2)


def neck(sd, spec, feats):
    """the five levels from the backbone's stride-8, -16 and -32 outputs feats (NCHW), every tensor float64"""
    lats = [conv_module(f, sd, 'neck.lateral_convs.%d' % i, 1, 0, spec) for i, f in enumerate(feats)]
    lats.append(conv_module(feats[-1], sd, 'neck.lateral_convs.3', 2, 1, spec))
    lats.append(conv_module(lats[-1], sd, 'neck.lateral_convs.4', 2, 1, spec))
    for i in range(4, 0, -1):
        lats[i - 1] = carafe_add(lats[i], upsample_logits(lats[i], sd, i - 1, spec), spec['up_kernel'], spec['up_group'],
                                 lats[i - 1])
    return [conv_module(x, sd, 'neck.fpn_convs.%d' % i, 1, 1, spec) for i, x in enumerate(lats)]


def level_sizes(h, w):
    """(H, W) of the five levels for backbone outputs of strides 8, 16, 32 at ceil-halving, then the two 3x3 / s2 extras"""
    s = [h, w]
    out = []
    for _ in range(3):
        s = [-(-v // 2) for v in s] if out else [-(-v // 8) for v in s]
        out.append(tuple(s))
    for _ in range(2):
        s = [(v - 1) // 2 + 1 for v in s]
        out.append(tuple(s))
    return out


# golden cases (tests/golden/gen_golden_fpn_carafe.py): R-50- and Swin-T-shaped inputs at 1024-like level sizes (every
# upsampled map fits) and 960-like ones (stride-8 30x30 at 240^2: the 8 -> 16 map is cut to 15, then 15 -> 30)
R50_WIDTHS, SWIN_T_WIDTHS = (256, 512, 1024, 2048), (192, 384, 768)
CASES = [
    dict(tag="r50_1024_k5g1_gn", widths=R50_WIDTHS, start_level=1, hw=(256, 256), norm=True, relu=False, k=5, g=1, ek=3, cc=64, seed=1),
    dict(tag="r50_960_k5g1_gn", widths=R50_WIDTHS, start_level=1, hw=(240, 240), norm=True, relu=False, k=5, g=1, ek=3, cc=64, seed=2),
    dict(tag="r50_960_k3g4_relu", widths=R50_WIDTHS, start_level=1, hw=(240, 256), norm=False, relu=True, k=3, g=4, ek=3, cc=64, seed=3),
    dict(tag="r50_1024_k7g1_gn_relu", widths=R50_WIDTHS, start_level=1, hw=(256, 256), norm=True, relu=True, k=7, g=1, ek=1, cc=32, seed=4),
    dict(tag="swin_1024_k7g4", widths=SWIN_T_WIDTHS, start_level=0, hw=(256, 256), norm=False, relu=False, k=7, g=4, ek=3, cc=64, seed=5),
    dict(tag="swin_960_k3g1_gn", widths=SWIN_T_WIDTHS, start_level=0, hw=(240, 240), norm=True, relu=False, k=3, g=1, ek=3, cc=64, seed=6),
    dict(tag="swin_960_k5g4_gn_relu", widths=SWIN_T_WIDTHS, start_level=0, hw=(240, 240), norm=True, relu=True, k=5, g=4, ek=1, cc=16, seed=7),
]
OUT_CHANNELS = 8
CARAFE_GAIN = 3.0


def neck_cfg(case):
    """the config dict of a case's neck"""
    return dict(type='FPN_CARAFE', in_channels=list(case["widths"]), out_channels=256, num_outs=5, start_level=case["start_level"],
                norm_cfg=dict(type='GN', num_groups=32, requires_grad=True) if case["norm"] else None,
                act_cfg=dict(type='ReLU') if case["relu"] else None,
                upsample_cfg=dict(type='carafe', up_kernel=case["k"], up_group=case["g"], encoder_kernel=case["ek"],
                                  encoder_dilation=1, compressed_channels=case["cc"]))


def spec_of(case):
    from orientedreppoints_b200.weights import fpn_carafe_spec
    c = neck_cfg(case)
    return fpn_carafe_spec(c["in_channels"][c["start_level"]:], 256, c["norm_cfg"], c["act_cfg"], upsample_cfg=c["upsample_cfg"])


def weights(case):
    """the case's neck.* tensors (float32 draws)"""
    from orientedreppoints_b200.weights import _draw_fpn_carafe
    sd = {}
    _draw_fpn_carafe(sd, torch.Generator().manual_seed(case["seed"]), spec_of(case), False, CARAFE_GAIN)
    return sd


def inputs(case, dtype=torch.float64):
    """the backbone's stride-8, -16 and -32 outputs of the case (N = 1)"""
    g = torch.Generator().manual_seed(100 + case["seed"])
    sizes = level_sizes(*case["hw"])[:3]
    return [torch.randn((1, c, h, w), generator=g, dtype=torch.float64).to(dtype)
            for c, (h, w) in zip(case["widths"][-3:], sizes)]
