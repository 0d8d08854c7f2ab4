"""State-dict layout and random initialisation of OrientedRepPointsDetector (R-50 / R-101 / R-152 or ResNeXt + FPN + head;
HRNet + HRFPN + head in random_hrnet_state_dict, keys as mmdet/models/backbones/hrnet.py and necks/hrfpn.py name them).

Key names follow the reference modules so published checkpoints load unchanged (SURVEY.md section 5):
  backbone.conv1.weight, backbone.bn1.*, backbone.layer{1..4}.{i}.conv{1,2,3}.weight / bn{1,2,3}.* /
  downsample.{0,1}.*            (mmdet/models/backbones/resnet.py:84-239, 345-515; ResNeXt: resnext.py:11-70, the same
                                 keys with conv1 / conv2 / bn1 / bn2 `width` wide and conv2 grouped)
  neck.lateral_convs.{i}.{conv,gn}.*, neck.fpn_convs.{i}.{conv,gn}.*   (necks/fpn.py:88-128)
  or, for FPN_CARAFE, neck.lateral_convs.{0..4}.*, neck.fpn_convs.{0..4}.*, neck.upsample_modules.{0..3}.{channel_compressor,
  content_encoder}.*                                                   (necks/fpn_carafe.py:34-200, ops/carafe/carafe.py:161-214)
  bbox_head.{cls,reg}_convs.{i}.{conv,gn}.*, bbox_head.reppoints_*     (orientedreppoints_head.py:91-132)
Tensors are in the reference's layouts (conv weights [Cout, Cin, KH, KW]).
"""
import math

import torch

STAGE_BLOCKS = {50: (3, 4, 6, 3), 101: (3, 4, 23, 3), 152: (3, 8, 36, 3)}
# group widths (channels per group of conv2) the grouped kernels are built for: those of ResNeXt 32x4d, 64x4d and 32x8d
GROUP_WIDTHS = (4, 8, 16, 32, 64)


def block_width(planes, groups=1, base_width=4):
    """the bottleneck width of resnext.py:20-23: planes for groups == 1, else floor(planes * base_width / 64) * groups"""
    return planes if groups == 1 else math.floor(planes * (base_width / 64)) * groups


def check_groups(groups, base_width):
    """NotImplementedError unless every stage's conv2 is one the grouped kernels run: width a multiple of 64 and a group width
    in GROUP_WIDTHS (groups == 1 is a ResNet and always passes)"""
    if groups == 1:
        return
    if not isinstance(groups, int) or groups < 1:
        raise NotImplementedError("groups=%r: ResNeXt needs a positive integer number of groups" % (groups,))
    for planes in (64, 128, 256, 512):
        width = block_width(planes, groups, base_width)
        if width % 64:
            raise NotImplementedError("groups=%d, base_width=%r give a conv2 width of %d at planes=%d: liborp_b200 runs grouped "
                                      "convolutions whose width is a multiple of 64" % (groups, base_width, width, planes))
        if width // groups not in GROUP_WIDTHS:
            raise NotImplementedError("groups=%d, base_width=%r give %d channels per group at planes=%d: liborp_b200 runs group "
                                      "widths %s" % (groups, base_width, width // groups, planes, GROUP_WIDTHS))


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


# GeneralizedAttention's arguments and their defaults (generalized_attention.py:34-42)
GEN_ATTENTION_DEFAULTS = dict(spatial_range=-1, num_heads=9, position_embedding_dim=-1, position_magnitude=1, kv_stride=2,
                              q_stride=1, attention_type='1111')


def gen_attention_spec(cfg, planes):
    """the block that GeneralizedAttention(planes, **cfg) builds, as the engine runs it: dict(attention_type (four bools),
    num_heads, head_dim, kv_stride, position_embedding_dim, position_magnitude, channels).  NotImplementedError for what the
    kernels do not run (spatial_range >= 0, q_stride != 1, kv_stride other than 1 or 2, planes % num_heads, a head dimension
    other than 32 or 64), ValueError where the reference itself fails (an attention_type that is not four 0/1 digits, a position
    embedding that is not a positive multiple of 4 when the position terms use it), TypeError for an unknown argument"""
    unknown = sorted(set(cfg) - set(GEN_ATTENTION_DEFAULTS))
    if unknown:
        raise TypeError("GeneralizedAttention got unexpected arguments %s" % unknown)
    a = dict(GEN_ATTENTION_DEFAULTS, **cfg)
    t = a['attention_type']
    if not isinstance(t, str) or len(t) != 4 or any(ch not in '01' for ch in t):
        raise ValueError("attention_type=%r: generalized_attention.py reads four 0/1 digits" % (t,))
    t = tuple(ch == '1' for ch in t)
    if t[1] and not t[3]:
        raise NotImplementedError("gen_attention with attention_type=%r: without the geom_bias term the reference's query-position "
                                  "branch (generalized_attention.py:308-326) pairs the y-offset features with the query at the "
                                  "transposed position and fails on maps that are not square; liborp_b200 runs the '0100' term "
                                  "together with '0001' only" % (a['attention_type'],))
    if a['spatial_range'] >= 0:
        raise NotImplementedError("gen_attention with spatial_range=%r: the reference's local mask is hard-coded for 256 / 512 "
                                  "channels and maps up to 84 / 42; liborp_b200 runs spatial_range=-1" % (a['spatial_range'],))
    if a['q_stride'] != 1:
        raise NotImplementedError("gen_attention with q_stride=%r: liborp_b200 runs q_stride=1" % (a['q_stride'],))
    if a['kv_stride'] not in (1, 2):
        raise NotImplementedError("gen_attention with kv_stride=%r: liborp_b200 runs kv_stride 1 or 2" % (a['kv_stride'],))
    heads = a['num_heads']
    if not isinstance(heads, int) or heads < 1:
        raise ValueError("gen_attention with num_heads=%r: needs a positive integer" % (heads,))
    if planes % heads or planes // heads not in (32, 64):
        raise NotImplementedError("gen_attention with num_heads=%d on %d channels: liborp_b200 runs head dimensions "
                                  "(channels / num_heads) of 32 and 64 that divide the channels" % (heads, planes))
    e = a['position_embedding_dim'] if a['position_embedding_dim'] > 0 else planes
    if (t[1] or t[3]) and e % 4:
        raise ValueError("gen_attention with position_embedding_dim=%r: the embedding (generalized_attention.py:182-194) has "
                         "2 * ceil(dim / 4) features where appr_geom_fc takes dim // 2; dim must be a multiple of 4" % (e,))
    return dict(attention_type=t, num_heads=heads, head_dim=planes // heads, kv_stride=a['kv_stride'],
                position_embedding_dim=e, position_magnitude=a['position_magnitude'], channels=planes)


def gen_attention_layout(depth, gen_attention=None, stage_with_gen_attention=((), (), (), ())):
    """what ResNet(depth, gen_attention=..., stage_with_gen_attention=...) builds after each block's conv2, per stage and
    block: None or the block's gen_attention_spec.  An index past the stage's last block builds nothing (resnet.py:283-300)"""
    return tuple(tuple(gen_attention_spec(gen_attention, 64 << li) if gen_attention is not None and b in stage_with_gen_attention[li]
                       else None for b in range(nblk))
                 for li, nblk in enumerate(STAGE_BLOCKS[depth]))


def gen_attention_keys(spec):
    """the parameter names (after `gen_attention_block.`) of a block with this spec, with their shapes"""
    t, c, e = spec['attention_type'], spec['channels'], spec['position_embedding_dim']
    keys = {}
    if t[0] or t[1]:
        keys['query_conv.weight'] = (c, c, 1, 1)
    if t[0] or t[2]:
        keys['key_conv.weight'] = (c, c, 1, 1)
    keys['value_conv.weight'] = (c, c, 1, 1)
    if t[1] or t[3]:
        keys['appr_geom_fc_x.weight'] = (c, e // 2)
        keys['appr_geom_fc_y.weight'] = (c, e // 2)
    if t[2]:
        keys['appr_bias'] = (c,)
    if t[3]:
        keys['geom_bias'] = (c,)
    keys['proj_conv.weight'] = (c, c, 1, 1)
    keys['proj_conv.bias'] = (c,)
    keys['gamma'] = (1,)
    return keys


def _draw_gen_attention(sd, p, spec, g, gamma):
    """a gen_attention_block as the reference initialises it: ResNet.init_weights' kaiming (fan_out, normal, zero bias) on
    its four convolutions (resnet.py:474-476 re-draws every nn.Conv2d), kaiming_uniform(a=1) on appr_geom_fc_{x,y}
    (generalized_attention.py:374-383), appr_bias / geom_bias uniform in +-1/sqrt(2 d), gamma 0.
    gamma > 0 (tests only): gamma is that value, and query_conv / key_conv / appr_geom_fc are drawn 1/d^(1/4) narrower, so
    that content and position energies have about unit spread for unit-variance inputs instead of ~sqrt(d)"""
    c, d = spec['channels'], spec['head_dim']
    shrink = d ** -0.25 if gamma > 0 else 1.0
    for name, shape in gen_attention_keys(spec).items():
        k = p + '.gen_attention_block.' + name
        w = torch.empty(shape)
        if name.endswith('conv.weight'):
            _kaiming_fan_out(w, g)
            if name.startswith(('query', 'key')):
                w *= shrink
        elif name.startswith('appr_geom_fc'):
            bound = math.sqrt(3.0 / shape[1])
            w.uniform_(-bound, bound, generator=g).mul_(shrink)
        elif name in ('appr_bias', 'geom_bias'):
            stdv = 1.0 / math.sqrt(2 * d)
            w.uniform_(-stdv, stdv, generator=g)
        elif name == 'gamma':
            w.fill_(gamma)
        else:                                                          # proj_conv.bias
            w.zero_()
        sd[k] = w


# ContextBlock's arguments besides inplanes (context_block.py:15-19) and the fusions it knows, in the order it applies them
GCB_ARGS = ('ratio', 'pooling_type', 'fusion_types')
GCB_FUSIONS = ('channel_add', 'channel_mul')
GCB_MAX_PLANES = 2048


def gcb_spec(cfg, channels):
    """the block that ContextBlock(channels, **cfg) builds, as the engine runs it: dict(channels, planes = int(channels * ratio),
    pooling_type, fusion_types - the fusions used, in GCB_FUSIONS order).  ValueError where the reference itself fails (a
    pooling_type other than 'avg' / 'att', fusion_types that are not a non-empty list or tuple of known fusions, planes < 1),
    NotImplementedError for more than GCB_MAX_PLANES planes, TypeError for a missing ratio or an unknown argument"""
    if not isinstance(cfg, dict):
        raise ValueError("gcb must be a dict of ContextBlock arguments, not %r" % (cfg,))
    unknown = sorted(set(cfg) - set(GCB_ARGS))
    if unknown:
        raise TypeError("ContextBlock got unexpected arguments %s" % unknown)
    if 'ratio' not in cfg:
        raise TypeError("ContextBlock needs a ratio (context_block.py:15-19)")
    pooling, fusions = cfg.get('pooling_type', 'att'), cfg.get('fusion_types', ('channel_add',))
    if pooling not in ('avg', 'att'):
        raise ValueError("gcb with pooling_type=%r: context_block.py:21 takes 'avg' or 'att'" % (pooling,))
    if not isinstance(fusions, (list, tuple)) or not fusions or any(f not in GCB_FUSIONS for f in fusions):
        raise ValueError("gcb with fusion_types=%r: context_block.py:22-25 needs a non-empty list or tuple of %s"
                         % (fusions, GCB_FUSIONS))
    planes = int(channels * cfg['ratio'])
    if planes < 1:
        raise ValueError("gcb with ratio=%r on %d channels gives int(%d * ratio) = %d planes: the MLP needs at least one"
                         % (cfg['ratio'], channels, channels, planes))
    if planes > GCB_MAX_PLANES:
        raise NotImplementedError("gcb with ratio=%r on %d channels gives %d planes: liborp_b200 runs up to %d"
                                  % (cfg['ratio'], channels, planes, GCB_MAX_PLANES))
    return dict(channels=channels, planes=planes, pooling_type=pooling, fusion_types=tuple(f for f in GCB_FUSIONS if f in fusions))


def gcb_layout(depth, gcb=None, stage_with_gcb=(False, False, False, False)):
    """what ResNet(depth, gcb=..., stage_with_gcb=...) builds after each block's bn3, per stage and block: None or the block's
    gcb_spec.  Every block of a selected stage has one (resnet.py:411, 282-298).  ValueError unless stage_with_gcb names the
    four stages"""
    if gcb is None:
        return tuple((None,) * nblk for nblk in STAGE_BLOCKS[depth])
    if len(stage_with_gcb) != len(STAGE_BLOCKS[depth]):
        raise ValueError("stage_with_gcb=%r: needs one entry per stage (%d), as resnet.py:397-398 asserts"
                         % (tuple(stage_with_gcb), len(STAGE_BLOCKS[depth])))
    return tuple(tuple(gcb_spec(gcb, 256 << li) if stage_with_gcb[li] else None for _ in range(nblk))
                 for li, nblk in enumerate(STAGE_BLOCKS[depth]))


def gcb_keys(spec):
    """the parameter names (after `context_block.`) of a block with this spec, with their shapes"""
    c, p = spec['channels'], spec['planes']
    keys = {}
    if spec['pooling_type'] == 'att':
        keys['conv_mask.weight'] = (1, c, 1, 1)
        keys['conv_mask.bias'] = (1,)
    for f in spec['fusion_types']:
        keys[f + '_conv.0.weight'] = (p, c, 1, 1)
        keys[f + '_conv.0.bias'] = (p,)
        keys[f + '_conv.1.weight'] = (p, 1, 1)
        keys[f + '_conv.1.bias'] = (p, 1, 1)
        keys[f + '_conv.3.weight'] = (c, p, 1, 1)
        keys[f + '_conv.3.bias'] = (c,)
    return keys


def _draw_gcb(sd, p, spec, g, gain):
    """a context_block as the reference initialises it: ResNet.init_weights' kaiming (fan_out, normal, zero bias) on every
    nn.Conv2d, conv_mask and the last convolution included (resnet.py:474-476 re-draws what ContextBlock.reset_parameters set),
    LayerNorm weight 1 and bias 0.
    gain > 0 (tests only): conv_mask from N(0, 1 / C) (logits of about unit spread for unit-variance inputs) with an N(0, 1)
    bias, N(0, 0.1^2) biases on the first convolution, LayerNorm weight in [0.5, 1.5] and bias N(0, 0.1^2), and the last
    convolution and its N(0, 0.1^2) bias times gain, so every term acts"""
    c = spec['channels']
    for name, shape in gcb_keys(spec).items():
        w = torch.empty(shape)
        if name == 'conv_mask.weight' and gain > 0:
            w.normal_(0, math.sqrt(1.0 / c), generator=g)
        elif name.endswith('weight') and len(shape) == 4:
            _kaiming_fan_out(w, g)
            if name.endswith('.3.weight') and gain > 0:
                w *= gain
        elif gain <= 0:
            w.fill_(1.0 if name.endswith('.1.weight') else 0.0)
        elif name.endswith('.1.weight'):
            w.uniform_(0.5, 1.5, generator=g)
        else:
            w.normal_(0, 1.0 if name == 'conv_mask.bias' else 0.1, generator=g)
            if name.endswith('.3.bias'):
                w *= gain
        sd[p + '.context_block.' + name] = w


CARAFE_KERNELS = (1, 3, 5, 7)
CARAFE_GROUPS = (1, 2, 4)


def fpn_carafe_spec(in_channels, out_channels, norm_cfg=None, act_cfg=None, order=('conv', 'norm', 'act'),
                    upsample_cfg=dict(type='carafe', up_kernel=5, up_group=1, encoder_kernel=3, encoder_dilation=1)):
    """the engine's description of an FPN_CARAFE neck (fpn_carafe.py:34-200) on the backbone's stride-8, -16 and -32 outputs,
    whose widths are `in_channels`, with two extra levels (3x3 stride-2 laterals): dict(in_channels, out_channels, norm
    (None or 'GN'), relu, up_kernel, up_group, encoder_kernel, compressed_channels).  ValueError where the reference itself
    fails, NotImplementedError (naming the argument) for what the engine does not build"""
    if tuple(order) not in (('conv', 'norm', 'act'), ('act', 'conv', 'norm')):
        raise ValueError("FPN_CARAFE order=%r: the reference accepts ('conv', 'norm', 'act') and ('act', 'conv', 'norm')" % (order,))
    if act_cfg is not None:
        if tuple(order) != ('conv', 'norm', 'act'):
            raise NotImplementedError("FPN_CARAFE order=%r with an activation: liborp_b200 builds order ('conv', 'norm', 'act'), "
                                      "or ('act', 'conv', 'norm') with act_cfg=None" % (order,))
        if dict(act_cfg, inplace=None) != dict(type='ReLU', inplace=None):
            raise NotImplementedError("FPN_CARAFE act_cfg=%r: liborp_b200 builds None or ReLU" % (act_cfg,))
    if norm_cfg is not None:
        n = dict(norm_cfg)
        n.pop('requires_grad', None)
        if n != dict(type='GN', num_groups=32):
            raise NotImplementedError("FPN_CARAFE norm_cfg=%r: liborp_b200 builds None or GN with 32 groups" % (norm_cfg,))
    if out_channels != 256:
        raise NotImplementedError("FPN_CARAFE out_channels=%r: liborp_b200 builds the head's 256" % (out_channels,))
    cfg = dict(upsample_cfg) if upsample_cfg is not None else dict(type=None)
    kind = cfg.pop('type', None)
    if kind in ('nearest', 'bilinear'):
        raise NotImplementedError("FPN_CARAFE upsample_cfg type %r: liborp_b200 builds 'carafe'" % (kind,))
    if kind != 'carafe':
        raise ValueError("FPN_CARAFE upsample_cfg type %r: the reference fails on it (%s)"
                         % (kind, "slice_as asserts on the un-upsampled lateral" if kind is None else
                            "hasattr(dict, 'upsample_kernel') is False" if kind in ('deconv', 'pixel_shuffle') else
                            "it is not one of its upsample types"))
    args = dict(up_kernel=5, up_group=1, encoder_kernel=3, encoder_dilation=1, compressed_channels=64)
    unknown = set(cfg) - set(args)
    if unknown:
        raise ValueError("FPN_CARAFE upsample_cfg: CARAFEPack takes no argument %s" % sorted(unknown))
    args.update(cfg)
    k, grp = args['up_kernel'], args['up_group']
    if not isinstance(k, int) or k < 1 or k % 2 == 0:
        raise ValueError("FPN_CARAFE up_kernel=%r: the carafe op asserts an odd kernel >= 1" % (k,))
    if k not in CARAFE_KERNELS:
        raise NotImplementedError("FPN_CARAFE up_kernel=%r: liborp_b200 builds %s" % (k, CARAFE_KERNELS))
    if not isinstance(grp, int) or grp < 1 or out_channels % grp:
        raise ValueError("FPN_CARAFE up_group=%r: the carafe op asserts that it divides the %d channels" % (grp, out_channels))
    if grp not in CARAFE_GROUPS:
        raise NotImplementedError("FPN_CARAFE up_group=%r: liborp_b200 builds %s" % (grp, CARAFE_GROUPS))
    if args['encoder_kernel'] not in (1, 3):
        raise NotImplementedError("FPN_CARAFE encoder_kernel=%r: liborp_b200 builds 1 and 3" % (args['encoder_kernel'],))
    if args['encoder_dilation'] != 1:
        raise NotImplementedError("FPN_CARAFE encoder_dilation=%r: liborp_b200 builds 1" % (args['encoder_dilation'],))
    cc = args['compressed_channels']
    if not isinstance(cc, int) or cc < 8 or cc % 8:
        raise NotImplementedError("FPN_CARAFE compressed_channels=%r: liborp_b200 builds positive multiples of 8" % (cc,))
    return dict(in_channels=tuple(in_channels), out_channels=out_channels, norm=None if norm_cfg is None else 'GN',
                relu=act_cfg is not None, up_kernel=k, up_group=grp, encoder_kernel=args['encoder_kernel'], compressed_channels=cc)


def fpn_carafe_keys(spec):
    """{key: shape} of the neck.* parameters of an FPN_CARAFE of spec (fpn_carafe_spec): every ConvModule has a bias iff it
    has no norm; laterals 0..2 are 1x1 on the backbone levels, 3 a 3x3 / s2 on the last of them, 4 a 3x3 / s2 on lateral 3"""
    out, keys = spec['out_channels'], {}

    def cm(name, cin, k):
        keys[name + '.conv.weight'] = (out, cin, k, k)
        if spec['norm'] is None:
            keys[name + '.conv.bias'] = (out,)
        else:
            keys[name + '.gn.weight'] = keys[name + '.gn.bias'] = (out,)
    for i, cin in enumerate(spec['in_channels']):
        cm('neck.lateral_convs.%d' % i, cin, 1)
    cm('neck.lateral_convs.3', spec['in_channels'][-1], 3)
    cm('neck.lateral_convs.4', out, 3)
    for i in range(5):
        cm('neck.fpn_convs.%d' % i, out, 3)
    cc, ek = spec['compressed_channels'], spec['encoder_kernel']
    ce = spec['up_kernel'] ** 2 * spec['up_group'] * 4
    for j in range(4):
        p = 'neck.upsample_modules.%d.' % j
        keys[p + 'channel_compressor.weight'], keys[p + 'channel_compressor.bias'] = (cc, out, 1, 1), (cc,)
        keys[p + 'content_encoder.weight'], keys[p + 'content_encoder.bias'] = (ce, cc, ek, ek), (ce,)
    return keys


def _draw_fpn_carafe(sd, g, spec, reference_init, carafe_gain):
    """FPN_CARAFE.init_weights (fpn_carafe.py:203-209): xavier-uniform on every conv with zero biases, then CARAFEPack's
    normal_init(std=0.001) on content_encoder; norms 1 / 0.  reference_init=False randomises the norms and the biases.
    carafe_gain > 0 (tests only) draws content_encoder from N(0, gain^2 / fan_in) with N(0, (gain / 2)^2) biases instead, so
    that the logits spread over several units: with the reference's init the softmax is almost uniform"""
    for k, shape in fpn_carafe_keys(spec).items():
        if k.endswith('.gn.weight'):
            sd[k] = torch.ones(shape) if reference_init else torch.empty(shape).uniform_(0.5, 1.5, generator=g)
        elif k.endswith('.bias'):
            sd[k] = torch.zeros(shape) if reference_init else torch.empty(shape).normal_(0, 0.1, generator=g)
        elif 'content_encoder' in k:
            fan_in = shape[1] * shape[2] * shape[3]
            sd[k] = torch.empty(shape).normal_(0, carafe_gain / math.sqrt(fan_in) if carafe_gain > 0 else 0.001, generator=g)
        else:
            sd[k] = _xavier_uniform(torch.empty(shape), g)
    if carafe_gain > 0:
        for j in range(4):
            b = 'neck.upsample_modules.%d.content_encoder.bias' % j
            sd[b] = torch.empty(sd[b].shape).normal_(0, carafe_gain / 2, generator=g)


def _drawers(sd, g, reference_init, residual_gain):
    """the (conv, norm) draws of the random state dicts into sd from generator g"""

    def conv(name, cout, cin, k, init, bias=False, std=0.01):
        w = torch.empty(cout, cin, k, k)                              # (grouped conv2: cin = channels per group)
        if init == "kaiming":
            _kaiming_fan_out(w, g)
        elif init == "xavier":
            _xavier_uniform(w, g)
        elif init == "fan_in":
            w.normal_(0, math.sqrt(1.0 / (cin * k * k)), generator=g)
        elif init == "caffe2_xavier":
            # mmcv caffe2_xavier_init = kaiming_init(a=1, mode='fan_in', nonlinearity='leaky_relu', distribution='uniform')
            bound = math.sqrt(3.0 / (cin * k * k))
            w.uniform_(-bound, bound, generator=g)
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

    return conv, norm


def _draw_head(sd, g, conv, norm, reference_init, num_classes, feat):
    """OrientedRepPointsHead (orientedreppoints_head.py:134-146)"""
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



def random_state_dict(depth=50, seed=0, reference_init=True, num_classes=16, feat=256, residual_gain=1.0, dcn=None,
                      stage_with_dcn=(False, False, False, False), dcn_offset_scale=0.0, groups=1, base_width=4,
                      gen_attention=None, stage_with_gen_attention=((), (), (), ()), gen_attention_gamma=0.0, gcb=None,
                      stage_with_gcb=(False, False, False, False), gcb_gain=0.0, neck=None, carafe_gain=0.0):
    """reference_init=True reproduces the reference's init_weights (incl. zero_init_residual and all-ones
    norm scales); False randomises norm parameters / running statistics so that every branch of the graph
    carries signal (used by the parity tests); residual_gain scales the randomised scale of every block's last norm
    (1.0 doubles the activation variance per block: fine for 16 blocks, ~1e5 after R-101's 33 - use 0.3 there).
    dcn / stage_with_dcn: the backbone's deformable conv2 layers as ResNet takes them (dcn_layout).  Their weights follow
    the reference (resnet.py:474-484): DeformConv.reset_parameters' uniform +-1/sqrt(9 planes) (kaiming_init skips a layer
    that is not an nn.Conv2d; with reference_init=False the kaiming draw of a plain conv2 instead) and an all-zero
    conv_offset.  dcn_offset_scale > 0 (tests only) draws conv_offset from N(0, scale^2 / fan_in) with N(0, scale^2) biases
    instead, so that the samples leave the grid by about `scale` pixels per unit of input and the DCNv2 mask logits vary;
    with zero offsets a deformable layer is a plain convolution.
    groups / base_width: a ResNeXt (resnext.py): conv1 / conv2 / bn1 / bn2 are block_width() wide and conv2 has `groups` groups,
    its kaiming fan_out width * 9 as for any nn.Conv2d.  groups=1 draws exactly the ResNet's tensors.
    gen_attention / stage_with_gen_attention: the blocks' gen_attention_block as ResNet takes them (gen_attention_layout),
    drawn by _draw_gen_attention after the block's other tensors; gen_attention_gamma > 0 (tests only) makes them act (see
    there).  Without attention blocks every draw is what it was without these arguments.
    gcb / stage_with_gcb: the blocks' context_block as ResNet / ResNeXt take them (gcb_layout), drawn by _draw_gcb after the
    block's other tensors; gcb_gain > 0 (tests only) makes every term act (see there; use it with reference_init=False and
    a residual_gain).  Without context blocks every draw is what it was without these arguments.
    neck: None (the FPN of configs/dota/*.py) or an fpn_carafe_spec, drawn by _draw_fpn_carafe in the FPN's place; carafe_gain
    > 0 (tests only) spreads its encoder logits (see there).  Without `neck` every draw is what it was without these arguments."""
    check_groups(groups, base_width)
    if groups > 1 and dcn is not None and any(stage_with_dcn):
        raise NotImplementedError("dcn with groups=%d would be a grouped deformable convolution (resnext.py:56-66): not built" % groups)
    g = torch.Generator().manual_seed(seed)
    sd = {}
    layout = dcn_layout(depth, dcn, stage_with_dcn)
    ga_layout = gen_attention_layout(depth, gen_attention, stage_with_gen_attention)
    if groups > 1 and any(sp is not None for st in ga_layout for sp in st):
        raise NotImplementedError("gen_attention on ResNeXt: the reference's ResNeXt builds no attention blocks (resnext.py:196-216)")
    gcb_lay = gcb_layout(depth, gcb, stage_with_gcb)
    conv, norm = _drawers(sd, g, reference_init, residual_gain)

    # ---------------------------------------------------------------- backbone (resnet.py)
    conv("backbone.conv1", 64, 3, 7, "kaiming")
    norm("backbone.bn1", 64, True)
    inplanes = 64
    for li, (nblk, planes) in enumerate(zip(STAGE_BLOCKS[depth], (64, 128, 256, 512))):
        for b in range(nblk):
            p = "backbone.layer%d.%d" % (li + 1, b)
            width = block_width(planes, groups, base_width)
            conv(p + ".conv1", width, inplanes, 1, "kaiming")
            norm(p + ".bn1", width, True)
            kind = layout[li][b]
            if kind is None:
                conv(p + ".conv2", width, width // groups, 3, "kaiming")
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
            norm(p + ".bn2", width, True)
            conv(p + ".conv3", planes * 4, width, 1, "kaiming")
            norm(p + ".bn3", planes * 4, True, zero_gamma=True)           # zero_init_residual, resnet.py:486-491
            if b == 0:
                conv(p + ".downsample.0", planes * 4, inplanes, 1, "kaiming")
                norm(p + ".downsample.1", planes * 4, True)
            if ga_layout[li][b] is not None:
                _draw_gen_attention(sd, p, ga_layout[li][b], g, gen_attention_gamma)
            if gcb_lay[li][b] is not None:
                _draw_gcb(sd, p, gcb_lay[li][b], g, gcb_gain)
            inplanes = planes * 4
    # ---------------------------------------------------------------- neck (fpn.py, start_level=1, 5 outs)
    if neck is not None:
        _draw_fpn_carafe(sd, g, neck, reference_init, carafe_gain)
        _draw_head(sd, g, conv, norm, reference_init, num_classes, feat)
        return sd
    for i, cin in enumerate((512, 1024, 2048)):
        conv("neck.lateral_convs.%d.conv" % i, feat, cin, 1, "xavier")
        norm("neck.lateral_convs.%d.gn" % i, feat, False)
        conv("neck.fpn_convs.%d.conv" % i, feat, feat, 3, "xavier")
        norm("neck.fpn_convs.%d.gn" % i, feat, False)
    conv("neck.fpn_convs.3.conv", feat, 2048, 3, "xavier")                 # extra_convs_on_inputs: on C5
    norm("neck.fpn_convs.3.gn", feat, False)
    conv("neck.fpn_convs.4.conv", feat, feat, 3, "xavier")
    norm("neck.fpn_convs.4.gn", feat, False)
    _draw_head(sd, g, conv, norm, reference_init, num_classes, feat)
    return sd


def fold_bn(w, bn_w, bn_b, mean, var, eps=1e-5):
    """eval-mode BatchNorm folded into the preceding bias-free conv - the reference-sanctioned fold of
    tools/fuse_conv_bn.py:10-24.  Returns (w', b')."""
    factor = bn_w / torch.sqrt(var + eps)
    return w * factor.reshape(-1, 1, 1, 1), bn_b - mean * factor


def random_hrnet_state_dict(arch="hrnetv2p_w32", seed=0, reference_init=True, num_classes=16, residual_gain=1.0, feat=256,
                            zero_init_residual=False):
    """state dict of HRNet(arch) + HRFPN(arch.out_widths, feat) + the head, with the reference's keys.
    arch: a key of hrnet.ARCHS or an hrnet.HRNetArch.  reference_init=True reproduces the reference's init_weights: kaiming
    (fan_out, normal) on every backbone conv and constant-1 norms (hrnet.py:462-478; with zero_init_residual, each residual
    block's last norm constant 0),
    caffe2_xavier_init with zero biases on HRFPN (hrfpn.py:73-76), the head's own init.  False randomises the norms as
    random_state_dict does, draws the backbone convs from N(0, 1 / fan_in) (kaiming's fan_out would amplify the 1x1 fuse
    convs, 8 * w channels into w, 16-fold in variance) and HRFPN's biases from N(0, 0.1^2), so every branch and fuse path
    carries signal at a bounded scale;
    residual_gain scales the randomised scale of each residual block's last norm (BasicBlock bn2, Bottleneck bn3)"""
    from .hrnet import ARCHS, backbone_convs
    arch = ARCHS[arch] if isinstance(arch, str) else arch
    g = torch.Generator().manual_seed(seed)
    sd = {}
    conv, norm = _drawers(sd, g, reference_init, residual_gain)
    for ck, bk, cout, cin, k, last in backbone_convs(arch):
        conv("backbone." + ck, cout, cin, k, "kaiming" if reference_init else "fan_in")
        norm("backbone." + bk, cout, True, zero_gamma=last and (zero_init_residual or not reference_init))
    conv("neck.reduction_conv.conv", feat, sum(arch.out_widths), 1, "caffe2_xavier", bias=True)
    for i in range(5):
        conv("neck.fpn_convs.%d.conv" % i, feat, feat, 3, "caffe2_xavier", bias=True)
    if not reference_init:
        for k in list(sd):
            if k.startswith("neck."):
                if k.endswith(".bias"):
                    sd[k] = torch.empty_like(sd[k]).normal_(0, 0.1, generator=g)
    _draw_head(sd, g, conv, norm, reference_init, num_classes, feat)
    return sd
