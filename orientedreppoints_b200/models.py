"""Module-structure layer of the drop-in boundary (SURVEY.md 8(b), last row): the registries and the nn.Module parameter
containers the reference's configs name - ResNet (mmdet/models/backbones/resnet.py:345-515), ResNeXt (resnext.py), SwinTransformer
(backbones/swin_transformer.py:449-631), FPN (necks/fpn.py:50-136), OrientedRepPointsHead
(anchor_heads/orientedreppoints_head.py:18-146), HRNet (backbones/hrnet.py) with HRFPN (necks/hrfpn.py), FPN_CARAFE
(necks/fpn_carafe.py) with CARAFEPack (ops/carafe/carafe.py), OrientedRepPointsDetector (detectors/orientedreppoints_detector.py,
single_stage.py) - with the reference's attribute names, so `build_detector(cfg.model, test_cfg=cfg.test_cfg)` builds from
the reference's config dicts and `state_dict()` / `load_state_dict()` use the reference's keys (published checkpoints load).

These classes hold parameters and configuration; they do not re-implement the layers in PyTorch.  Inference
(`simple_test` / `aug_test` / `forward(return_loss=False)`) hands the state_dict to the engine in detector.py, whose every
layer is a kernel of liborp_b200.so.  Training entry points raise NotImplementedError (out of scope, SURVEY.md 8)."""
import torch
import torch.nn as nn

from .ops.conv import build_conv_layer
from .ops.conv_module import ConvModule
from .ops.dcn import DeformConv, DeformConvPack, ModulatedDeformConvPack
from .ops.norm import build_norm_layer
from .utils.registry import Registry, build_from_cfg
from .weights import STAGE_BLOCKS, block_width, check_groups, fpn_carafe_spec, gcb_spec, gen_attention_spec

BACKBONES = Registry('backbone')
NECKS = Registry('neck')
HEADS = Registry('head')
DETECTORS = Registry('detector')
LOSSES = Registry('loss')


def build(cfg, registry, default_args=None):
    if isinstance(cfg, list):
        return nn.Sequential(*[build_from_cfg(c, registry, default_args) for c in cfg])
    return build_from_cfg(cfg, registry, default_args)


def build_backbone(cfg):
    return build(cfg, BACKBONES)


def build_neck(cfg):
    return build(cfg, NECKS)


def build_head(cfg):
    return build(cfg, HEADS)


def build_detector(cfg, train_cfg=None, test_cfg=None):
    return build(cfg, DETECTORS, dict(train_cfg=train_cfg, test_cfg=test_cfg))


def build_loss(cfg):
    return build(cfg, LOSSES)


class _EngineOnly(nn.Module):
    def forward(self, *a, **k):
        raise NotImplementedError("%s is a parameter container here; it runs inside OrientedRepPointsDetector.simple_test "
                                  "on the liborp_b200 engine" % type(self).__name__)


class GeneralizedAttention(_EngineOnly):
    """the parameter tree of generalized_attention.py:34-150 for a spec of weights.gen_attention_spec: only the layers that
    attention_type uses exist (query_conv for t0 / t1, key_conv for t0 / t2, appr_geom_fc_{x,y} for t1 / t3, appr_bias for t2,
    geom_bias for t3); value_conv, proj_conv (with bias) and gamma always"""

    def __init__(self, in_dim, spec):
        super().__init__()
        t, c, e = spec['attention_type'], in_dim, spec['position_embedding_dim']
        self.spec = spec
        if t[0] or t[1]:
            self.query_conv = nn.Conv2d(c, c, 1, bias=False)
        if t[0] or t[2]:
            self.key_conv = nn.Conv2d(c, c, 1, bias=False)
        self.value_conv = nn.Conv2d(c, c, 1, bias=False)
        if t[1] or t[3]:
            self.appr_geom_fc_x = nn.Linear(e // 2, c, bias=False)
            self.appr_geom_fc_y = nn.Linear(e // 2, c, bias=False)
        if t[2]:
            self.appr_bias = nn.Parameter(torch.zeros(c))
        if t[3]:
            self.geom_bias = nn.Parameter(torch.zeros(c))
        self.proj_conv = nn.Conv2d(c, c, 1, bias=True)
        self.gamma = nn.Parameter(torch.zeros(1))


class ContextBlock(_EngineOnly):
    """the parameter tree of context_block.py:13-52 for a spec of weights.gcb_spec: conv_mask for 'att' pooling, and a
    channel_{add,mul}_conv (1x1 C -> P, LayerNorm([P, 1, 1]), ReLU, 1x1 P -> C) for each fusion used"""

    def __init__(self, inplanes, spec):
        super().__init__()
        c, p = inplanes, spec['planes']
        self.spec = spec
        if spec['pooling_type'] == 'att':
            self.conv_mask = nn.Conv2d(c, 1, 1)
        for f in spec['fusion_types']:
            setattr(self, f + '_conv', nn.Sequential(nn.Conv2d(c, p, 1), nn.LayerNorm([p, 1, 1]), nn.ReLU(inplace=True),
                                                     nn.Conv2d(p, c, 1)))


class Bottleneck(_EngineOnly):
    """resnet.py:84-239 (style 'pytorch': the stride sits on the 3x3).  dcn: the conv2 config of resnet.py:146-168 - a
    DCN / DCNv2 layer (DeformConvPack / ModulatedDeformConvPack) unless `fallback_on_stride`, which is popped from the dict
    itself: ResNet hands every block the same dict, so only the first block built from it sees the value.
    groups / base_width: the ResNeXt block (resnext.py:11-70): conv1 / conv2 are block_width() wide, conv2 has `groups` groups"""
    expansion = 4

    def __init__(self, inplanes, planes, stride, downsample, norm_cfg, conv_cfg=None, dcn=None, groups=1, base_width=4,
                 gen_attention=None, gcb=None):
        super().__init__()
        width = block_width(planes, groups, base_width)
        self.conv1 = nn.Conv2d(inplanes, width, 1, bias=False)
        self.add_module('bn1', build_norm_layer(norm_cfg, width, 1)[1])
        fallback_on_stride = dcn.pop('fallback_on_stride', False) if dcn is not None else False
        if dcn is None or fallback_on_stride:
            self.conv2 = nn.Conv2d(width, width, 3, stride, 1, groups=groups, bias=False)
        else:
            assert conv_cfg is None, 'conv_cfg cannot be None for DCN'
            self.conv2 = build_conv_layer(dcn, width, width, kernel_size=3, stride=stride, padding=1, dilation=1, bias=False)
        self.add_module('bn2', build_norm_layer(norm_cfg, width, 2)[1])
        self.conv3 = nn.Conv2d(width, planes * 4, 1, bias=False)
        self.add_module('bn3', build_norm_layer(norm_cfg, planes * 4, 3)[1])
        self.downsample = downsample
        if gen_attention is not None:                                 # resnet.py:186-189, applied after relu(bn2(conv2))
            self.gen_attention_block = GeneralizedAttention(planes, gen_attention_spec(gen_attention, planes))
        if gcb is not None:                                           # resnet.py:182-184, applied to bn3(conv3(.))
            self.context_block = ContextBlock(planes * 4, gcb_spec(gcb, planes * 4))


@BACKBONES.register_module
class ResNet(_EngineOnly):
    arch_settings = STAGE_BLOCKS                                      # depth -> blocks per stage, shared with weights / the engine

    def __init__(self, depth, in_channels=3, num_stages=4, strides=(1, 2, 2, 2), dilations=(1, 1, 1, 1), out_indices=(0, 1, 2, 3),
                 style='pytorch', frozen_stages=-1, conv_cfg=None, norm_cfg=dict(type='BN', requires_grad=True), norm_eval=True,
                 dcn=None, stage_with_dcn=(False, False, False, False), gcb=None, stage_with_gcb=(False, False, False, False),
                 gen_attention=None, stage_with_gen_attention=((), (), (), ()), with_cp=False, zero_init_residual=True):
        super().__init__()
        if depth not in self.arch_settings:
            raise KeyError('invalid depth {} for resnet'.format(depth))
        if style != 'pytorch' or num_stages != 4 or tuple(strides) != (1, 2, 2, 2) or tuple(dilations) != (1, 1, 1, 1):
            raise NotImplementedError("liborp_b200 builds the configuration of configs/dota/*.py: 4 stages, style 'pytorch', "
                                      "strides (1,2,2,2), no dilation in the backbone")
        if gcb is not None:
            if len(stage_with_gcb) != num_stages:
                raise ValueError("stage_with_gcb=%r: needs one entry per stage (%d), as resnet.py:397-398 asserts"
                                 % (tuple(stage_with_gcb), num_stages))
            if not any(stage_with_gcb):
                raise NotImplementedError("gcb=%r selects no block: stage_with_gcb is all False, so the reference builds no "
                                          "context block; set stage_with_gcb (e.g. (False, True, True, True)) or drop gcb" % (gcb,))
        if dcn is not None:
            assert isinstance(dcn, dict) and len(stage_with_dcn) == num_stages
            if dcn.get('deformable_groups', 1) != 1:
                raise NotImplementedError("liborp_b200 builds backbone DCN / DCNv2 layers with deformable_groups=1, not "
                                          "deformable_groups=%r" % (dcn['deformable_groups'],))
        self.depth, self.out_indices, self.frozen_stages, self.norm_eval = depth, out_indices, frozen_stages, norm_eval
        self.zero_init_residual = zero_init_residual
        self.dcn, self.stage_with_dcn = dcn, tuple(stage_with_dcn)
        self.dcn_cfg = None if dcn is None else dict(dcn)           # as given, before the blocks pop fallback_on_stride
        self.gen_attention = None if gen_attention is None else dict(gen_attention)
        self.stage_with_gen_attention = tuple(tuple(s) for s in stage_with_gen_attention)
        if gen_attention is not None:
            assert isinstance(gen_attention, dict) and len(self.stage_with_gen_attention) == num_stages
        self.gcb = None if gcb is None else dict(gcb)
        self.stage_with_gcb = tuple(stage_with_gcb)
        self.conv1 = nn.Conv2d(in_channels, 64, 7, 2, 3, bias=False)
        self.add_module('bn1', build_norm_layer(norm_cfg, 64, 1)[1])
        inplanes = 64
        for i, nblk in enumerate(self.arch_settings[depth]):
            planes, blocks = 64 << i, []
            stage_dcn = dcn if self.stage_with_dcn[i] else None      # the one shared dict (resnet.py:402, 146-147)
            stage_gcb = self.gcb if gcb is not None and self.stage_with_gcb[i] else None   # every block of the stage (resnet.py:411)
            for b in range(nblk):
                stride = strides[i] if b == 0 else 1
                ds = None
                if b == 0:
                    ds = nn.Sequential(nn.Conv2d(inplanes, planes * 4, 1, stride, bias=False), build_norm_layer(norm_cfg, planes * 4)[1])
                # make_res_layer (resnet.py:283-300): block b gets the dict when b is listed; an index past the stage builds nothing
                ga = self.gen_attention if b in self.stage_with_gen_attention[i] else None
                blocks.append(Bottleneck(inplanes, planes, stride, ds, norm_cfg, conv_cfg, stage_dcn, gen_attention=ga,
                                         gcb=stage_gcb, **self._block_args()))
                inplanes = planes * 4
            self.add_module('layer%d' % (i + 1), nn.Sequential(*blocks))

    def _block_args(self):
        """extra Bottleneck arguments of this backbone (ResNeXt: groups, base_width)"""
        return {}

    def dcn_layout(self):
        """per stage, per block: None for a plain conv2, else 'DCN' or 'DCNv2' - what the engine builds for that conv2"""
        kinds = {ModulatedDeformConvPack: 'DCNv2', DeformConvPack: 'DCN', nn.Conv2d: None}
        return tuple(tuple(kinds[type(blk.conv2)] for blk in getattr(self, 'layer%d' % (i + 1)))
                     for i in range(len(self.arch_settings[self.depth])))

    def gen_attention_layout(self):
        """per stage, per block: None, or the spec (weights.gen_attention_spec) of that block's gen_attention_block - what the
        engine builds after its conv2"""
        return tuple(tuple(blk.gen_attention_block.spec if hasattr(blk, 'gen_attention_block') else None
                           for blk in getattr(self, 'layer%d' % (i + 1)))
                     for i in range(len(self.arch_settings[self.depth])))

    def gcb_layout(self):
        """per stage, per block: None, or the spec (weights.gcb_spec) of that block's context_block - what the engine runs on
        bn3(conv3(.)) before the residual add"""
        return tuple(tuple(blk.context_block.spec if hasattr(blk, 'context_block') else None
                           for blk in getattr(self, 'layer%d' % (i + 1)))
                     for i in range(len(self.arch_settings[self.depth])))


@BACKBONES.register_module
class ResNeXt(ResNet):
    """resnext.py:128-206: a ResNet whose bottlenecks are block_width() wide with a grouped conv2.  The engine runs the group
    widths of the published models (32x4d, 64x4d, 32x8d); other (groups, base_width) and DCN on a grouped conv2 raise
    NotImplementedError.  groups=1 is the ResNet, DCN included."""

    def __init__(self, groups=1, base_width=4, **kwargs):
        check_groups(groups, base_width)
        if kwargs.get('gen_attention') is not None and any(len(s) for s in kwargs.get('stage_with_gen_attention', ())):
            raise NotImplementedError("gen_attention on ResNeXt: the reference's ResNeXt rebuilds every stage without it "
                                      "(resnext.py:196-216), so its checkpoints hold no attention blocks; liborp_b200 does not build them")
        if groups > 1 and kwargs.get('dcn') is not None and any(kwargs.get('stage_with_dcn', ())):
            raise NotImplementedError("dcn with groups=%d would be a grouped deformable convolution (resnext.py:56-66): "
                                      "liborp_b200 does not build it" % groups)
        self.groups, self.base_width = groups, base_width            # read by _block_args while ResNet.__init__ builds
        super().__init__(**kwargs)

    def _block_args(self):
        return dict(groups=self.groups, base_width=self.base_width)


@BACKBONES.register_module()
class SwinTransformer(_EngineOnly):
    """parameter tree of swin_transformer.py:449-631 for every architecture the engine builds (swin.check_arch: four stages,
    head dimension 32, embed_dim a multiple of 32 up to 192, window 7 or 12 - Swin-T/S/B/L), the other arguments as
    configs/dota/orientedrepoints_swin_tiny_demo.py has them"""

    def __init__(self, embed_dim=96, depths=(2, 2, 6, 2), num_heads=(3, 6, 12, 24), window_size=7, mlp_ratio=4., qkv_bias=True,
                 qk_scale=None, drop_rate=0., attn_drop_rate=0., drop_path_rate=0.2, ape=False, patch_norm=True,
                 out_indices=(0, 1, 2, 3), frozen_stages=-1, use_checkpoint=False, pretrain_img_size=224, patch_size=4, in_chans=3):
        super().__init__()
        from .swin import check_arch
        self.arch = check_arch(embed_dim, depths, num_heads, window_size, qk_scale)
        for name, value, built in (("mlp_ratio", float(mlp_ratio), 4.0), ("qkv_bias", bool(qkv_bias), True), ("ape", bool(ape), False),
                                   ("patch_norm", bool(patch_norm), True), ("out_indices", tuple(out_indices), (1, 2, 3)),
                                   ("patch_size", patch_size, 4), ("in_chans", in_chans, 3)):
            if value != built:
                raise NotImplementedError("liborp_b200 builds Swin backbones with %s=%r (configs/dota/orientedrepoints_swin_tiny_demo.py), "
                                          "not %s=%r" % (name, built, name, value))
        self.out_indices = tuple(out_indices)
        self.embed_dim, self.depths, self.num_heads = self.arch.embed, self.arch.depths, self.arch.heads
        self.window_size, self.qk_scale = self.arch.window, self.arch.qk_scale

        def block(c, heads):
            m = nn.Module()
            m.norm1, m.norm2 = nn.LayerNorm(c), nn.LayerNorm(c)
            m.attn = nn.Module()
            m.attn.qkv, m.attn.proj = nn.Linear(c, 3 * c, bias=True), nn.Linear(c, c)
            m.attn.relative_position_bias_table = nn.Parameter(torch.zeros((2 * window_size - 1) ** 2, heads))
            m.mlp = nn.Module()
            m.mlp.fc1, m.mlp.fc2 = nn.Linear(c, 4 * c), nn.Linear(4 * c, c)
            return m

        self.patch_embed = nn.Module()
        self.patch_embed.proj = nn.Conv2d(in_chans, embed_dim, patch_size, patch_size)
        self.patch_embed.norm = nn.LayerNorm(embed_dim)
        self.layers = nn.ModuleList()
        for i, (d, h) in enumerate(zip(depths, num_heads)):
            c = embed_dim << i
            layer = nn.Module()
            layer.blocks = nn.ModuleList([block(c, h) for _ in range(d)])
            if i < len(depths) - 1:
                layer.downsample = nn.Module()
                layer.downsample.norm = nn.LayerNorm(4 * c)
                layer.downsample.reduction = nn.Linear(4 * c, 2 * c, bias=False)
            self.layers.append(layer)
        for i in self.out_indices:
            self.add_module('norm%d' % i, nn.LayerNorm(embed_dim << i))


class BasicBlock(_EngineOnly):
    """resnet.py:13-83: conv1 3x3 (stride) + bn1 + ReLU, conv2 3x3 + bn2, + identity or downsample, ReLU"""
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None, norm_cfg=dict(type='BN')):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 3, stride, 1, bias=False)
        self.add_module('bn1', build_norm_layer(norm_cfg, planes, 1)[1])
        self.conv2 = nn.Conv2d(planes, planes, 3, 1, 1, bias=False)
        self.add_module('bn2', build_norm_layer(norm_cfg, planes, 2)[1])
        self.downsample = downsample


def _conv_bn(cin, cout, k, stride, norm_cfg, relu=False, upsample=None):
    layers = [nn.Conv2d(cin, cout, k, stride, k // 2, bias=False), build_norm_layer(norm_cfg, cout)[1]]
    if relu:
        layers.append(nn.ReLU(inplace=False))
    if upsample:
        layers.append(nn.Upsample(scale_factor=upsample, mode='nearest'))
    return nn.Sequential(*layers)


class HRModule(_EngineOnly):
    """hrnet.py:12-191: branches.{b} (BasicBlocks), fuse_layers.{i}.{j} (1x1 + BN + upsample for j > i, a chain of 3x3 / s2
    convs for j < i, None for j == i)"""

    def __init__(self, num_branches, num_blocks, in_channels, num_channels, norm_cfg):
        super().__init__()
        from .hrnet import fuse_convs
        self.num_branches = num_branches
        branches = []
        for b in range(num_branches):
            ds = None
            if in_channels[b] != num_channels[b]:
                ds = nn.Sequential(nn.Conv2d(in_channels[b], num_channels[b], 1, bias=False), build_norm_layer(norm_cfg, num_channels[b])[1])
            blocks = [BasicBlock(in_channels[b], num_channels[b], 1, ds, norm_cfg)]
            blocks += [BasicBlock(num_channels[b], num_channels[b], norm_cfg=norm_cfg) for _ in range(1, num_blocks[b])]
            branches.append(nn.Sequential(*blocks))
        self.branches = nn.ModuleList(branches)
        self.fuse_layers = None
        if num_branches > 1:
            rows = []
            for i, row in enumerate(fuse_convs(tuple(num_channels))):
                mods = []
                for j, path in enumerate(row):
                    if path is None:
                        mods.append(None)
                    elif j > i:
                        mods.append(_conv_bn(num_channels[j], num_channels[i], 1, 1, norm_cfg, upsample=2 ** (j - i)))
                    else:
                        mods.append(nn.Sequential(*[_conv_bn(cin, cout, 3, 2, norm_cfg, relu=k < len(path) - 1)
                                                    for k, (_, _, cout, cin, _, _) in enumerate(path)]))
                rows.append(nn.ModuleList(mods))
            self.fuse_layers = nn.ModuleList(rows)


@BACKBONES.register_module
class HRNet(_EngineOnly):
    """hrnet.py:194-525 for every architecture hrnet.HRNetArch.from_extra accepts (stages 1-4 of 1, 2, 3, 4 branches, stage 1
    BOTTLENECK or BASIC, stages 2-4 BASIC, any widths and module / block counts); `arch` is that description"""

    def __init__(self, extra, in_channels=3, conv_cfg=None, norm_cfg=dict(type='BN'), norm_eval=True, with_cp=False,
                 zero_init_residual=False):
        super().__init__()
        from .hrnet import HRNetArch, transition_convs
        if in_channels != 3:
            raise NotImplementedError("HRNet with in_channels=%r: liborp_b200 builds 3-channel (RGB) inputs" % (in_channels,))
        if conv_cfg is not None:
            raise NotImplementedError("HRNet with conv_cfg=%r: liborp_b200 builds plain convolutions" % (conv_cfg,))
        if norm_cfg is None or norm_cfg.get('type') != 'BN':
            raise NotImplementedError("HRNet with norm_cfg=%r: liborp_b200 builds BN norms (folded into the convolutions)" % (norm_cfg,))
        self.arch = HRNetArch.from_extra(extra)
        self.extra, self.norm_cfg, self.norm_eval, self.with_cp = extra, norm_cfg, norm_eval, with_cp
        self.zero_init_residual = zero_init_residual
        self.conv1 = nn.Conv2d(3, 64, 3, 2, 1, bias=False)
        self.add_module('bn1', build_norm_layer(norm_cfg, 64, 1)[1])
        self.conv2 = nn.Conv2d(64, 64, 3, 2, 1, bias=False)
        self.add_module('bn2', build_norm_layer(norm_cfg, 64, 2)[1])
        s1 = self.arch.stages[0]
        ch, out1 = s1.num_channels[0], s1.widths[0]
        ds = None if out1 == 64 else nn.Sequential(nn.Conv2d(64, out1, 1, bias=False), build_norm_layer(norm_cfg, out1)[1])
        if s1.block == 'BOTTLENECK':
            blocks = [Bottleneck(64, ch, 1, ds, norm_cfg)] + [Bottleneck(out1, ch, 1, None, norm_cfg) for _ in range(1, s1.num_blocks[0])]
        else:
            blocks = [BasicBlock(64, ch, 1, ds, norm_cfg)] + [BasicBlock(out1, ch, norm_cfg=norm_cfg) for _ in range(1, s1.num_blocks[0])]
        self.layer1 = nn.Sequential(*blocks)
        pre = s1.widths
        for s in range(1, 4):
            st = self.arch.stages[s]
            trans = []
            for t in transition_convs(pre, st.widths):
                if t is None:
                    trans.append(None)
                elif len(t) == 1 and t[0][4] == 1:
                    trans.append(_conv_bn(t[0][3], t[0][2], 3, 1, norm_cfg, relu=True))
                else:
                    trans.append(nn.Sequential(*[_conv_bn(cin, cout, 3, 2, norm_cfg, relu=True) for _, _, cout, cin, _ in t]))
            self.add_module('transition%d' % s, nn.ModuleList(trans))
            self.add_module('stage%d' % (s + 1), nn.Sequential(*[HRModule(st.num_branches, st.num_blocks, list(st.widths),
                                                                           list(st.widths), norm_cfg)
                                                                  for _ in range(st.num_modules)]))
            pre = st.widths


@NECKS.register_module
class HRFPN(_EngineOnly):
    """hrfpn.py:11-100: reduction_conv and fpn_convs.{i} are ConvModules with a bias and NO norm, whatever norm_cfg says
    (hrfpn.py:49-66 never passes it on).  Built: num_outs=5 with stride=2 (the head's strides 8..128), pooling 'MAX' or
    anything else for average, as the reference reads it"""

    def __init__(self, in_channels, out_channels, num_outs=5, pooling_type='AVG', conv_cfg=None, norm_cfg=None, with_cp=False,
                 stride=1):
        super().__init__()
        assert isinstance(in_channels, list)
        if num_outs != 5 or stride != 2:
            raise NotImplementedError("HRFPN with num_outs=%r, stride=%r: liborp_b200 builds num_outs=5 with stride=2, whose "
                                      "five levels have the head's strides 8..128" % (num_outs, stride))
        if conv_cfg is not None:
            raise NotImplementedError("HRFPN with conv_cfg=%r: liborp_b200 builds plain convolutions" % (conv_cfg,))
        self.in_channels, self.out_channels, self.num_ins, self.num_outs = in_channels, out_channels, len(in_channels), num_outs
        self.with_cp, self.conv_cfg, self.norm_cfg, self.stride = with_cp, conv_cfg, norm_cfg, stride
        self.pooling_type = 'MAX' if pooling_type == 'MAX' else 'AVG'
        self.reduction_conv = ConvModule(sum(in_channels), out_channels, 1, conv_cfg=conv_cfg, act_cfg=None)
        self.fpn_convs = nn.ModuleList([ConvModule(out_channels, out_channels, 3, padding=1, stride=stride, conv_cfg=conv_cfg,
                                                   act_cfg=None) for _ in range(num_outs)])


@NECKS.register_module
class FPN(_EngineOnly):
    def __init__(self, in_channels, out_channels, num_outs, start_level=0, end_level=-1, add_extra_convs=False,
                 extra_convs_on_inputs=True, relu_before_extra_convs=False, no_norm_on_lateral=False, conv_cfg=None,
                 norm_cfg=None, act_cfg=None):
        super().__init__()
        assert isinstance(in_channels, list)
        if end_level != -1 or relu_before_extra_convs or no_norm_on_lateral or act_cfg is not None or norm_cfg is None:
            raise NotImplementedError("liborp_b200 builds the FPN of configs/dota/*.py: GN laterals, no activation, end_level -1")
        self.in_channels, self.out_channels, self.num_ins, self.num_outs = in_channels, out_channels, len(in_channels), num_outs
        self.start_level, self.add_extra_convs, self.extra_convs_on_inputs = start_level, add_extra_convs, extra_convs_on_inputs
        assert num_outs >= self.num_ins - start_level
        self.lateral_convs, self.fpn_convs = nn.ModuleList(), nn.ModuleList()
        for i in range(start_level, self.num_ins):
            self.lateral_convs.append(ConvModule(in_channels[i], out_channels, 1, conv_cfg=conv_cfg, norm_cfg=norm_cfg, act_cfg=None, inplace=False))
            self.fpn_convs.append(ConvModule(out_channels, out_channels, 3, padding=1, conv_cfg=conv_cfg, norm_cfg=norm_cfg, act_cfg=None, inplace=False))
        extra = num_outs - self.num_ins + start_level
        if add_extra_convs:
            for i in range(extra):
                cin = in_channels[-1] if (i == 0 and extra_convs_on_inputs) else out_channels
                self.fpn_convs.append(ConvModule(cin, out_channels, 3, stride=2, padding=1, conv_cfg=conv_cfg, norm_cfg=norm_cfg, act_cfg=None, inplace=False))


class CARAFEPack(_EngineOnly):
    """the parameter tree of carafe.py:161-214 with scale factor 2: channel_compressor (1x1 C -> compressed_channels) and
    content_encoder (encoder_kernel, C' -> up_kernel^2 * up_group * 4), both with a bias"""

    def __init__(self, channels, up_kernel=5, up_group=1, encoder_kernel=3, compressed_channels=64):
        super().__init__()
        self.channels, self.up_kernel, self.up_group = channels, up_kernel, up_group
        self.channel_compressor = nn.Conv2d(channels, compressed_channels, 1)
        self.content_encoder = nn.Conv2d(compressed_channels, up_kernel * up_kernel * up_group * 4, encoder_kernel,
                                         padding=(encoder_kernel - 1) // 2)


@NECKS.register_module
class FPN_CARAFE(_EngineOnly):
    """fpn_carafe.py:34-200 with the reference's tree and keys.  Built: five outputs at the head's strides 8..128 - the
    backbone's stride-8, -16 and -32 outputs (in_channels[start_level:], end_level=-1) and two extra levels - with
    upsample_cfg type 'carafe' and the arguments weights.fpn_carafe_spec accepts; `spec` is that description"""

    def __init__(self, in_channels, out_channels, num_outs, start_level=0, end_level=-1, norm_cfg=None, act_cfg=None,
                 order=('conv', 'norm', 'act'),
                 upsample_cfg=dict(type='carafe', up_kernel=5, up_group=1, encoder_kernel=3, encoder_dilation=1)):
        super().__init__()
        assert isinstance(in_channels, list)
        if end_level != -1:
            raise NotImplementedError("FPN_CARAFE end_level=%r: liborp_b200 builds end_level=-1, with two extra levels" % (end_level,))
        if not 0 <= start_level < len(in_channels) or num_outs < len(in_channels) - start_level:
            raise ValueError("FPN_CARAFE start_level=%r, num_outs=%r on %d inputs: the reference asserts num_outs >= %d inputs - "
                             "start_level" % (start_level, num_outs, len(in_channels), len(in_channels)))
        if len(in_channels) - start_level != 3 or num_outs != 5:
            raise NotImplementedError("FPN_CARAFE start_level=%r, num_outs=%r on %d inputs: liborp_b200 builds three backbone "
                                      "levels (strides 8, 16, 32) and num_outs=5" % (start_level, num_outs, len(in_channels)))
        self.spec = fpn_carafe_spec(in_channels[start_level:], out_channels, norm_cfg, act_cfg, order, upsample_cfg)
        self.in_channels, self.out_channels, self.num_ins, self.num_outs = in_channels, out_channels, len(in_channels), num_outs
        self.start_level, self.end_level, self.norm_cfg, self.act_cfg, self.order = start_level, end_level, norm_cfg, act_cfg, order
        sp = self.spec
        kw = dict(norm_cfg=norm_cfg, bias=norm_cfg is None, act_cfg=act_cfg, inplace=False, order=tuple(order))
        self.lateral_convs, self.fpn_convs, self.upsample_modules = nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
        for cin in sp['in_channels']:
            self.lateral_convs.append(ConvModule(cin, out_channels, 1, **kw))
        self.lateral_convs.append(ConvModule(sp['in_channels'][-1], out_channels, 3, stride=2, padding=1, **kw))
        self.lateral_convs.append(ConvModule(out_channels, out_channels, 3, stride=2, padding=1, **kw))
        for _ in range(5):
            self.fpn_convs.append(ConvModule(out_channels, out_channels, 3, padding=1, **kw))
        for _ in range(4):
            self.upsample_modules.append(CARAFEPack(out_channels, sp['up_kernel'], sp['up_group'], sp['encoder_kernel'],
                                                    sp['compressed_channels']))


@HEADS.register_module
class OrientedRepPointsHead(_EngineOnly):
    def __init__(self, num_classes, in_channels, feat_channels=256, point_feat_channels=256, stacked_convs=3, num_points=9,
                 gradient_mul=0.1, point_strides=[8, 16, 32, 64, 128], point_base_scale=4, conv_cfg=None, norm_cfg=None,
                 loss_cls=None, loss_rbox_init=None, loss_rbox_refine=None, loss_spatial_init=None, loss_spatial_refine=None,
                 center_init=True, top_ratio=0.4):
        super().__init__()
        k = int(round(num_points ** 0.5))
        assert k * k == num_points, 'The points number should be a square number.'
        assert k % 2 == 1, 'The points number should be an odd square number.'
        use_sigmoid = True if loss_cls is None else loss_cls.get('use_sigmoid', False)
        self.num_classes, self.in_channels, self.feat_channels = num_classes, in_channels, feat_channels
        self.point_feat_channels, self.stacked_convs, self.num_points = point_feat_channels, stacked_convs, num_points
        self.gradient_mul, self.point_strides, self.point_base_scale = gradient_mul, point_strides, point_base_scale
        self.cls_out_channels = num_classes - 1 if use_sigmoid else num_classes
        self.dcn_kernel, self.dcn_pad = k, (k - 1) // 2
        self.relu = nn.ReLU(inplace=True)
        self.cls_convs, self.reg_convs = nn.ModuleList(), nn.ModuleList()
        for i in range(stacked_convs):
            chn = in_channels if i == 0 else feat_channels
            self.cls_convs.append(ConvModule(chn, feat_channels, 3, stride=1, padding=1, conv_cfg=conv_cfg, norm_cfg=norm_cfg))
            self.reg_convs.append(ConvModule(chn, feat_channels, 3, stride=1, padding=1, conv_cfg=conv_cfg, norm_cfg=norm_cfg))
        self.reppoints_cls_conv = DeformConv(feat_channels, point_feat_channels, k, 1, self.dcn_pad)
        self.reppoints_cls_out = nn.Conv2d(point_feat_channels, self.cls_out_channels, 1, 1, 0)
        self.reppoints_pts_init_conv = nn.Conv2d(feat_channels, point_feat_channels, 3, 1, 1)
        self.reppoints_pts_init_out = nn.Conv2d(point_feat_channels, 2 * num_points, 1, 1, 0)
        self.reppoints_pts_refine_conv = DeformConv(feat_channels, point_feat_channels, k, 1, self.dcn_pad)
        self.reppoints_pts_refine_out = nn.Conv2d(point_feat_channels, 2 * num_points, 1, 1, 0)


@DETECTORS.register_module
class OrientedRepPointsDetector(nn.Module):
    """single_stage.py:10-50 + orientedreppoints_detector.py:11-144: backbone / neck / bbox_head built from their config dicts;
    inference runs on the liborp_b200 engine (detector.py) fed with this module's state_dict"""

    def __init__(self, backbone, neck=None, bbox_head=None, train_cfg=None, test_cfg=None, pretrained=None, precision="f16x3"):
        super().__init__()
        self.backbone = build_backbone(backbone)
        self.neck = build_neck(neck) if neck is not None else None
        self.bbox_head = build_head(bbox_head)
        if isinstance(self.backbone, HRNet) != isinstance(self.neck, HRFPN):
            raise NotImplementedError("%s with %s: liborp_b200 builds HRNet with the HRFPN neck, and the ResNet / Swin backbones "
                                      "with FPN or FPN_CARAFE" % (type(self.backbone).__name__, type(self.neck).__name__))
        if isinstance(self.neck, FPN_CARAFE):
            if isinstance(self.backbone, ResNet):
                widths = [256 << i for i in self.backbone.out_indices]
            else:
                widths = [self.backbone.embed_dim << i for i in self.backbone.out_indices]
            if list(self.neck.in_channels) != widths or list(self.neck.spec['in_channels']) != widths[-3:]:
                raise ValueError("FPN_CARAFE in_channels %s with start_level %d are not the backbone's outputs %s ending in its "
                                 "stride-8, -16 and -32 levels" % (list(self.neck.in_channels), self.neck.start_level, widths))
            if self.neck.out_channels != self.bbox_head.in_channels:
                raise ValueError("FPN_CARAFE out_channels %d are not the head's in_channels %d"
                                 % (self.neck.out_channels, self.bbox_head.in_channels))
        if isinstance(self.neck, HRFPN):
            if list(self.neck.in_channels) != list(self.backbone.arch.out_widths):
                raise ValueError("HRFPN in_channels %s are not the HRNet's stage-4 widths %s"
                                 % (list(self.neck.in_channels), list(self.backbone.arch.out_widths)))
            if self.neck.out_channels != self.bbox_head.in_channels:
                raise ValueError("HRFPN out_channels %d are not the head's in_channels %d"
                                 % (self.neck.out_channels, self.bbox_head.in_channels))
        self.train_cfg, self.test_cfg, self.precision = train_cfg, test_cfg, precision
        self._engine = None
        self.init_weights(pretrained)

    with_neck = property(lambda self: self.neck is not None)

    def init_weights(self, pretrained=None):
        """the reference's initialisation (resnet.py:443-491, fpn.py:132-135, head :134-146) through the shared generator in
        weights.py; `pretrained` is a checkpoint path (torchvision:// / http URLs need the network and are ignored)"""
        import os
        if isinstance(self.backbone, ResNet):
            from .weights import random_state_dict
            ga = dict(gen_attention=self.backbone.gen_attention,
                      stage_with_gen_attention=self.backbone.stage_with_gen_attention) if self.backbone.gen_attention else {}
            if self.backbone.gcb is not None:
                ga.update(gcb=self.backbone.gcb, stage_with_gcb=self.backbone.stage_with_gcb)
            if isinstance(self.neck, FPN_CARAFE):
                ga.update(neck=self.neck.spec)
            sd = random_state_dict(self.backbone.depth, seed=0, reference_init=True, num_classes=self.bbox_head.num_classes,
                                   dcn=self.backbone.dcn_cfg, stage_with_dcn=self.backbone.stage_with_dcn,
                                   **self.backbone._block_args(), **ga)
        elif isinstance(self.backbone, HRNet):
            from .weights import random_hrnet_state_dict
            sd = random_hrnet_state_dict(self.backbone.arch, seed=0, reference_init=True, num_classes=self.bbox_head.num_classes,
                                         feat=self.neck.out_channels, zero_init_residual=self.backbone.zero_init_residual)
        else:
            from .swin import random_swin_state_dict
            sd = random_swin_state_dict(0, num_classes=self.bbox_head.num_classes, arch=self.backbone.arch,
                                        neck=self.neck.spec if isinstance(self.neck, FPN_CARAFE) else None)
        self.load_state_dict(sd, strict=True)
        if isinstance(pretrained, str) and os.path.isfile(pretrained):
            ck = torch.load(pretrained, map_location='cpu')
            self.backbone.load_state_dict(ck.get('state_dict', ck.get('model', ck)), strict=False)
        self._engine = None

    def load_state_dict(self, *a, **k):
        self._engine = None                                   # the engine caches folded / split weights
        return super().load_state_dict(*a, **k)

    def engine(self, device=None):
        if self._engine is None:
            from .detector import OrientedRepPointsDetector as Engine
            dev = torch.device(device) if device is not None else next(self.parameters()).device
            if dev.type != 'cuda':
                raise NotImplementedError("OrientedRepPointsDetector inference needs a CUDA (sm_90a) device: there is no CPU path")
            resnet = isinstance(self.backbone, ResNet)
            depth = self.backbone.depth if resnet else self.backbone.arch
            hr = isinstance(self.neck, HRFPN)
            self._engine = Engine({k: v.detach() for k, v in self.state_dict().items()}, depth, dev, self.precision,
                                  test_cfg=dict(self.test_cfg) if self.test_cfg else None,
                                  dcn=self.backbone.dcn_layout() if resnet else None,
                                  gen_attention=self.backbone.gen_attention_layout() if resnet else None,
                                  gcb=self.backbone.gcb_layout() if resnet else None,
                                  pooling_type=self.neck.pooling_type if hr else 'AVG',
                                  neck=self.neck.spec if isinstance(self.neck, FPN_CARAFE) else None)
        return self._engine

    def extract_feat(self, img):
        return self.engine().extract_feat(img)

    def simple_test(self, img, img_meta=None, rescale=False):
        return self.engine().simple_test(img, img_meta, rescale=rescale)

    def aug_test(self, imgs, img_metas, rescale=False, valid_hws=None, return_tensors=False):
        return self.engine().aug_test(imgs, img_metas, rescale, valid_hws, return_tensors=return_tensors)

    def forward_test(self, imgs, img_metas, **kwargs):
        """base.py:104-141: lists of augmented views; one view -> simple_test"""
        if not isinstance(imgs, (list, tuple)):
            imgs, img_metas = [imgs], [img_metas]
        if len(imgs) != len(img_metas):
            raise ValueError('num of augmentations ({}) != num of image meta ({})'.format(len(imgs), len(img_metas)))
        if len(imgs) == 1:
            return self.simple_test(imgs[0], img_metas[0], **kwargs)
        return self.aug_test(imgs, img_metas, **kwargs)

    def forward(self, img, img_meta=None, return_loss=True, **kwargs):
        if return_loss:
            raise NotImplementedError("training (forward_train / losses) is out of scope of liborp_b200")
        return self.forward_test(img, img_meta, **kwargs)


from . import losses  # noqa: E402,F401  (registers GIoULoss in LOSSES)
