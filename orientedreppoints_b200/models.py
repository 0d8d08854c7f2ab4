"""Module-structure layer of the drop-in boundary (SURVEY.md 8(b), last row): the registries and the nn.Module parameter
containers the reference's configs name - ResNet (mmdet/models/backbones/resnet.py:345-515), SwinTransformer
(backbones/swin_transformer.py:449-631), FPN (necks/fpn.py:50-136), OrientedRepPointsHead
(anchor_heads/orientedreppoints_head.py:18-146), OrientedRepPointsDetector (detectors/orientedreppoints_detector.py,
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


class Bottleneck(_EngineOnly):
    """resnet.py:84-239 (style 'pytorch': the stride sits on the 3x3).  dcn: the conv2 config of resnet.py:146-168 - a
    DCN / DCNv2 layer (DeformConvPack / ModulatedDeformConvPack) unless `fallback_on_stride`, which is popped from the dict
    itself: ResNet hands every block the same dict, so only the first block built from it sees the value"""
    expansion = 4

    def __init__(self, inplanes, planes, stride, downsample, norm_cfg, conv_cfg=None, dcn=None):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 1, bias=False)
        self.add_module('bn1', build_norm_layer(norm_cfg, planes, 1)[1])
        fallback_on_stride = dcn.pop('fallback_on_stride', False) if dcn is not None else False
        if dcn is None or fallback_on_stride:
            self.conv2 = nn.Conv2d(planes, planes, 3, stride, 1, bias=False)
        else:
            assert conv_cfg is None, 'conv_cfg cannot be None for DCN'
            self.conv2 = build_conv_layer(dcn, planes, planes, kernel_size=3, stride=stride, padding=1, dilation=1, bias=False)
        self.add_module('bn2', build_norm_layer(norm_cfg, planes, 2)[1])
        self.conv3 = nn.Conv2d(planes, planes * 4, 1, bias=False)
        self.add_module('bn3', build_norm_layer(norm_cfg, planes * 4, 3)[1])
        self.downsample = downsample


@BACKBONES.register_module
class ResNet(_EngineOnly):
    arch_settings = {50: (3, 4, 6, 3), 101: (3, 4, 23, 3)}

    def __init__(self, depth, in_channels=3, num_stages=4, strides=(1, 2, 2, 2), dilations=(1, 1, 1, 1), out_indices=(0, 1, 2, 3),
                 style='pytorch', frozen_stages=-1, conv_cfg=None, norm_cfg=dict(type='BN', requires_grad=True), norm_eval=True,
                 dcn=None, stage_with_dcn=(False, False, False, False), gcb=None, stage_with_gcb=(False, False, False, False),
                 gen_attention=None, stage_with_gen_attention=((), (), (), ()), with_cp=False, zero_init_residual=True):
        super().__init__()
        if depth not in self.arch_settings:
            raise KeyError('invalid depth {} for resnet'.format(depth))
        if style != 'pytorch' or num_stages != 4 or tuple(strides) != (1, 2, 2, 2) or tuple(dilations) != (1, 1, 1, 1) \
                or gcb is not None or gen_attention is not None:
            raise NotImplementedError("liborp_b200 builds the configuration of configs/dota/*.py: 4 stages, style 'pytorch', "
                                      "strides (1,2,2,2), no dilation / GCB / attention in the backbone")
        if dcn is not None:
            assert isinstance(dcn, dict) and len(stage_with_dcn) == num_stages
            if dcn.get('deformable_groups', 1) != 1:
                raise NotImplementedError("liborp_b200 builds backbone DCN / DCNv2 layers with deformable_groups=1, not "
                                          "deformable_groups=%r" % (dcn['deformable_groups'],))
        self.depth, self.out_indices, self.frozen_stages, self.norm_eval = depth, out_indices, frozen_stages, norm_eval
        self.zero_init_residual = zero_init_residual
        self.dcn, self.stage_with_dcn = dcn, tuple(stage_with_dcn)
        self.dcn_cfg = None if dcn is None else dict(dcn)           # as given, before the blocks pop fallback_on_stride
        self.conv1 = nn.Conv2d(in_channels, 64, 7, 2, 3, bias=False)
        self.add_module('bn1', build_norm_layer(norm_cfg, 64, 1)[1])
        inplanes = 64
        for i, nblk in enumerate(self.arch_settings[depth]):
            planes, blocks = 64 << i, []
            stage_dcn = dcn if self.stage_with_dcn[i] else None      # the one shared dict (resnet.py:402, 146-147)
            for b in range(nblk):
                stride = strides[i] if b == 0 else 1
                ds = None
                if b == 0:
                    ds = nn.Sequential(nn.Conv2d(inplanes, planes * 4, 1, stride, bias=False), build_norm_layer(norm_cfg, planes * 4)[1])
                blocks.append(Bottleneck(inplanes, planes, stride, ds, norm_cfg, conv_cfg, stage_dcn))
                inplanes = planes * 4
            self.add_module('layer%d' % (i + 1), nn.Sequential(*blocks))

    def dcn_layout(self):
        """per stage, per block: None for a plain conv2, else 'DCN' or 'DCNv2' - what the engine builds for that conv2"""
        kinds = {ModulatedDeformConvPack: 'DCNv2', DeformConvPack: 'DCN', nn.Conv2d: None}
        return tuple(tuple(kinds[type(blk.conv2)] for blk in getattr(self, 'layer%d' % (i + 1)))
                     for i in range(len(self.arch_settings[self.depth])))


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
            sd = random_state_dict(self.backbone.depth, seed=0, reference_init=True, num_classes=self.bbox_head.num_classes,
                                   dcn=self.backbone.dcn_cfg, stage_with_dcn=self.backbone.stage_with_dcn)
        else:
            from .swin import random_swin_state_dict
            sd = random_swin_state_dict(0, num_classes=self.bbox_head.num_classes, arch=self.backbone.arch)
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
            self._engine = Engine({k: v.detach() for k, v in self.state_dict().items()}, depth, dev, self.precision,
                                  test_cfg=dict(self.test_cfg) if self.test_cfg else None,
                                  dcn=self.backbone.dcn_layout() if resnet else None)
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
