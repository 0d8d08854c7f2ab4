"""`mmdet.ops.conv` surface (mmdet/ops/conv.py:6-40): config strings -> convolution layer classes; 'DCN' / 'DCNv2' resolve to
this repository's tensor-core (wgmma) deformable convolutions (ops/dcn.py)."""
from torch import nn as nn

from .dcn import DeformConvPack, ModulatedDeformConvPack

conv_cfg = {
    'Conv': nn.Conv2d,
    'DCN': DeformConvPack,
    'DCNv2': ModulatedDeformConvPack,
}


def build_conv_layer(cfg, *args, **kwargs):
    """cfg None -> plain nn.Conv2d; else cfg['type'] names the layer and the remaining keys are passed to it.
    Unknown type -> KeyError (conv.py:31-33; 'ConvWS' of the reference is a training-time variant and is not built)."""
    if cfg is None:
        spec = dict(type='Conv')
    else:
        assert isinstance(cfg, dict) and 'type' in cfg
        spec = dict(cfg)
    kind = spec.pop('type')
    if kind not in conv_cfg:
        raise KeyError('Unrecognized norm type {}'.format(kind))      # the reference's message, typo included
    return conv_cfg[kind](*args, **kwargs, **spec)
