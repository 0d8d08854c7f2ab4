"""The FPN_CARAFE neck (mmdet/models/necks/fpn_carafe.py, CARAFEPack of mmdet/ops/carafe/carafe.py) on the engines of
detector.py, for the five levels the head reads (strides 8..128).

  laterals  0..2: 1x1 ConvModules on the backbone's stride-8, -16 and -32 outputs; 3: a 3x3 / s2 ConvModule on the stride-32
            output; 4: a 3x3 / s2 ConvModule on lateral 3 (fpn_carafe.py:231-238)
  top-down  for i = 4..1: lateral[i-1] = lateral[i-1] + CARAFEPack_{i-1}(lateral[i]), cut to lateral[i-1]'s extent
  outputs   3x3 ConvModules (fpn_convs) on the five laterals
A ConvModule is the existing convolution with bias (no norm) or the convolution + GroupNorm(32), each + ReLU when act_cfg
has one.  A CARAFEPack is its channel_compressor (1x1 + bias), its content_encoder (+ bias) writing fp32 logits, and one
orp_carafe_add_* launch (include/orp_b200_carafe.h): the pixel shuffle, the softmax, the reassembly and the top-down add.
"""
from . import _lib
from .detector import ConvLayer, Norm
from .gen_attention import alloc, dims
from .weights import fpn_carafe_keys

_SUFFIX = {"fp32": "f32", "bf16": "bf16", "f16x3": "f16x3"}


def check_neck(sd, spec):
    """ValueError unless the state dict's neck.* parameters are exactly those of spec (weights.fpn_carafe_spec), in their
    shapes"""
    have = {k: tuple(v.shape) for k, v in sd.items() if k.startswith('neck.')}
    want = fpn_carafe_keys(spec)
    if have != want:
        missing, extra = sorted(set(want) - set(have)), sorted(set(have) - set(want))
        shape = sorted(k for k in set(want) & set(have) if want[k] != have[k])
        raise ValueError("the state dict's neck does not match the FPN_CARAFE spec: missing %s, unexpected %s, wrong shape %s"
                         % (missing, extra, ["%s %s != %s" % (k, have[k], want[k]) for k in shape]))


def carafe_add(e, x, logits, k, group, residual):
    """residual + carafe(x, softmax(pixel_shuffle(logits))) over the residual's extent: one orp_carafe_add_* launch"""
    n, h, w, c = dims(e, x)
    _, hr, wr, cr = dims(e, residual)
    assert cr == c and tuple(logits.shape) == (n, h, w, k * k * group * 4), (dims(e, x), dims(e, residual), tuple(logits.shape))
    y = alloc(e, n, hr, wr, c)
    fn = "orp_carafe_add_" + _SUFFIX[e.name]
    _lib.check(getattr(_lib.lib(), fn)(_lib.ptr(x), n, h, w, c, _lib.ptr(logits), k, group, _lib.ptr(residual), hr, wr, _lib.ptr(y),
                                       _lib.current_stream_ptr()), fn)
    return y


class CarafeFPN:
    """the engine form of an FPN_CARAFE neck of spec (weights.fpn_carafe_spec) from the state dict's neck.* tensors"""

    def __init__(self, sd, spec, device):
        check_neck(sd, spec)
        self.spec, self.relu = spec, spec['relu']
        self.k, self.group = spec['up_kernel'], spec['up_group']

        def module(p, stride, pad):
            b = sd.get(p + '.conv.bias')
            return (ConvLayer(sd[p + '.conv.weight'].float(), None if b is None else b.float(), stride, pad, device),
                    Norm(sd, p + '.gn', device) if spec['norm'] else None)
        self.lat = [module('neck.lateral_convs.%d' % i, 1, 0) for i in range(3)] + \
                   [module('neck.lateral_convs.%d' % i, 2, 1) for i in (3, 4)]
        self.fpn = [module('neck.fpn_convs.%d' % i, 1, 1) for i in range(5)]
        ek = spec['encoder_kernel']
        self.up = []
        for j in range(4):
            p = 'neck.upsample_modules.%d.' % j
            self.up.append((ConvLayer(sd[p + 'channel_compressor.weight'].float(), sd[p + 'channel_compressor.bias'].float(), 1, 0,
                                      device),
                            ConvLayer(sd[p + 'content_encoder.weight'].float(), sd[p + 'content_encoder.bias'].float(), 1,
                                      (ek - 1) // 2, device)))

    def _module(self, e, x, m):
        L, norm = m
        return e.conv(x, L, relu=self.relu) if norm is None else e.conv_gn(x, L, norm, relu=self.relu)

    def upsample_add(self, e, x, j, residual):
        """residual + CARAFEPack_j(x) over the residual's extent, in the engine's format"""
        comp, enc = self.up[j]
        logits = e.conv(e.conv(x, comp), enc, out_f32=True)              # fp32 [N, H, W, k^2 * G * 4]
        return carafe_add(e, x, logits, self.k, self.group, residual)

    def __call__(self, e, feats):
        """the five output levels from the backbone's stride-8, -16 and -32 outputs"""
        lats = [self._module(e, f, self.lat[i]) for i, f in enumerate(feats)]
        lats.append(self._module(e, feats[-1], self.lat[3]))
        lats.append(self._module(e, lats[-1], self.lat[4]))
        for i in range(4, 0, -1):
            lats[i - 1] = self.upsample_add(e, lats[i], i - 1, lats[i - 1])
        return [self._module(e, x, self.fpn[i]) for i, x in enumerate(lats)]
