"""Deformable convolution operator surface of `mmdet.ops.dcn` over liborp_b200.so.

Mirrors mmdet/ops/dcn/deform_conv.py - `deform_conv` / `DeformConv` / `DeformConvPack` (:14-58, :192-255, :258-323) and
`modulated_deform_conv` / `ModulatedDeformConv` / `ModulatedDeformConvPack` (:115-189, :326-374, :377-446): same names,
constructor / forward signatures, parameter names and shapes (`weight [out, in/groups, kh, kw]`, `conv_offset.*`), NCHW
fp32 tensors in and out, and the same error behaviour (`assert not bias`, ValueError for non-4-D input, CPU tensors ->
NotImplementedError, `RuntimeError` for an offset of the wrong shape as deform_conv_cuda.cpp:130-136 raises).

What runs underneath is NOT the reference's im2col + SGEMM (deform_conv_cuda.cpp:152-260: a 151 MB `columns` buffer per
level): the sampling happens inside a convolution kernel's A-operand loads.  `_route` picks the kernel from the shapes:

- the wgmma implicit-GEMM kernel (csrc/dense_tc.cu), in f16x3 arithmetic by default (fp32-faithful: |err| ~1e-5 of max,
  see include/orp_b200.h) or single-pass bf16 (`set_precision('bf16')`), when Cin % 64 == 0, dilation == 1, stride <= 256
  and the input holds fewer than 2^31 16-bit elements (N*H*W*Cin, twice that in f16x3: its producers use 32-bit offsets);
- the fp32 CUDA-core kernel `orp_deform_conv2d_f32` (csrc/dense_f32.cu) for every other shape and for
  `set_precision('fp32')`.  It reads float4 channel groups, so Cin is zero-padded to a multiple of 4 (input and weights;
  the padded channels add exactly 0).

Any kernel size (KH x KW), square stride / padding / dilation, bias and DCNv2 mask are accepted on both.  groups /
deformable_groups > 1 and non-square stride / padding / dilation are not built (the reference's configs use neither,
orientedreppoints_head.py:117-131).  Forward only: this repository is the inference path.
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.autograd import Function
from torch.nn.modules.utils import _pair, _single

from .. import _lib

_PRECISION = "f16x3"


def set_precision(p):
    """arithmetic of the tensor-core path: 'f16x3' (default, fp32-faithful) | 'bf16' (3x the rate, ~1e-2) | 'fp32' (CUDA cores)"""
    global _PRECISION
    if p not in ("f16x3", "bf16", "fp32"):
        raise ValueError("precision must be 'f16x3', 'bf16' or 'fp32'")
    _PRECISION = p


_TC_MAX_ELEMENTS = 1 << 31           # 16-bit input elements the tensor-core producers can address (32-bit offsets)
_TC_MAX_STRIDE = 256                 # a tensor-core tile spans at least one output column: BW * stride <= 256


def _route(precision, n, h, w, cin, stride, dilation):
    """the kernel a deformable convolution of this shape runs on: 'tc' (wgmma, csrc/dense_tc.cu) or 'f32'
    (orp_deform_conv2d_f32, csrc/dense_f32.cu)"""
    if precision == "fp32" or cin % 64 or dilation != 1 or stride > _TC_MAX_STRIDE:
        return "f32"
    planes = 2 if precision == "f16x3" else 1                # f16x3 holds every value as an fp16 (hi, lo) pair
    return "tc" if n * h * w * cin * planes < _TC_MAX_ELEMENTS else "f32"


def _cin4(cin):
    """the fp32 kernel reads float4 channel groups: Cin is zero-padded to a multiple of 4"""
    return (cin + 3) // 4 * 4


class _W:
    """weight holder in the layout the engines expect (same fields as detector.ConvLayer)"""

    def __init__(self, weight, bias, stride, pad):
        w = weight.detach().permute(0, 2, 3, 1).contiguous()
        self.w_raw = w.float().cpu()
        self.cout, self.kh, self.kw, self.cin = w.shape
        self.w = F.pad(w.float(), (0, _cin4(self.cin) - self.cin)).contiguous()     # fp32 kernel: [Cout, KH, KW, Cin4]
        self.bias = None if bias is None else bias.detach().float().contiguous()
        self.stride, self.pad = stride, pad
        self.tc = None


_cache = {}


def _layer(weight, bias, stride, pad):
    # keyed by address, layout and version counter; every view of a tensor shares its counter, so a caller passing
    # `m.weight.detach()` on each call hits too.  An entry holds the weight's and the bias's storage: while it is cached no
    # other tensor can be allocated at that address, so a key match is the same memory, not written since (writes through
    # a `.data` alias bump a counter of its own and are not seen).  At most 65 entries, i.e. their weights, are kept.
    key = (weight.data_ptr(), weight._version, tuple(weight.shape), weight.stride(), stride, pad,
           None if bias is None else (bias.data_ptr(), bias._version, tuple(bias.shape), bias.stride()))
    hit = _cache.get(key)
    if hit is not None:
        return hit[1]
    if len(_cache) > 64:
        _cache.clear()
    L = _W(weight, bias, stride, pad)
    _cache[key] = ((weight.untyped_storage(), None if bias is None else bias.untyped_storage()), L)
    return L


def _to_nhwc(x):
    """NCHW fp32 -> NHWC fp32 through the library's transpose kernel"""
    n, c, h, w = x.shape
    y = torch.empty((n, h, w, c), dtype=torch.float32, device=x.device)
    _lib.check(_lib.lib().orp_transpose_f32(_lib.ptr(x), n, c, h * w, _lib.ptr(y), _lib.current_stream_ptr()), "orp_transpose_f32")
    return y


def _to_nchw(y):
    n, h, w, c = y.shape
    x = torch.empty((n, c, h, w), dtype=torch.float32, device=y.device)
    _lib.check(_lib.lib().orp_transpose_f32(_lib.ptr(y), n, h * w, c, _lib.ptr(x), _lib.current_stream_ptr()), "orp_transpose_f32")
    return x


def _out_hw(h, w, kh, kw, stride, pad, dil):
    ho = (h + 2 * pad[0] - (dil[0] * (kh - 1) + 1)) // stride[0] + 1
    wo = (w + 2 * pad[1] - (dil[1] * (kw - 1) + 1)) // stride[1] + 1
    return ho, wo


def _forward(input, offset, mask, weight, bias, stride, padding, dilation, groups, deformable_groups):
    stride, padding, dilation = _pair(stride), _pair(padding), _pair(dilation)
    if not input.is_cuda:
        raise NotImplementedError
    if groups != 1 or deformable_groups != 1:
        raise NotImplementedError("liborp_b200: deformable convolution is built for groups = deformable_groups = 1")
    if stride[0] != stride[1] or padding[0] != padding[1] or dilation[0] != dilation[1]:
        raise NotImplementedError("liborp_b200: deformable convolution needs square stride / padding / dilation")
    n, cin, h, w = input.shape
    cout, cin_w, kh, kw = weight.shape
    if cin_w != cin:
        raise RuntimeError("deform_conv: weight has %d input channels, input has %d" % (cin_w, cin))
    ho, wo = _out_hw(h, w, kh, kw, stride, padding, dilation)
    if ho <= 0 or wo <= 0:
        raise ValueError('convolution input is too small (output would be {})'.format('x'.join(map(str, (n, cout, ho, wo)))))
    if tuple(offset.shape) != (n, 2 * kh * kw, ho, wo):
        # deform_conv_cuda.cpp:130-136 (AT_CHECK on the offset's shape)
        raise RuntimeError("invalid offset shape %s, expected %s" % (tuple(offset.shape), (n, 2 * kh * kw, ho, wo)))
    if mask is not None and tuple(mask.shape) != (n, kh * kw, ho, wo):
        raise RuntimeError("invalid mask shape %s, expected %s" % (tuple(mask.shape), (n, kh * kw, ho, wo)))
    dev = input.device
    with torch.cuda.device(dev):
        x = input.detach().float().contiguous()
        off = _to_nhwc(offset.detach().float().contiguous())
        msk = None if mask is None else _to_nhwc(mask.detach().float().contiguous())
        L = _layer(weight, bias, stride[0], padding[0])
        L.w, L.bias = L.w.to(dev), None if L.bias is None else L.bias.to(dev)
        if _route(_PRECISION, n, h, w, cin, stride[0], dilation[0]) == "tc":
            from ..engine_tc import EngineTC, EngineTCSplit
            if _PRECISION == "f16x3":
                eng = EngineTCSplit(dev)
                xs = torch.empty((n, h, w, 2, cin), dtype=torch.float16, device=dev)
                _lib.check(_lib.lib().orp_nchw_f32_to_split(_lib.ptr(x), n, cin, h * w, _lib.ptr(xs), _lib.current_stream_ptr()),
                           "orp_nchw_f32_to_split")
            else:
                eng = EngineTC(dev)
                xs = _to_nhwc(x).to(torch.bfloat16)
            tc = eng._tc(L)
            y = torch.empty((n, ho, wo, cout), dtype=torch.float32, device=dev)     # fp32 straight from the accumulator
            eng._launch([xs], [y], tc, cout, kh, kw, cin, stride[0], padding[0], L.bias, False, True, True,
                        offsets=[off], masks=None if msk is None else [msk])
        else:
            y = torch.empty((n, ho, wo, cout), dtype=torch.float32, device=dev)
            c4 = _cin4(cin)
            xp = x if c4 == cin else F.pad(x, (0, 0, 0, 0, 0, c4 - cin))
            rc = _lib.lib().orp_deform_conv2d_f32(_lib.ptr(_to_nhwc(xp)), n, h, w, c4, _lib.ptr(off), _lib.ptr(msk), _lib.ptr(L.w),
                                                  cout, kh, kw, stride[0], padding[0], dilation[0], _lib.ptr(L.bias), 0,
                                                  _lib.ptr(y), _lib.current_stream_ptr())
            _lib.check(rc, "orp_deform_conv2d_f32")
        return _to_nchw(y)


class DeformConvFunction(Function):
    """deform_conv.py:14-58; im2col_step is accepted and ignored (there is no columns buffer to chunk)"""

    @staticmethod
    def forward(ctx, input, offset, weight, stride=1, padding=0, dilation=1, groups=1, deformable_groups=1, im2col_step=64):
        if input is not None and input.dim() != 4:
            raise ValueError('Expected 4D tensor as input, got {}D tensor instead.'.format(input.dim()))
        return _forward(input, offset, None, weight, None, stride, padding, dilation, groups, deformable_groups)

    @staticmethod
    def backward(ctx, grad_output):
        raise NotImplementedError("liborp_b200 is the inference path: DeformConv has no backward")


class ModulatedDeformConvFunction(Function):
    """deform_conv.py:115-189"""

    @staticmethod
    def forward(ctx, input, offset, mask, weight, bias=None, stride=1, padding=0, dilation=1, groups=1, deformable_groups=1):
        if not input.is_cuda:
            raise NotImplementedError
        return _forward(input, offset, mask, weight, bias, stride, padding, dilation, groups, deformable_groups)

    @staticmethod
    def backward(ctx, grad_output):
        raise NotImplementedError("liborp_b200 is the inference path: ModulatedDeformConv has no backward")


deform_conv = DeformConvFunction.apply
modulated_deform_conv = ModulatedDeformConvFunction.apply


def _uniform_fan_in(weight, in_channels, kernel_size):
    n = in_channels
    for k in kernel_size:
        n *= k
    bound = 1. / math.sqrt(n)
    weight.data.uniform_(-bound, bound)


class DeformConv(nn.Module):
    """deform_conv.py:192-255"""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 deformable_groups=1, bias=False):
        super(DeformConv, self).__init__()
        assert not bias
        assert in_channels % groups == 0, 'in_channels {} cannot be divisible by groups {}'.format(in_channels, groups)
        assert out_channels % groups == 0, 'out_channels {} cannot be divisible by groups {}'.format(out_channels, groups)
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size = _pair(kernel_size)
        self.stride, self.padding, self.dilation = _pair(stride), _pair(padding), _pair(dilation)
        self.groups, self.deformable_groups = groups, deformable_groups
        self.transposed, self.output_padding = False, _single(0)            # nn.Conv2d compatibility
        self.weight = nn.Parameter(torch.Tensor(out_channels, in_channels // self.groups, *self.kernel_size))
        self.reset_parameters()

    def reset_parameters(self):
        _uniform_fan_in(self.weight, self.in_channels, self.kernel_size)

    def forward(self, x, offset):
        # inputs smaller than the kernel are zero padded on the right / bottom and the output cropped back (:239-255)
        ph, pw = max(self.kernel_size[0] - x.size(2), 0), max(self.kernel_size[1] - x.size(3), 0)
        if ph or pw:
            x = nn.functional.pad(x, (0, pw, 0, ph), 'constant', 0).contiguous()
            offset = nn.functional.pad(offset, (0, pw, 0, ph), 'constant', 0).contiguous()
        out = deform_conv(x, offset, self.weight, self.stride, self.padding, self.dilation, self.groups, self.deformable_groups)
        if ph or pw:
            out = out[:, :, :out.size(2) - ph, :out.size(3) - pw].contiguous()
        return out


def _rename_legacy_offset_keys(state_dict, prefix, local_metadata):
    """checkpoints written before version 2 name the offset branch `<name>_offset.*` (:302-316, :425-440)"""
    version = local_metadata.get('version', None)
    if version is None or version < 2:
        for leaf in ('weight', 'bias'):
            new, old = prefix + 'conv_offset.' + leaf, prefix[:-1] + '_offset.' + leaf
            if new not in state_dict and old in state_dict:
                state_dict[new] = state_dict.pop(old)


class DeformConvPack(DeformConv):
    """deform_conv.py:258-323: the offsets come from a plain convolution of the input"""
    _version = 2

    def __init__(self, *args, **kwargs):
        super(DeformConvPack, self).__init__(*args, **kwargs)
        self.conv_offset = nn.Conv2d(self.in_channels, self.deformable_groups * 2 * self.kernel_size[0] * self.kernel_size[1],
                                     kernel_size=self.kernel_size, stride=_pair(self.stride), padding=_pair(self.padding), bias=True)
        self.init_offset()

    def init_offset(self):
        self.conv_offset.weight.data.zero_()
        self.conv_offset.bias.data.zero_()

    def forward(self, x):
        offset = self.conv_offset(x)
        return deform_conv(x, offset, self.weight, self.stride, self.padding, self.dilation, self.groups, self.deformable_groups)

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, *rest):
        _rename_legacy_offset_keys(state_dict, prefix, local_metadata)
        super()._load_from_state_dict(state_dict, prefix, local_metadata, *rest)


class ModulatedDeformConv(nn.Module):
    """deform_conv.py:326-374"""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 deformable_groups=1, bias=True):
        super(ModulatedDeformConv, self).__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size = _pair(kernel_size)
        self.stride, self.padding, self.dilation = stride, padding, dilation
        self.groups, self.deformable_groups = groups, deformable_groups
        self.with_bias = bias
        self.transposed, self.output_padding = False, _single(0)
        self.weight = nn.Parameter(torch.Tensor(out_channels, in_channels // groups, *self.kernel_size))
        if bias:
            self.bias = nn.Parameter(torch.Tensor(out_channels))
        else:
            self.register_parameter('bias', None)
        self.reset_parameters()

    def reset_parameters(self):
        _uniform_fan_in(self.weight, self.in_channels, self.kernel_size)
        if self.bias is not None:
            self.bias.data.zero_()

    def forward(self, x, offset, mask):
        return modulated_deform_conv(x, offset, mask, self.weight, self.bias, self.stride, self.padding, self.dilation,
                                     self.groups, self.deformable_groups)


class ModulatedDeformConvPack(ModulatedDeformConv):
    """deform_conv.py:377-446: offsets and the sigmoid mask come from one plain convolution (3 * kh * kw channels)"""
    _version = 2

    def __init__(self, *args, **kwargs):
        super(ModulatedDeformConvPack, self).__init__(*args, **kwargs)
        self.conv_offset = nn.Conv2d(self.in_channels, self.deformable_groups * 3 * self.kernel_size[0] * self.kernel_size[1],
                                     kernel_size=self.kernel_size, stride=_pair(self.stride), padding=_pair(self.padding), bias=True)
        self.init_offset()

    def init_offset(self):
        self.conv_offset.weight.data.zero_()
        self.conv_offset.bias.data.zero_()

    def forward(self, x):
        o1, o2, mask = torch.chunk(self.conv_offset(x), 3, dim=1)
        return modulated_deform_conv(x, torch.cat((o1, o2), dim=1), torch.sigmoid(mask), self.weight, self.bias, self.stride,
                                     self.padding, self.dilation, self.groups, self.deformable_groups)

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, *rest):
        _rename_legacy_offset_keys(state_dict, prefix, local_metadata)
        super()._load_from_state_dict(state_dict, prefix, local_metadata, *rest)
