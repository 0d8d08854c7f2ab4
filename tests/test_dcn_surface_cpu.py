"""CPU: which kernel a deformable convolution of the `mmdet.ops.dcn` surface (ops/dcn.py) runs on, and the host-side
preparation of the fp32 kernel's operands.  The tensor-core producers address the input with 32-bit element offsets, so
problems of 2^31 or more 16-bit input elements must go to the fp32 kernel; the library refuses them before touching a
device.  Like tests/test_abi.py, the library tests need liborp_b200.so as build() leaves it (they make no compute
call)."""
import ctypes

import pytest
import torch

from orientedreppoints_b200 import _lib
from orientedreppoints_b200.ops import dcn


@pytest.mark.parametrize("prec,n,h,w,cin,dil,want", [
    ("f16x3", 1, 33, 33, 256, 1, "tc"),          # the head's DCN
    ("f16x3", 16, 128, 128, 256, 1, "tc"),        # the detector's largest level at 16 tiles: 2^27 16-bit elements
    ("f16x3", 64, 256, 255, 256, 1, "tc"),        # 2^31 - 2^23
    ("f16x3", 64, 256, 256, 256, 1, "f32"),       # exactly 2^31 (hi and lo planes)
    ("bf16", 64, 256, 256, 256, 1, "tc"),         # the same tensor holds 2^30 bf16 elements
    ("bf16", 128, 256, 255, 256, 1, "tc"),        # 2^31 - 2^23
    ("bf16", 128, 256, 256, 256, 1, "f32"),       # exactly 2^31
    ("f16x3", 1, 65536, 32768, 64, 1, "f32"),
    ("f16x3", 1, 8, 8, 192, 1, "tc"),
    ("f16x3", 1, 8, 8, 96, 1, "f32"),            # Cin % 64
    ("bf16", 1, 8, 8, 3, 1, "f32"),
    ("f16x3", 1, 8, 8, 256, 2, "f32"),           # dilation
    ("bf16", 1, 8, 8, 64, 2, "f32"),
    ("fp32", 1, 8, 8, 256, 1, "f32"),
])
def test_route(prec, n, h, w, cin, dil, want):
    assert dcn._route(prec, n, h, w, cin, 1, dil) == want
    assert dcn._route(prec, n, h, w, cin, 256, dil) == want
    assert dcn._route(prec, n, h, w, cin, 257, dil) == "f32"     # beyond the tensor-core tile's 256 input columns


def _tc_call(split, n, h, w, stride=1):
    """a deformable orp_conv2d_* call whose problem has no input or output pointer (only the weight pointer must be
    non-NULL to get past the first check): whatever check rejects it, nothing is launched"""
    q = _lib.TcProblem()
    q.N, q.H, q.W = n, h, w
    l = _lib.lib()
    if split:
        rc = l.orp_conv2d_f16x3(1, ctypes.byref(q), 16, 256, 256, 3, 3, 256, stride, 1, None, 0, 0, 1, 1, None)
    else:
        rc = l.orp_conv2d_bf16(1, ctypes.byref(q), 16, 256, 256, 3, 3, 256, stride, 1, None, 0, 1, 1, None)
    return rc, l.orp_last_error()


@pytest.mark.parametrize("split,n,h,w", [(1, 64, 256, 256), (0, 128, 256, 256), (1, 128, 256, 256), (0, 1, 65536, 32768),
                                         (1, 1, 65536, 32768)])
def test_tensor_core_refuses_inputs_past_32_bit_offsets(split, n, h, w):
    """orp_conv2d_bf16 / orp_conv2d_f16x3 with a deformable problem (Cin 256) of >= 2^31 16-bit elements: ORP_EINVAL
    from the argument checks, which run before any device work"""
    assert n * h * w * 256 * (2 if split else 1) >= 1 << 31
    rc, err = _tc_call(split, n, h, w)
    assert rc == -1 and b"2^31" in err                # ORP_EINVAL, from the size check


@pytest.mark.parametrize("split", [0, 1])
@pytest.mark.parametrize("stride", [257, 1000, -1])
def test_tensor_core_refuses_strides_past_the_tile(split, stride):
    """a tile spans BW * stride <= 256 input columns with BW >= 1: other strides are ORP_EINVAL before any device work"""
    rc, err = _tc_call(split, 2, 300, 300, stride)
    assert rc == -1 and b"stride" in err


def test_fp32_operands_pad_cin_to_four():
    """any Cin: the fp32 kernel's weights are [Cout, KH, KW, Cin rounded up to 4], the extra channels exactly 0; the
    tensor-core engines keep the unpadded weights (they pad to 64 themselves)"""
    for cin in (1, 3, 4, 18, 30):
        wt = torch.randn(7, cin, 2, 3)
        L = dcn._W(wt, None, 1, 0)
        c4 = (cin + 3) // 4 * 4
        assert tuple(L.w.shape) == (7, 2, 3, c4) and L.w.is_contiguous()
        assert torch.equal(L.w[..., :cin], wt.permute(0, 2, 3, 1))
        assert not bool(L.w[..., cin:].any())
        assert torch.equal(L.w_raw, wt.permute(0, 2, 3, 1))


def test_weight_cache_follows_the_memory():
    """a cached layer is reused for the same weight memory - the tensor itself or any view of it, e.g. the
    `m.weight.detach()` a caller may pass on every call - and rebuilt when it is written in place or the key (address,
    layout, version, bias, stride, padding) differs.  The entry holds the weight's storage, so no new tensor can be placed
    at a cached address while the entry lives"""
    wt = torch.randn(8, 64, 3, 3)
    L = dcn._layer(wt, None, 1, 1)
    assert dcn._layer(wt, None, 1, 1) is L
    assert dcn._layer(wt.detach(), None, 1, 1) is L and dcn._layer(wt.view(8, 64, 3, 3), None, 1, 1) is L
    assert dcn._layer(wt, None, 2, 1) is not L and dcn._layer(wt, None, 1, 0) is not L
    assert dcn._layer(wt.view(8, 64, 9, 1), None, 1, 1) is not L
    assert dcn._layer(wt.transpose(2, 3), None, 1, 1) is not L           # same address and shape, another layout
    ptr = wt.data_ptr()
    entry = next(v for k, v in dcn._cache.items() if v[1] is L)
    del wt
    assert entry[0][0].data_ptr() == ptr                               # the memory stays with the entry
    wt = torch.randn(8, 64, 3, 3)
    L1 = dcn._layer(wt, None, 1, 1)
    with torch.no_grad():
        wt.mul_(2)
    L2 = dcn._layer(wt, None, 1, 1)
    assert L2 is not L1 and torch.equal(L2.w_raw, wt.permute(0, 2, 3, 1))
    with torch.no_grad():
        wt.detach().add_(1)                                            # a view's write bumps the shared counter
    L3 = dcn._layer(wt, None, 1, 1)
    assert L3 is not L2 and torch.equal(L3.w_raw, wt.permute(0, 2, 3, 1))
    b = torch.randn(8)
    Lb = dcn._layer(wt, b, 1, 1)
    assert Lb is not L3 and dcn._layer(wt, b, 1, 1) is Lb and dcn._layer(wt, b.detach(), 1, 1) is Lb
    with torch.no_grad():
        b.add_(1)
    assert dcn._layer(wt, b, 1, 1) is not Lb
