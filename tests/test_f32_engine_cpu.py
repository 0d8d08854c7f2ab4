"""CPU: the argument checks of the fp32 CUDA-core entry points (csrc/dense_f32.cu).  Every refusal is ORP_EINVAL with a
message, returned before the device is touched and before any arithmetic on the arguments: no launch is counted, and on a
host without a GPU the call does not reach the no-device error.  The pointers are placeholders that are only tested for
NULL; every call here is refused, so none is dereferenced."""
import re

import pytest

from orientedreppoints_b200 import _lib

ORP_EINVAL = -1
PH = 256                                            # a non-NULL placeholder address


def _conv_args(**kw):
    a = dict(x=PH, N=2, H=16, W=16, Cin=64, w=PH, Cout=64, KH=3, KW=3, stride=1, pad=1, bias=None, residual=None, relu=0,
             y=PH, gn_stats=None, groups=32, stream=None)
    a.update(kw)
    return list(a.values())


def _deform_args(**kw):
    a = dict(x=PH, N=2, H=16, W=16, Cin=64, offset=PH, mask=None, w=PH, Cout=64, KH=3, KW=3, stride=1, pad=1, dilation=1,
             bias=None, relu=0, y=PH, stream=None)
    a.update(kw)
    return list(a.values())


def _gn_args(**kw):
    a = dict(x=PH, N=2, H=16, W=16, C=256, stats=PH, groups=32, gamma=PH, beta=PH, eps=1e-5, relu=0, up_src=None, y=PH,
             stream=None)
    a.update(kw)
    return list(a.values())


def _pool_args(**kw):
    a = dict(x=PH, N=2, H=16, W=16, C=64, y=PH, stream=None)
    a.update(kw)
    return list(a.values())


ARGS = {"orp_conv2d_f32": _conv_args, "orp_deform_conv2d_f32": _deform_args, "orp_gn_apply_f32": _gn_args,
        "orp_maxpool3x3s2_f32": _pool_args}

CONV_SIZES = "N, H, W, Cin, Cout, KH and KW must be >= 1"
CONV_GEOM = "stride and dilation must be >= 1, pad >= 0"
CONV_EMPTY = "the kernel does not fit the padded input"

# (id, entry point, overrides, message after "<name>: ")
CASES = [
    # orp_conv2d_f32
    ("conv-stride0", "orp_conv2d_f32", dict(stride=0), CONV_GEOM),
    ("conv-stride-1", "orp_conv2d_f32", dict(stride=-1), CONV_GEOM),
    ("conv-pad-3", "orp_conv2d_f32", dict(pad=-3), CONV_GEOM),
    ("conv-7x7-on-1x1", "orp_conv2d_f32", dict(H=1, W=1, KH=7, KW=7, pad=0), CONV_EMPTY),        # Ho = Wo = -5 before
    ("conv-7x7-on-1x1-stride2", "orp_conv2d_f32", dict(H=1, W=1, Cin=4, KH=7, KW=7, stride=2, pad=0), CONV_EMPTY),
    ("conv-Ho0", "orp_conv2d_f32", dict(H=2, KH=3, KW=1, pad=0), CONV_EMPTY),                   # Ho = 0, Wo = 16
    ("conv-Wo0", "orp_conv2d_f32", dict(W=2, KH=1, KW=3, pad=0), CONV_EMPTY),                   # Ho = 16, Wo = 0
    ("conv-Ho-truncated", "orp_conv2d_f32", dict(H=2, KH=3, KW=1, stride=2, pad=0), CONV_EMPTY),  # -1 / 2 + 1 = 1
    ("conv-Ho-negative-Wo-negative", "orp_conv2d_f32", dict(H=1, W=1, KH=5, KW=5, pad=1), CONV_EMPTY),  # product positive
    ("conv-KH0", "orp_conv2d_f32", dict(KH=0), CONV_SIZES),
    ("conv-KW0", "orp_conv2d_f32", dict(KW=0), CONV_SIZES),
    ("conv-KH-1", "orp_conv2d_f32", dict(KH=-1), CONV_SIZES),
    ("conv-N0", "orp_conv2d_f32", dict(N=0), CONV_SIZES),
    ("conv-N-1", "orp_conv2d_f32", dict(N=-1), CONV_SIZES),
    ("conv-H0", "orp_conv2d_f32", dict(H=0), CONV_SIZES),
    ("conv-W-1", "orp_conv2d_f32", dict(W=-1), CONV_SIZES),
    ("conv-Cin0", "orp_conv2d_f32", dict(Cin=0), CONV_SIZES),
    ("conv-Cout0", "orp_conv2d_f32", dict(Cout=0), CONV_SIZES),
    ("conv-Cin6", "orp_conv2d_f32", dict(Cin=6), "Cin must be a multiple of 4"),
    ("conv-w-null", "orp_conv2d_f32", dict(w=None), "x, w and y must not be NULL"),
    ("conv-x-null", "orp_conv2d_f32", dict(x=None), "x, w and y must not be NULL"),
    ("conv-y-null", "orp_conv2d_f32", dict(y=None), "x, w and y must not be NULL"),
    ("conv-stats-groups0", "orp_conv2d_f32", dict(gn_stats=PH, groups=0), "Cout must divide into groups >= 1"),
    ("conv-stats-groups-1", "orp_conv2d_f32", dict(gn_stats=PH, groups=-1), "Cout must divide into groups >= 1"),
    ("conv-stats-groups-not-dividing", "orp_conv2d_f32", dict(gn_stats=PH, groups=24), "Cout must divide into groups >= 1"),
    # orp_deform_conv2d_f32
    ("deform-stride0", "orp_deform_conv2d_f32", dict(stride=0), CONV_GEOM),
    ("deform-dilation0", "orp_deform_conv2d_f32", dict(dilation=0), CONV_GEOM),
    ("deform-dilation-1", "orp_deform_conv2d_f32", dict(dilation=-1), CONV_GEOM),
    ("deform-pad-1", "orp_deform_conv2d_f32", dict(pad=-1), CONV_GEOM),
    ("deform-dilated-kernel-too-large", "orp_deform_conv2d_f32", dict(H=4, W=4, dilation=3, pad=0), CONV_EMPTY),
    ("deform-KW0", "orp_deform_conv2d_f32", dict(KW=0), CONV_SIZES),
    ("deform-N-1", "orp_deform_conv2d_f32", dict(N=-1), CONV_SIZES),
    ("deform-w-null", "orp_deform_conv2d_f32", dict(w=None), "x, w and y must not be NULL"),
    ("deform-offset-null", "orp_deform_conv2d_f32", dict(offset=None), "offset is NULL"),
    # orp_gn_apply_f32
    ("gn-groups0", "orp_gn_apply_f32", dict(groups=0), "C must divide into groups >= 1"),      # SIGFPE before (C % 0)
    ("gn-groups-1", "orp_gn_apply_f32", dict(groups=-1), "C must divide into groups >= 1"),
    ("gn-groups-not-dividing", "orp_gn_apply_f32", dict(groups=24), "C must divide into groups >= 1"),
    ("gn-N-1", "orp_gn_apply_f32", dict(N=-1), "N, H, W and C must be >= 1"),
    ("gn-N0", "orp_gn_apply_f32", dict(N=0), "N, H, W and C must be >= 1"),
    ("gn-H0", "orp_gn_apply_f32", dict(H=0), "N, H, W and C must be >= 1"),
    ("gn-W-1", "orp_gn_apply_f32", dict(W=-1), "N, H, W and C must be >= 1"),
    ("gn-C0", "orp_gn_apply_f32", dict(C=0, groups=1), "N, H, W and C must be >= 1"),
    ("gn-C6", "orp_gn_apply_f32", dict(C=6, groups=2), "C must be a multiple of 4"),
    ("gn-stats-null", "orp_gn_apply_f32", dict(stats=None), "x, stats, gamma, beta and y must not be NULL"),
    ("gn-gamma-null", "orp_gn_apply_f32", dict(gamma=None), "x, stats, gamma, beta and y must not be NULL"),
    ("gn-y-null", "orp_gn_apply_f32", dict(y=None), "x, stats, gamma, beta and y must not be NULL"),
    # orp_maxpool3x3s2_f32
    ("pool-N-1", "orp_maxpool3x3s2_f32", dict(N=-1), "N, H, W and C must be >= 1"),
    ("pool-N0", "orp_maxpool3x3s2_f32", dict(N=0), "N, H, W and C must be >= 1"),
    ("pool-H0", "orp_maxpool3x3s2_f32", dict(H=0), "N, H, W and C must be >= 1"),
    ("pool-W0", "orp_maxpool3x3s2_f32", dict(W=0), "N, H, W and C must be >= 1"),
    ("pool-C0", "orp_maxpool3x3s2_f32", dict(C=0), "N, H, W and C must be >= 1"),
    ("pool-C6", "orp_maxpool3x3s2_f32", dict(C=6), "C must be a multiple of 4"),
    ("pool-x-null", "orp_maxpool3x3s2_f32", dict(x=None), "x and y must not be NULL"),
]


@pytest.mark.parametrize("c", CASES, ids=[c[0] for c in CASES])
def test_refused(c):
    _, ep, kw, msg = c
    lib = _lib.lib()
    before = _lib.launch_count()
    rc = getattr(lib, ep)(*ARGS[ep](**kw))
    err = lib.orp_last_error().decode()
    assert rc == ORP_EINVAL, (rc, err)
    assert re.fullmatch(re.escape(ep[len("orp_"):] + ": " + msg) + ".*", err), err
    assert _lib.launch_count() == before, "a refused call launched"
