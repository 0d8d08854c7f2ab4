"""CPU: the launch plans of the wgmma convolution, from the dry run orp_tc_plan_conv (the planner the launches use, run
without a device on a 132-SM H100).  Every parity case of tests/conv_plan_cases.py must plan to its signature, the way the
engine launches it; tests/test_conv_plans_gpu.py checks on the GPU that the launch reports the same plan, field for field.
The argument checks of the convolution entry points answer the dry run with the same errors."""
import pytest

from orientedreppoints_b200 import _lib

from conv_plan_cases import PARITY, SIG_FIELDS, case_id, planned, signature


@pytest.mark.parametrize("c", PARITY, ids=[case_id(c) for c in PARITY])
def test_parity_case_plans(c):
    p = planned(c)
    assert signature(p) == c[0], "the case left its plan: %s" % dict(zip(SIG_FIELDS, signature(p)))
    assert len(p["BW"]) == p["nprob"] and all(bw * bh * bi == 128 for bw, bh, bi in zip(p["BW"], p["BH"], p["BI"]))
    assert 1 <= p["grid"] <= min(p["num_tiles"], 132)


def test_grid_follows_the_sm_count():
    """a launch with more tiles than SMs runs one persistent CTA per SM"""
    args = ([(1, 133, 130)], 256, 256, 3, 3, 256, 1, 1)
    assert _lib.tc_plan_for(*args)["grid"] == 132
    assert _lib.tc_plan_for(*args, sms=100)["grid"] == 100


def _refused(match, *args, **kw):
    with pytest.raises(_lib.OrpError, match=r"\(-1\): " + match):
        _lib.tc_plan_for(*args, **kw)


@pytest.mark.parametrize("stride", [0, -1, 257])
def test_stride_outside_the_tile(stride):
    _refused("conv2d_tc: stride must be in 1..256", [(1, 300, 300)], 64, 64, 1, 1, 64, stride, 0)


def test_cin_multiple_of_8():
    _refused(r"conv2d_tc: Cin must be a multiple of 8", [(1, 16, 16)], 64, 64, 1, 1, 12, 1, 0)


def test_deformable_cin_multiple_of_64():
    _refused(r"conv2d_tc: deformable conv needs Cin % 64 == 0", [(1, 16, 16)], 64, 64, 3, 3, 96, 1, 1, deform=True)


@pytest.mark.parametrize("split,n", [(1, 64), (0, 128)])
def test_deformable_input_past_32_bit_offsets(split, n):
    _refused(r"conv2d_tc: deformable input has 2\^31", [(n, 256, 256)], 256, 256, 3, 3, 256, 1, 1, deform=True, split=split)
    _lib.tc_plan_for([(n, 256, 255)], 256, 256, 3, 3, 256, 1, 1, deform=True, split=split)


def test_split_k_preconditions():
    base = ([(1, 16, 16)], 256, 256, 3, 3, 256, 1, 1)
    assert _lib.tc_plan_for(*base, ksplit=3)["ksplit"] == 3
    _refused("conv2d_tc: split-K serves one plain problem", *base, ksplit=2)                 # 9 taps % 2
    _refused("conv2d_tc: split-K serves one plain problem", *base, ksplit=3, residual=1)
    _refused("conv2d_tc: split-K serves one plain problem", *base, ksplit=3, residual=2)
    _refused("conv2d_tc_splitk: bad arguments", [(1, 16, 16)], 15, 32, 3, 3, 256, 1, 1, ksplit=3)   # Cout % 8
    _refused("conv2d_tc_splitk: bad problem", [(1, 1, 1)], 256, 256, 3, 3, 256, 1, 0, ksplit=3)
    _refused("orp_tc_plan_conv: the stem and split-K plan one problem", [(1, 16, 16)] * 2, 256, 256, 3, 3, 256, 1, 1, ksplit=3)


def test_problem_and_output_checks():
    _refused("conv2d_tc: bad problem", [(1, 1, 1)], 64, 64, 3, 3, 64, 1, 0)                 # empty output map
    _refused("conv2d_tc: padded Cout must be a multiple of 32", [(1, 16, 16)], 64, 48, 1, 1, 64, 1, 0)
    _refused("conv2d_f16x3: 16-bit outputs need Cout % 8 == 0", [(1, 16, 16)], 20, 32, 1, 1, 64, 1, 0, split=True)
    _refused("conv2d_f16x3: fp32 outputs take an fp32 residual only", [(1, 16, 16)], 32, 32, 1, 1, 64, 1, 0, split=True,
             out_f32=True, residual=1)
    _refused("stem_conv_s2d_bf16: needs even H, W", [(1, 15, 16)], 64, 64, 4, 1, 64, 1, 0, stem=2)
