"""CPU: the N-tile pairs of the head's deformable convolution (cls_dcn / ref_dcn: 256 -> 256, 3x3, the five FPN levels of a
batch of 1024 x 1024 tiles in one launch), from the dry run orp_tc_plan_conv on a 132-SM H100.

A CTA computes both 128-wide N tiles of an M tile on one sampled A operand (n_pair = 2), so every sample is gathered once
per M tile instead of once per N tile.  Pairs need f16x3 operands and a 16-bit output (the fragment epilogue writes through
the TMA store); every other deformable launch keeps one N tile per CTA: bf16, fp32 outputs (the NCHW operator surface),
128 output channels (one N tile) and GELU."""
import pytest

from orientedreppoints_b200 import _lib

SMEM_PER_BLOCK = 227 * 1024        # what one H100 thread block can opt into
STATIC_DEFORM = 14336              # static shared memory the planner sets aside for the deformable variant
ACC_PASS = 128 * 68 * 4            # the staged accumulator pass the other variants keep (kAccBytes)


def _levels(batch):
    return [(batch, 1024 // s, 1024 // s) for s in (8, 16, 32, 64, 128)]


def _dcn(probs, cout=256, **kw):
    kw.setdefault("split", True)
    return _lib.tc_plan_for(probs, cout, cout, 3, 3, 256, 1, 1, relu=1, deform=True, **kw)


# the bench workloads' head DCN: R-50 x16, R-101 x4, Swin-T x8 and x1 tiles per step
@pytest.mark.parametrize("batch", [16, 4, 8, 1], ids=["r50x16", "r101x4", "swinx8", "x1"])
def test_production_dcn_runs_n_tile_pairs(batch):
    p = _dcn(_levels(batch))
    assert (p["BN"], p["n_tiles_n"], p["n_pair"], p["stages"], p["dcat"], p["tma_epi"]) == (128, 2, 2, 2, 1, 1), p
    assert (p["epi_merge"], p["gn_fused"], p["out_f32"]) == (0, 0, 0), p
    assert p["grid"] == 132 and p["num_tiles"] > 2 * p["grid"]
    # two 96 KiB stages (x_hi | x_lo | w_hi | w_lo of a K block, both N tiles) and one 16 KiB output staging tile fit beside
    # the static shared memory only without the staged accumulator pass
    stage = 2 * 128 * 128 + 2 * 256 * 128
    dyn = 1024 + p["stages"] * stage + p["epi_bufs"] * 16384
    assert dyn + STATIC_DEFORM <= SMEM_PER_BLOCK
    assert dyn + ACC_PASS + STATIC_DEFORM > SMEM_PER_BLOCK


def test_small_launch_pairs_too():
    """the pairing does not depend on the size: the small DCN parity case of tests/conv_plan_cases.py runs it too"""
    p = _dcn([(5, 33, 33), (5, 17, 17), (5, 9, 9), (5, 5, 5), (5, 3, 3)])
    assert (p["BN"], p["n_tiles_n"], p["n_pair"]) == (128, 2, 2), p
    assert p["grid"] == min(p["num_tiles"] // 2, 132)


@pytest.mark.parametrize("what", ["bf16", "out_f32", "cout128", "gelu"])
def test_other_deformable_plans_do_not_pair(what):
    probs = _levels(16)
    if what == "bf16":
        p = _dcn(probs, split=False)
    elif what == "out_f32":
        p = _dcn(probs, out_f32=True)
    elif what == "cout128":
        p = _dcn(probs, cout=128)
    elif what == "gelu":
        p = _lib.tc_plan_for(probs, 256, 256, 3, 3, 256, 1, 1, relu=2, deform=True, split=True)
    assert p["BN"] == 128 and p["n_tiles_n"] == p["Cout_padded"] // 128 and p["n_pair"] == 1, p
