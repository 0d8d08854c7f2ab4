"""GPU: the N-tile pairs of the deformable plan (csrc/dense_tc.cu: both 128-wide N tiles of an M tile in one CTA, the A operand
sampled once per M tile, epilogue from the accumulator fragments) at a production size - the head DCN of one 1024 x 1024 tile, the five FPN levels in one launch -
against deform_conv_ref (oracle/torch_reference.py) in fp64.

Offsets are random and large (many samples leave the image), or carry NaN and +-inf (the sample is then zero), with and
without a DCNv2 mask.  Each case launches twice into outputs pre-filled with different NaN patterns between guard
regions: the results must be bitwise equal and the guards untouched."""
import pytest
import torch

from orientedreppoints_b200 import _lib

from test_conv_plans_gpu import DCN_F16X3_TOL, PATTERNS, Guarded, _rel

pytestmark = pytest.mark.gpu

LEVELS = [(1, 128, 128), (1, 64, 64), (1, 32, 32), (1, 16, 16), (1, 8, 8)]


def _offsets(mode, n, h, w, g):
    """[N, 18, H, W]: random with a spread of 4 pixels; "nonfinite": 5 % each NaN, +inf and -inf on top"""
    off = torch.randn(n, 18, h, w, generator=g) * 4.0
    if mode.startswith("nonfinite"):
        r = torch.rand(off.shape, generator=g)
        off[r < 0.05] = float("nan")
        off[(r >= 0.05) & (r < 0.10)] = float("inf")
        off[(r >= 0.10) & (r < 0.15)] = -float("inf")
    return off


def _oracle(x, off, wt, mask):
    """deform_conv_ref in fp64 at the sample positions the kernel forms: the tap's integer position plus the offset,
    rounded to fp32.  A NaN or infinite position fails the validity test (the tap adds 0): it is replaced by one far
    outside the image, which fails the same test"""
    from oracle import torch_reference as tr
    _, _, h, w = x.shape
    hb = (torch.arange(h, device=off.device) - 1).view(1, h, 1).double()
    wb = (torch.arange(w, device=off.device) - 1).view(1, 1, w).double()
    pos = off.double().clone()
    for t in range(9):
        i, j = divmod(t, 3)
        for c, base in ((2 * t, hb + i), (2 * t + 1, wb + j)):
            pos[:, c] = (base.float() + off[:, c].float()).double() - base
    pos = torch.where(torch.isfinite(pos), pos, torch.full_like(pos, -1e4))
    return torch.relu(tr.deform_conv_ref(x.double(), pos, wt.double(), 1, 1, 1, mask=None if mask is None else mask.double()))


@pytest.mark.parametrize("mode", ["random", "random_mask", "nonfinite", "nonfinite_mask"])
def test_dcn_pairs_vs_fp64(cuda, mode):
    from orientedreppoints_b200.detector import ConvLayer
    from orientedreppoints_b200.engine_tc import EngineTCSplit
    eng = EngineTCSplit(cuda)
    g = torch.Generator().manual_seed(len(mode))
    wt = torch.randn(256, 256, 3, 3, generator=g) / 48.0                 # 1 / sqrt(K)
    L = ConvLayer(wt, None, 1, 1, cuda)
    xs, offs, masks, refs, outs = [], [], [], [], []
    for n, h, w in LEVELS:
        x = torch.randn(n, 256, h, w, generator=g).to(cuda)
        off = _offsets(mode, n, h, w, g).to(cuda)
        m = torch.rand(n, 9, h, w, generator=g).to(cuda) if mode.endswith("mask") else None
        xs.append(eng.from_float(x.permute(0, 2, 3, 1)))
        offs.append(off.permute(0, 2, 3, 1).contiguous())
        masks.append(None if m is None else m.permute(0, 2, 3, 1).contiguous())
        refs.append(_oracle(x, off, wt.to(cuda), m))
        outs.append(Guarded((n, h, w, 2, 256), torch.float16, cuda))
    eng.overflow_count()
    bits, plan = [], None
    for pat in PATTERNS:
        for o in outs:
            o.fill(pat)
        eng._launch(xs, [o.t for o in outs], eng._tc(L), 256, 3, 3, 256, 1, 1, None, 1, False, True, offsets=offs,
                    masks=None if masks[0] is None else masks)
        plan = _lib.tc_last_plan()
        torch.cuda.synchronize()
        for o in outs:
            assert o.guards_intact(pat), "a store landed outside the output"
        bits.append([o.bits() for o in outs])
    for i, (a, b) in enumerate(zip(*bits)):
        assert torch.equal(a, b), "level %d: outputs differ between launches" % i
    assert (plan["BN"], plan["n_tiles_n"], plan["n_pair"], plan["dcat"], plan["stages"]) == (128, 2, 2, 1, 2), plan
    assert plan["num_tiles"] > 2 * plan["grid"]                           # some CTAs compute several pairs
    errs = []
    for o, ref in zip(outs, refs):
        y = eng.to_float(o.t).permute(0, 3, 1, 2)
        assert bool(torch.isfinite(y).all())
        errs.append(_rel(y, ref))
    assert eng.overflow_count() == 0
    print("%s: %d tiles on %d CTAs, rel err per level %s" % (mode, plan["num_tiles"], plan["grid"], ["%.2e" % e for e in errs]))
    assert max(errs) < DCN_F16X3_TOL, (errs, DCN_F16X3_TOL)
