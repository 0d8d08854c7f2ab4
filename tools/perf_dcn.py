"""the head's deformable convolution (cls_dcn / ref_dcn: 256 -> 256, 3x3, the five FPN levels of a 1024 x 1024 tile batch in
one launch) alone, f16x3, timed with CUDA events
    python tools/perf_dcn.py [tiles=16] [launches=30]
Prints the launch plan, ms per launch, algorithmic TFLOP/s and the bilinear gather's bytes per second.  Gathered bytes
are counted from the shapes: an M tile is sampled once per N tile, or once per N-tile pair (n_pair = 2), and each sampling
reads 4 corners x 128 pixels x 256 B (hi and lo planes of 64 channels) per tap and channel block."""
import sys
import torch
sys.path.insert(0, '.')
from orientedreppoints_b200 import _lib
from orientedreppoints_b200.detector import ConvLayer
from orientedreppoints_b200.engine_tc import EngineTCSplit

B = int(sys.argv[1]) if len(sys.argv) > 1 else 16
R = int(sys.argv[2]) if len(sys.argv) > 2 else 30
dev = torch.device('cuda', 0)
e = EngineTCSplit(dev)
g = torch.Generator().manual_seed(0)
cin = cout = 256
L = ConvLayer(torch.randn(cout, cin, 3, 3, generator=g) / (cin * 9) ** 0.5, None, 1, 1, dev)
sizes = [1024 // s for s in (8, 16, 32, 64, 128)]
xs = [e.from_float(torch.randn(B, s, s, cin, generator=g).to(dev)) for s in sizes]
offs = [(torch.randn(B, s, s, 18, generator=g) * 2.0).to(dev).contiguous() for s in sizes]


def run():
    return e.deform_conv_multi(xs, offs, L, relu=True)


for _ in range(5):
    run()
torch.cuda.synchronize()
plan = _lib.tc_last_plan()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(R):
    run()
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / R
pix = sum(B * s * s for s in sizes)
flops = 2.0 * pix * cout * cin * 9
mtiles = plan["num_tiles"] // plan["n_tiles_n"]
npair = plan.get("n_pair") or 1                 # (0 from a library that predates the field)
gathered = float(mtiles) * (plan["n_tiles_n"] // npair) * 9 * (cin // 64) * 128 * 4 * 256
assert e.overflow_count() == 0
print("dcn %d tiles: BN=%d n_tiles_n=%d n_pair=%d stages=%d grid=%d  %.3f ms  %.1f TFLOP/s algorithmic  %.1f GB/s gathered (%.2f GB)"
      % (B, plan["BN"], plan["n_tiles_n"], npair, plan["stages"], plan["grid"], ms, flops / ms / 1e9, gathered / ms / 1e6,
         gathered / 1e9))
