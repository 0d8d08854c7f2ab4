"""R-50 against R-50-DCN and R-50-DCNv2 (deformable conv2 in c3-c5), f16x3, the dense graph (backbone + FPN + head) of a
16-tile batch of 1024 x 1024 tiles replayed as one CUDA graph each, timed with CUDA events
    python tools/perf_dcn_backbone.py [tiles=16] [replays=10] [rounds=5]
The three models alternate in every round (a round times `replays` replays of each); the step time reported per model is
the median over the rounds.  Then every new backbone launch alone at the same batch, timed over 20 launches: the offset
convolution, the DCNv2 offset / mask split, and the deformable conv2 in DCN and DCNv2 form.  The weights are random with
offsets of 1-2 pixels rms in every stage (weights.random_state_dict(residual_gain=0.3, dcn_offset_scale=1)), so the gather
leaves the grid as a trained model's does.  Prints the card's name and power limit and one JSON line."""
import json
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, '.')
from orientedreppoints_b200 import _lib  # noqa: E402
from orientedreppoints_b200.detector import ConvLayer, OrientedRepPointsDetector  # noqa: E402
from orientedreppoints_b200.weights import dcn_layout, random_state_dict  # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 16
R = int(sys.argv[2]) if len(sys.argv) > 2 else 10
ROUNDS = int(sys.argv[3]) if len(sys.argv) > 3 else 5
C3_C5 = (False, True, True, True)
dev = torch.device('cuda', 0)
torch.cuda.set_device(dev)
card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print("card:", card)


def events_ms(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


img = torch.randn(B, 3, 1024, 1024, generator=torch.Generator().manual_seed(0)).to(dev)
models = {}
for name, kind in (("R-50", None), ("R-50-DCN", "DCN"), ("R-50-DCNv2", "DCNv2")):
    dcn = None if kind is None else dict(type=kind)
    sd = random_state_dict(50, seed=0, reference_init=False, residual_gain=0.3, dcn=dcn, stage_with_dcn=C3_C5,
                           dcn_offset_scale=1.0)
    det = OrientedRepPointsDetector(sd, 50, dev, "f16x3", dcn=None if kind is None else dcn_layout(50, dcn, C3_C5))
    det.capture(img.shape)
    det.forward_dense_graph(img)
    models[name] = det
torch.cuda.synchronize()
times = {k: [] for k in models}
for _ in range(ROUNDS):
    for name, det in models.items():
        times[name].append(events_ms(lambda: det.forward_dense_graph(img), R))
step = {k: statistics.median(v) for k, v in times.items()}
for k in models:
    print("%-11s %8.2f ms / step of %d tiles  (%.1f tiles/s; rounds %s)" % (k, step[k], B, B * 1e3 / step[k],
                                                                          " ".join("%.2f" % t for t in times[k])))
for det in models.values():
    assert det.eng.overflow_count() == 0
del models
torch.cuda.empty_cache()

# every new launch alone, f16x3, at the batch above: (planes, input H = W, stride) of c3-c5
from orientedreppoints_b200.engine_tc import EngineTCSplit  # noqa: E402
e = EngineTCSplit(dev)
g = torch.Generator().manual_seed(1)
launches = {}
for planes, h, s in [(128, 256, 2), (128, 128, 1), (256, 128, 2), (256, 64, 1), (512, 64, 2), (512, 32, 1)]:
    ho = (h - 1) // s + 1
    x = e.from_float(torch.relu(torch.randn(B, h, h, planes, generator=g)).to(dev))
    L = ConvLayer(torch.randn(planes, planes, 3, 3, generator=g) * (2.0 / (9 * planes)) ** 0.5, torch.randn(planes, generator=g) * 0.1,
                  s, 1, dev)
    Lo = ConvLayer(torch.randn(27, planes, 3, 3, generator=g) / (9 * planes) ** 0.5, torch.randn(27, generator=g), s, 1, dev)
    om = e.conv(x, Lo, out_f32=True)
    off = torch.empty((B, ho, ho, 18), device=dev)
    mask = torch.empty((B, ho, ho, 9), device=dev)

    def split():
        _lib.check(_lib.lib().orp_dcnv2_offset_mask(_lib.ptr(om), B * ho * ho, _lib.ptr(off), _lib.ptr(mask),
                                                    _lib.current_stream_ptr()), "orp_dcnv2_offset_mask")

    split()
    fns = {"offset_conv27": lambda: e.conv(x, Lo, out_f32=True), "offset_mask_split": split,
           "dcn": lambda: e.deform_conv(x, off, L, relu=True), "dcnv2": lambda: e.deform_conv(x, off, L, relu=True, mask=mask)}
    row = {}
    for k, fn in fns.items():
        for _ in range(3):
            fn()
        row[k] = round(events_ms(fn, 20), 4)
    e.deform_conv(x, off, L, relu=True)
    p = _lib.tc_last_plan()
    row["plan"] = "BN%d n_pair%d stages%d grid%d" % (p["BN"], p["n_pair"], p["stages"], p["grid"])
    launches["C%d-H%d-s%d" % (planes, h, s)] = row
    print("C%-4d H%-4d s%d  offset conv %.3f ms  split %.3f ms  DCN %.3f ms  DCNv2 %.3f ms  (%s)"
          % (planes, h, s, row["offset_conv27"], row["offset_mask_split"], row["dcn"], row["dcnv2"], row["plan"]))
assert e.overflow_count() == 0
print(json.dumps({"tool": "perf_dcn_backbone", "card": card, "tiles": B, "tile": 1024, "precision": "f16x3",
                  "step_ms_median": {k: round(v, 3) for k, v in step.items()},
                  "step_ms_rounds": {k: [round(t, 3) for t in v] for k, v in times.items()}, "launch_ms": launches}))
