"""R-101 against X-101-32x4d and X-101-64x4d: the dense graph (backbone + FPN + head) of a batch of 1024 x 1024 tiles replayed as
one CUDA graph per model, in f16x3 and in bf16, at 4 tiles (the batch of the benchmark's R-101 configuration) and 16 tiles,
timed with CUDA events
    python tools/perf_resnext.py [replays=3] [rounds=5]
The three models alternate in every round (a round times `replays` replays of each); the step time reported per model is the
median over the rounds.  Then every grouped conv2 launch of the two ResNeXt models alone at 16 tiles, timed over 20 launches,
alternating with the zero-CUDA alternative on the same shape: the block-diagonal dense weight [width, width, 3, 3] through
orp_conv2d_* (width / gw times the useful MMA work).  Per launch: useful TFLOP/s (2 * pixels * width * 9 * gw), bytes/s counting
the input read once and the output written once, and which of the two bounds limits it against the H100 SXM data sheet
(989 TFLOP/s dense fp16 / bf16, 3.35 TB/s; an f16x3 product is three MMAs, a product of a group narrower than 16 is padded to 16).
Prints the card's name and power limit and one JSON line."""
import json
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, '.')
from orientedreppoints_b200 import _lib  # noqa: E402
from orientedreppoints_b200.detector import ConvLayer, OrientedRepPointsDetector  # noqa: E402
from orientedreppoints_b200.engine_tc import EngineTC, EngineTCSplit  # noqa: E402
from orientedreppoints_b200.weights import random_state_dict  # noqa: E402

R = int(sys.argv[1]) if len(sys.argv) > 1 else 3
ROUNDS = int(sys.argv[2]) if len(sys.argv) > 2 else 5
MODELS = (("R-101", 1, 4), ("X-101-32x4d", 32, 4), ("X-101-64x4d", 64, 4))
PEAK_FLOPS, PEAK_BW = 989e12, 3.35e12
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


steps = {}
for prec in ("f16x3", "bf16"):
    for tiles in (4, 16):
        img = torch.randn(tiles, 3, 1024, 1024, generator=torch.Generator().manual_seed(0)).to(dev)
        models = {}
        for name, groups, bw in MODELS:
            sd = random_state_dict(101, seed=0, reference_init=False, residual_gain=0.3, groups=groups, base_width=bw)
            det = OrientedRepPointsDetector(sd, 101, dev, prec)
            det.capture(img.shape)
            det.forward_dense_graph(img)
            models[name] = det
        torch.cuda.synchronize()
        times = {k: [] for k in models}
        for _ in range(ROUNDS):
            for name, det in models.items():
                times[name].append(events_ms(lambda: det.forward_dense_graph(img), R))
        for k, v in times.items():
            med = statistics.median(v)
            steps["%s/%s/%d" % (k, prec, tiles)] = dict(ms=round(med, 3), rounds=[round(t, 3) for t in v])
            print("%-12s %-5s %2d tiles %9.2f ms / step  (%.1f tiles/s; rounds %s)" % (k, prec, tiles, med, tiles * 1e3 / med,
                                                                                      " ".join("%.2f" % t for t in v)))
        if prec == "f16x3":
            for det in models.values():
                assert det.eng.overflow_count() == 0
        del models, det
        torch.cuda.empty_cache()

# every grouped conv2 launch alone at 16 tiles: (width, groups, input H = W, stride)
B = 16
shapes = []
for groups in (32, 64):
    for li in range(4):
        width, h = (64 << li) * 4 * groups // 64, 256 >> li
        if li > 0:
            shapes.append((width, groups, 2 * h, 2))
        shapes.append((width, groups, h, 1))
launches = {}
g = torch.Generator().manual_seed(1)
for prec, E in (("f16x3", EngineTCSplit), ("bf16", EngineTC)):
    e = E(dev)
    for width, groups, h, s in shapes:
        gw = width // groups
        ho = (h - 1) // s + 1
        x = e.from_float(torch.relu(torch.randn(B, h, h, width, generator=g)).to(dev))
        wt = torch.randn(width, gw, 3, 3, generator=g) * (2.0 / (9 * gw)) ** 0.5
        b = torch.randn(width, generator=g) * 0.1
        L = ConvLayer(wt, b, s, 1, dev)
        dense = torch.zeros(width, width, 3, 3)                              # the block-diagonal dense equivalent
        for k in range(groups):
            dense[k * gw:(k + 1) * gw, k * gw:(k + 1) * gw] = wt[k * gw:(k + 1) * gw]
        Ld = ConvLayer(dense, b, s, 1, dev)
        fns = {"group": lambda: e.group_conv(x, L, groups, relu=True), "dense": lambda: e.conv(x, Ld, relu=True)}
        ya, yb = fns["group"](), fns["dense"]()
        torch.cuda.synchronize()
        diff = float((e.to_float(ya) - e.to_float(yb)).abs().max()) if prec == "f16x3" else float((ya.float() - yb.float()).abs().max())
        t = {k: [] for k in fns}
        for _ in range(3):
            for k, fn in fns.items():
                fn()
                t[k].append(events_ms(fn, 20))
        tg, td = statistics.median(t["group"]), statistics.median(t["dense"])
        flops = 2.0 * B * ho * ho * width * 9 * gw
        planes = 2 if prec == "f16x3" else 1
        nbytes = 2.0 * planes * width * (B * h * h + B * ho * ho)
        mma = flops * (3 if prec == "f16x3" else 1) * max(16, gw) / gw
        t_c, t_m = mma / PEAK_FLOPS, nbytes / PEAK_BW
        e.group_conv(x, L, groups, relu=True)
        p = _lib.tc_last_plan()
        key = "%s/C%d-g%d-H%d-s%d" % (prec, width, groups, h, s)
        launches[key] = dict(group_ms=round(tg, 4), dense_ms=round(td, 4), speedup=round(td / tg, 2),
                             useful_tflops=round(flops / tg / 1e9, 2), gbps=round(nbytes / tg / 1e6, 1),
                             bound="memory" if t_m >= t_c else "compute", of_bound=round(max(t_c, t_m) * 1e3 / tg, 3),
                             max_abs_diff_vs_dense=diff, plan="stages%d grid%d b_resident%d epi_merge%d" % (
                                 p["stages"], p["grid"], p["b_resident"], p["epi_merge"]))
        r = launches[key]
        print("%-5s C%-4d g%-2d gw%-2d H%-3d s%d  grouped %.3f ms  dense %.3f ms  x%.2f  %.1f useful TFLOP/s  %.0f GB/s  %s-bound "
              "%.0f%% of it  (%s)" % (prec, width, groups, gw, h, s, tg, td, r["speedup"], r["useful_tflops"], r["gbps"], r["bound"],
                                     100 * r["of_bound"], r["plan"]))
        del x, ya, yb, L, Ld
    if prec == "f16x3":
        assert e.overflow_count() == 0
slower = [k for k, v in launches.items() if v["speedup"] <= 1.0]
print("grouped launches not faster than the dense block-diagonal route:", slower or "none")
print(json.dumps({"tool": "perf_resnext", "card": card, "tile": 1024, "replays": R, "rounds": ROUNDS, "steps": steps,
                  "launches_16_tiles": launches, "not_faster_than_dense": slower}))
