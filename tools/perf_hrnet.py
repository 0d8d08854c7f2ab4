"""R-50 against HRNetV2p-W18, W32 and W40 (+ HRFPN): the dense graph (backbone + neck + head) of a batch of 1024 x 1024 tiles
replayed as one CUDA graph per model, in f16x3 and in bf16, at 4 and 16 tiles, timed with CUDA events
    python tools/perf_hrnet.py [replays=3] [rounds=5]
The four models alternate in every round (a round times `replays` replays of each); the step time reported per model is the
median over the rounds.  Then every launch of orp_hr_fuse / orp_hrfpn_reduce / orp_hrfpn_pool that the W18, W32 and W40 graphs
make at 16 tiles, alone, timed over 20 launches (median of 3): bytes counted from shapes (every input element read once,
every output written once; fp32 parts of the reduction, 2 bytes per value in bf16, 4 in f16x3) and the achieved bandwidth as a
share of the H100 SXM's 3.35 TB/s.  Prints the card's name and power limit and one JSON line."""
import json
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, '.')
from orientedreppoints_b200.detector import OrientedRepPointsDetector  # noqa: E402
from orientedreppoints_b200.engine_tc import EngineTC, EngineTCSplit  # noqa: E402
from orientedreppoints_b200.hrnet import ARCHS, pad8  # noqa: E402
from orientedreppoints_b200.weights import random_hrnet_state_dict, random_state_dict  # noqa: E402

R = int(sys.argv[1]) if len(sys.argv) > 1 else 3
ROUNDS = int(sys.argv[2]) if len(sys.argv) > 2 else 5
MODELS = ("R-50", "hrnetv2p_w18", "hrnetv2p_w32", "hrnetv2p_w40")
PEAK_BW = 3.35e12
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


def detector(name, prec):
    if name == "R-50":
        return OrientedRepPointsDetector(random_state_dict(50, seed=0, reference_init=False), 50, dev, prec)
    return OrientedRepPointsDetector(random_hrnet_state_dict(name, seed=0, reference_init=False, residual_gain=0.3), name, dev, prec)


steps = {}
for prec in ("f16x3", "bf16"):
    for tiles in (4, 16):
        img = torch.randn(tiles, 3, 1024, 1024, generator=torch.Generator().manual_seed(0)).to(dev)
        models = {}
        for name in MODELS:
            det = detector(name, prec)
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
            print("%-13s %-5s %2d tiles %9.2f ms / step  (%.1f tiles/s; rounds %s)" % (k, prec, tiles, med, tiles * 1e3 / med,
                                                                                       " ".join("%.2f" % t for t in v)))
        if prec == "f16x3":
            for det in models.values():
                assert det.eng.overflow_count() == 0
        del models, det
        torch.cuda.empty_cache()

# every launch of the three HRNet kernels at 16 tiles of 1024^2: the stage-4 branch maps are 256 >> i on a side
B, S = 16, 256
launches = {}
g = torch.Generator().manual_seed(1)
for prec, E in (("f16x3", EngineTCSplit), ("bf16", EngineTC)):
    e = E(dev)
    vb = 4 if prec == "f16x3" else 2                                # bytes per activation value
    calls = set()
    for name in MODELS[1:]:
        st = ARCHS[name].stages
        for s in st[1:]:
            w = [pad8(c) for c in s.widths]
            for i in range(len(w) - 1):
                calls.add(("fuse", w[i], S >> i, len(w) - 1 - i))
    calls = sorted(calls) + [("reduce", 256, S, 4), ("pool_avg", 256, S, 0), ("pool_max", 256, S, 1)]
    for kind, c, h, k in calls:
        if kind == "fuse":
            base = e.from_float(torch.randn(B, h, h, c, generator=g).to(dev)) if prec == "f16x3" else \
                torch.randn(B, h, h, c, generator=g).to(dev, torch.bfloat16)
            srcs = [e.alloc(B, h >> j, h >> j, c, zero=True) for j in range(1, k + 1)]
            fn = (lambda base=base, srcs=srcs: e.hr_fuse(base, srcs))
            nbytes = vb * c * B * (2 * h * h + sum((h >> j) ** 2 for j in range(1, k + 1)))
            key = "%s/fuse-C%d-%d-src%d" % (prec, c, h, k)
        elif kind == "reduce":
            parts = [torch.randn(B, h >> j, h >> j, c, generator=g).to(dev) for j in range(4)]
            fn = (lambda parts=parts: e.hrfpn_reduce(parts))
            nbytes = 4 * c * B * sum((h >> j) ** 2 for j in range(4)) + vb * c * B * h * h
            key = "%s/reduce-C%d-%d" % (prec, c, h)
        else:
            x = e.alloc(B, h, h, c, zero=True)
            fn = (lambda x=x, k=k: e.hrfpn_pool(x, k))
            nbytes = vb * c * B * (h * h + sum((h >> j) ** 2 for j in range(1, 5)))
            key = "%s/%s-C%d-%d" % (prec, kind, c, h)
        fn()
        t = statistics.median(events_ms(fn, 20) for _ in range(3))
        launches[key] = dict(ms=round(t, 4), gbps=round(nbytes / t / 1e6, 1), of_hbm=round(nbytes / t / 1e-3 / PEAK_BW, 3))
        print("%-32s %.4f ms  %7.0f GB/s  %4.0f%% of 3.35 TB/s" % (key, t, launches[key]["gbps"], 100 * launches[key]["of_hbm"]))
        torch.cuda.empty_cache()
print(json.dumps({"tool": "perf_hrnet", "card": card, "tile": 1024, "replays": R, "rounds": ROUNDS, "steps": steps,
                  "launches_16_tiles": launches}))
