"""Swin-T/w7, Swin-S/w7, Swin-B/w7 and Swin-B/w12 steps: the dense graph (backbone + FPN + head) of a batch of 1024 x 1024 tiles
replayed as one CUDA graph per model, timed with CUDA events, in f16x3 and in bf16
    python tools/perf_swin.py [tiles=8] [replays=5] [rounds=5]
Within a format the four models alternate in every round (a round times `replays` replays of each); the step time reported per
model is the median over the rounds.  Then every window-attention launch of Swin-B at that batch (the four stage shapes, 7x7 and
12x12 windows, shifted) and the wide LayerNorms (Swin-B's 2048-wide and Swin-L's 3072-wide PatchMerging norm) alone, timed over
20 launches.  Weights: swin.random_swin_state_dict(0, arch).  Prints the card's name and power limit and one JSON line."""
import json
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, '.')
from orientedreppoints_b200 import _lib  # noqa: E402
from orientedreppoints_b200.detector import OrientedRepPointsDetector  # noqa: E402
from orientedreppoints_b200.engine_tc import EngineTC, EngineTCSplit  # noqa: E402
from orientedreppoints_b200.swin import ARCHS, random_swin_state_dict  # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 8
R = int(sys.argv[2]) if len(sys.argv) > 2 else 5
ROUNDS = int(sys.argv[3]) if len(sys.argv) > 3 else 5
MODELS = {"Swin-T/w7": "swin_tiny", "Swin-S/w7": "swin_small", "Swin-B/w7": "swin_base", "Swin-B/w12": "swin_base_w12"}
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
step, rounds = {}, {}
for prec in ("f16x3", "bf16"):
    models = {}
    for label, name in MODELS.items():
        det = OrientedRepPointsDetector(random_swin_state_dict(0, arch=ARCHS[name]), name, dev, prec)
        det.capture(img.shape)
        det.forward_dense_graph(img)
        models[label] = det
    torch.cuda.synchronize()
    times = {k: [] for k in models}
    for _ in range(ROUNDS):
        for label, det in models.items():
            times[label].append(events_ms(lambda: det.forward_dense_graph(img), R))
    for label in models:
        key = "%s %s" % (label, prec)
        step[key], rounds[key] = statistics.median(times[label]), times[label]
        print("%-17s %8.2f ms / step of %d tiles  (%.1f tiles/s; rounds %s)" % (key, step[key], B, B * 1e3 / step[key],
                                                                              " ".join("%.2f" % t for t in times[label])))
    if prec == "f16x3":
        for det in models.values():
            assert det.eng.overflow_count() == 0
    del models, det
    torch.cuda.empty_cache()

# every attention launch of Swin-B (heads 4 / 8 / 16 / 32) and the wide LayerNorms alone, at the batch above
lib = _lib.lib()
launches = {}
g = torch.Generator(device=dev).manual_seed(1)
for prec, e in (("f16x3", EngineTCSplit(dev)), ("bf16", EngineTC(dev))):
    for i in range(4):
        h, heads = 256 >> i, 4 << i
        c = heads * 32
        for ws, fn in ((7, "orp_window_attention_%s" % prec), (12, "orp_window_attention12_%s" % prec)):
            hp = -(-h // ws) * ws
            qkv = e.from_float(torch.randn(B, hp, hp, 3 * c, generator=g, device=dev))
            table = torch.randn((2 * ws - 1) ** 2, heads, generator=g, device=dev) * 0.5
            out = e.alloc(B, h, h, c)

            def attn():
                _lib.check(getattr(lib, fn)(_lib.ptr(qkv), B, h, h, hp, hp, c, heads, ws // 2, _lib.ptr(table), 32 ** -0.5,
                                            _lib.ptr(out), _lib.current_stream_ptr()), fn)
            for _ in range(3):
                attn()
            ms = events_ms(attn, 20)
            key = "attn w%d %s H%d heads%d" % (ws, prec, h, heads)
            launches[key] = round(ms, 4)
            print("%-36s %8.4f ms" % (key, ms))
            del qkv, out
    for cw, h in ((2048, 32), (3072, 32)):                 # Swin-B / Swin-L stage-2 PatchMerging norm: 4 x 512 / 4 x 768 wide
        x = e.from_float(torch.randn(B, h, h, cw, generator=g, device=dev))
        gamma, beta = torch.ones(cw, device=dev), torch.zeros(cw, device=dev)
        y = e.alloc(B, h, h, cw)

        def ln():
            _lib.check(getattr(lib, "orp_layernorm_wide_%s" % prec)(_lib.ptr(x), B, h, h, cw, _lib.ptr(gamma), _lib.ptr(beta), 1e-5,
                                                                     h, h, _lib.ptr(y), _lib.current_stream_ptr()), "ln")
        for _ in range(3):
            ln()
        ms = events_ms(ln, 20)
        key = "layernorm_wide %s C%d H%d" % (prec, cw, h)
        launches[key] = round(ms, 4)
        print("%-36s %8.4f ms" % (key, ms))
print(json.dumps({"tool": "perf_swin", "card": card, "tiles": B, "tile": 1024, "step_ms_median": {k: round(v, 3) for k, v in step.items()},
                  "step_ms_rounds": {k: [round(t, 3) for t in v] for k, v in rounds.items()}, "launch_ms": launches}))
