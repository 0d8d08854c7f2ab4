"""Speed of the FPN_CARAFE neck on the GPU: whole R-50 FPN against R-50 FPN_CARAFE (GN, the default upsample_cfg: up_kernel 5,
up_group 1, encoder_kernel 3, compressed_channels 64) steps, and every orp_carafe_add launch of FPN_CARAFE alone.

    python tools/perf_fpn_carafe.py [--reps 5] [--out perf_fpn_carafe.json]

Step times: 16 and 4 tiles of 1024^2, f16x3 and bf16, the dense graph (backbone + neck + head) captured as one CUDA graph per
model, models alternating, median of `reps` rounds of 10 replays.  Launch times: CUDA events over 50 launches after 5 warm-up
launches, at the four top-down steps of 1024^2 tiles (8 -> 16, 16 -> 32, 32 -> 64, 64 -> 128).  Bytes of a launch: x, the fp32
logits and the residual read once, y written once.  Bandwidth share: bytes / time over the H100 SXM data sheet's 3.35 TB/s.
The card's name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from orientedreppoints_b200 import carafe_fpn as cf                                # noqa: E402
from orientedreppoints_b200.detector import OrientedRepPointsDetector               # noqa: E402
from orientedreppoints_b200.weights import fpn_carafe_spec, random_state_dict      # noqa: E402

SPEC = fpn_carafe_spec((512, 1024, 2048), 256, dict(type='GN', num_groups=32))
MODELS = [("R-50 FPN", None), ("R-50 FPN_CARAFE", SPEC)]
HBM = 3.35e12                                           # H100 SXM data sheet, bytes/s


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def step_times(fmt, batch, reps, dev):
    img = torch.randn(batch, 3, 1024, 1024, device=dev)
    dets = {name: OrientedRepPointsDetector(random_state_dict(50, seed=0, neck=spec), 50, dev, fmt, neck=spec).capture(tuple(img.shape))
            for name, spec in MODELS}
    times = {k: [] for k in dets}
    for _ in range(reps):
        for name, d in dets.items():                                   # models alternate
            d.forward_dense_graph(img)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(10):
                d.forward_dense_graph(img)
            b.record()
            torch.cuda.synchronize()
            times[name].append(a.elapsed_time(b) / 10)
    del dets
    torch.cuda.empty_cache()
    return {k: round(statistics.median(v), 3) for k, v in times.items()}


def timed(fn):
    for _ in range(5):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(50):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 50 * 1e-3


def launch_times(fmt, batch, dev):
    from orientedreppoints_b200.engine_tc import EngineTC, EngineTCSplit
    e = EngineTCSplit(dev) if fmt == "f16x3" else EngineTC(dev)
    k, g = SPEC['up_kernel'], SPEC['up_group']
    out = []
    for h in (8, 16, 32, 64):
        x = e.from_float(torch.randn(batch, h, h, 256, device=dev))
        r = e.from_float(torch.randn(batch, 2 * h, 2 * h, 256, device=dev))
        logits = torch.randn(batch, h, h, k * k * g * 4, device=dev)
        t = timed(lambda: cf.carafe_add(e, x, logits, k, g, r))
        nbytes = x.numel() * x.element_size() + logits.numel() * 4 + 2 * r.numel() * r.element_size()
        out.append(dict(step="%d->%d" % (h, 2 * h), us=round(t * 1e6, 1), bytes=nbytes,
                        share_of_3_35_TBps=round(nbytes / t / HBM, 3)))
        del x, r, logits
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_fpn_carafe needs a GPU: there is no CPU measurement")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = dict(card=card(), tile=1024)
    for fmt in ("f16x3", "bf16"):
        for batch in (16, 4):
            res["%s_x%d" % (fmt, batch)] = dict(step_ms=step_times(fmt, batch, a.reps, dev), launches=launch_times(fmt, batch, dev))
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
