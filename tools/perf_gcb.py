"""Speed of the global context blocks (GCB) on the GPU: whole R-50 steps without GCB, with GCB r16 on c3-c5 ('att',
channel_add) and with GCB r4 on c3-c5 ('att', channel_add + channel_mul), and every pool, transform and fuse launch of those
layouts alone.

    python tools/perf_gcb.py [--reps 5] [--out perf_gcb.json]

Step times: 16 and 4 tiles of 1024^2, f16x3 and bf16, the dense graph (backbone + FPN + head) captured as one CUDA graph per
model, models alternating, median of `reps` rounds of 10 replays.  Launch times: CUDA events over 50 launches after 5 warm-up
launches, on the c3 / c4 / c5 maps of 1024^2 tiles.  Bytes of a launch: pool, x read once; fuse, x and the identity read and y
written; transform, the partials and the MLP weights read.  Bandwidth share: bytes / time over the H100 SXM data sheet's 3.35
TB/s.  The card's name and power limit are read in the same run."""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from orientedreppoints_b200 import _lib                                             # noqa: E402
from orientedreppoints_b200.context_block import ContextBlock                       # noqa: E402
from orientedreppoints_b200.detector import OrientedRepPointsDetector               # noqa: E402
from orientedreppoints_b200.weights import gcb_layout, gcb_spec, random_state_dict  # noqa: E402

C3_C5 = (False, True, True, True)
MODELS = [("R-50", None), ("R-50-GCB r16 c3-c5", dict(ratio=1. / 16.)),
          ("R-50-GCB r4 c3-c5 add+mul", dict(ratio=1. / 4., fusion_types=('channel_add', 'channel_mul')))]
HBM = 3.35e12                                           # H100 SXM data sheet, bytes/s
SUFFIX = {"bf16": "bf16", "f16x3": "f16x3"}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def detector(gcb, fmt, dev):
    kw = {} if gcb is None else dict(gcb=gcb, stage_with_gcb=C3_C5)
    sd = random_state_dict(50, seed=0, **kw)
    return OrientedRepPointsDetector(sd, 50, dev, fmt, gcb=None if gcb is None else gcb_layout(50, gcb, C3_C5))


def step_times(fmt, batch, reps, dev):
    img = torch.randn(batch, 3, 1024, 1024, device=dev)
    dets = {name: detector(g, fmt, dev).capture(tuple(img.shape)) for name, g in MODELS}
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
    bpe = 4 if fmt == "f16x3" else 2
    lib, stream = _lib.lib(), None
    out = []
    for name, gcb in MODELS[1:]:
        for li, h in ((1, 128), (2, 64), (3, 32)):
            c = 256 << li
            stages = [False] * 4
            stages[li] = True
            sd = random_state_dict(50, seed=1, reference_init=False, gcb=gcb, stage_with_gcb=stages, gcb_gain=1.0)
            blk = ContextBlock(sd, "backbone.layer%d.0" % (li + 1), gcb_spec(gcb, c), dev)
            x = e.from_float(torch.randn(batch, h, h, c, device=dev))
            idt = e.from_float(torch.randn(batch, h, h, c, device=dev))
            y = e.alloc(batch, h, h, c)
            plan = _lib.context_plan_for(fmt, batch, h, h, c)
            ws = torch.empty(plan["workspace_bytes"] // 4, dtype=torch.float32, device=dev)
            rows = {f: torch.empty(batch, c, dtype=torch.float32, device=dev) for f in blk.mlps}
            add, mul = blk.mlps.get('channel_add'), blk.mlps.get('channel_mul')
            stream = _lib.current_stream_ptr()
            pool = getattr(lib, "orp_context_pool_" + SUFFIX[fmt])
            fuse = getattr(lib, "orp_context_fuse_" + SUFFIX[fmt])
            t_pool = timed(lambda: pool(_lib.ptr(x), batch, h, h, c, _lib.ptr(blk.mask_w), _lib.ptr(ws), ws.numel() * 4, stream))
            t_tr = timed(lambda: lib.orp_context_transform(_lib.ptr(ws), batch, plan["chunks"], c, blk.planes,
                                                           ctypes.byref(add[0]) if add else None,
                                                           ctypes.byref(mul[0]) if mul else None, _lib.ptr(rows.get('channel_add')),
                                                           _lib.ptr(rows.get('channel_mul')), stream))
            t_fuse = timed(lambda: fuse(_lib.ptr(x), _lib.ptr(idt), batch, h, h, c, _lib.ptr(rows.get('channel_mul')),
                                        _lib.ptr(rows.get('channel_add')), _lib.ptr(y), stream))
            act = batch * h * h * c * bpe
            tr_bytes = ws.numel() * 4 * len(blk.mlps) + batch * len(blk.mlps) * (2 * c * blk.planes) * 4
            for kind, t, nbytes in (("pool", t_pool, act), ("transform", t_tr, tr_bytes), ("fuse", t_fuse, 3 * act)):
                out.append(dict(model=name, stage="c%d" % (li + 2), map=h, channels=c, planes=blk.planes, launch=kind,
                                us=round(t * 1e6, 1), bytes=nbytes, share_of_3_35_TBps=round(nbytes / t / HBM, 3)))
            del x, idt, y, ws, rows
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_gcb needs a GPU: there is no CPU measurement")
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
