"""Time convex_giou (orp_convex_giou, csrc/convex_iou.cu) and the GIoULoss forward + backward (losses.py) on realistic
pairs: quadrilaterals of the SURVEY 8(d) generator (synth.gen_rotated_boxes, 4000^2 px) with 9 points scattered around
each of them.

    python tools/perf_giou.py [--sizes 4096 65536 1048576] [--reps 5]

Prints one JSON line: the card (name and power limit, read-only nvidia-smi query) and, per size, the device time of the
orp_convex_giou call and of GIoULoss forward + backward (CUDA events, after a warm-up, median of --reps).  There is no
GPU baseline: the reference's convex_giou_cuda does not build against current torch (it needs the THC headers).
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def pairs(n, seed=0):
    from orientedreppoints_b200.synth import gen_rotated_boxes
    rng = np.random.RandomState(seed)
    q = gen_rotated_boxes(n, seed=seed, extent=4000.0)[:, :8].astype(np.float64)
    c = q.reshape(n, 4, 2).mean(1)
    u, v = q[:, 2:4] - q[:, 0:2], q[:, 6:8] - q[:, 0:2]
    size = np.sqrt(np.abs(u[:, 0] * v[:, 1] - u[:, 1] * v[:, 0]))
    th = rng.uniform(-np.pi, np.pi, (n, 1))
    local = (rng.rand(n, 9, 2) - 0.5) * (size[:, None] * rng.uniform(0.3, 1.8, (n, 2)))[:, None, :]
    rot = np.stack([np.cos(th) * local[..., 0] - np.sin(th) * local[..., 1],
                    np.sin(th) * local[..., 0] + np.cos(th) * local[..., 1]], -1)
    shift = rng.normal(0, 0.3, (n, 1, 2)) * size[:, None, None]
    return (c[:, None, :] + rot + shift).reshape(n, 18).astype(np.float32), q.astype(np.float32)


def timed(fn, reps):
    import torch
    fn()                                                             # warm-up
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[4096, 65536, 1048576])
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("perf_giou.py measures the GPU operator and needs a CUDA device")
    from perf_eval import gpu_identity
    from orientedreppoints_b200 import _lib
    from orientedreppoints_b200.losses import GIoULoss
    name, power = gpu_identity()
    dev = torch.device("cuda", 0)
    L = _lib.lib()
    res = {"gpu": name, "power_limit": power, "reps": args.reps, "sizes": {}}
    for n in args.sizes:
        p, q = pairs(n)
        pred = torch.from_numpy(p).to(dev).requires_grad_(True)
        target = torch.from_numpy(q).to(dev)
        weight = torch.rand(n, device=dev)
        out = torch.empty((n, 19), device=dev)
        call = lambda: _lib.check(L.orp_convex_giou(_lib.ptr(pred), _lib.ptr(target), n, _lib.ptr(out),  # noqa: E731
                                                    _lib.current_stream_ptr()), "orp_convex_giou")
        loss_fn = GIoULoss(loss_weight=1.0)

        def fwd_bwd():
            pred.grad = None
            loss_fn(pred, target, weight).backward()

        res["sizes"][str(n)] = {"call_ms": round(timed(call, args.reps), 4),
                                "loss_fwd_bwd_ms": round(timed(fwd_bwd, args.reps), 4),
                                "nan_rows": int(torch.isnan(out).any(1).sum())}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
