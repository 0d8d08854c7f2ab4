"""Time the DOTA mAOE evaluation (orientedreppoints_b200.dota.aoe_evaluation) on the seeded synthetic set of
tools/perf_eval.py, the size of the DOTA-v1.0 validation split: ~460 images of ~4000^2 px, ~30 000 objects over 15
classes, ~10^6 Task1 detections.

    python tools/perf_aoe.py [--images 460] [--objects 65] [--copies 29] [--fp 300] [--reps 5] [--ref-dets 2000]

Prints one JSON line: the card (name and power limit, read-only nvidia-smi query), the device time of the
orp_dota_eval_aoe call (CUDA events, after a warm-up, median of --reps) and of the whole device part (upload, call, the
one copy back; host clock after a synchronise), and, for context, the time of the numpy restatement of the reference's
per-detection loop (tests/aoe_ref.py) on a bounded sample of one class.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=460)
    ap.add_argument("--objects", type=float, default=65.0, help="mean objects per image")
    ap.add_argument("--copies", type=int, default=29, help="jittered detections per object")
    ap.add_argument("--fp", type=int, default=300, help="random false positives per image")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-dets", type=int, default=2000, help="detections of the restatement sample (0: skip)")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("perf_aoe.py measures the GPU evaluation and needs a CUDA device")
    from perf_eval import gpu_identity, synth
    from orientedreppoints_b200.dota import aoe_evaluation as ae
    from orientedreppoints_b200.dota import evaluation as ev
    from orientedreppoints_b200.dota.pipeline import DOTA_CLASSES
    name, power = gpu_identity()
    dev = torch.device("cuda", 0)

    gts, dets = synth(args.images, args.objects, args.copies, args.fp)
    nd = sum(len(v) for v in dets.values())
    ng = sum(len(v) for v in gts.values())
    arrays, nimg, _ = ev._host_arrays(dets, gts, DOTA_CLASSES)
    arrays = arrays[:7]

    inputs = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in arrays]
    ae._launch(inputs, len(DOTA_CLASSES), nimg, 0.7, dev)            # warm-up
    torch.cuda.synchronize()
    call_ms, device_ms = [], []
    for _ in range(args.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ae._launch(inputs, len(DOTA_CLASSES), nimg, 0.7, dev)
        e1.record()
        torch.cuda.synchronize()
        call_ms.append(e0.elapsed_time(e1))
        t0 = time.perf_counter()
        ins = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in arrays]
        buf, _ = ae._launch(ins, len(DOTA_CLASSES), nimg, 0.7, dev)
        buf.cpu()
        device_ms.append((time.perf_counter() - t0) * 1e3)
    res = ae.evaluate_aoe(dets, gts, DOTA_CLASSES, 0.7)

    out = {"gpu": name, "power_limit": power, "images": nimg, "gt_objects": ng, "detections": nd,
           "matched": sum(res["n"].values()), "aoe_call_ms_median": round(float(np.median(call_ms)), 3),
           "aoe_call_ms": [round(v, 3) for v in call_ms],
           "device_part_ms_median": round(float(np.median(device_ms)), 3), "maoe": res["maoe"]}
    if args.ref_dets > 0:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import aoe_ref
        from oracle import ref_driver
        c = "small-vehicle"
        f = [l.split(' ') for l in dets[c][:args.ref_dets]]
        gt = {img: np.array([o['bbox'] for o in objs if o['name'] == c], np.float64).reshape(-1, 8)
              for img, objs in gts.items()}
        t0 = time.perf_counter()
        aoe_ref.aoe_class([x[0] for x in f], np.array([float(x[1]) for x in f]),
                          np.array([[float(v) for v in x[2:]] for x in f]), gt, 0.7)
        dt = time.perf_counter() - t0
        out["restatement_sample"] = {"what": "numpy restatement of aoe_eval's per-detection loop, one class, IoU from %s"
                                             % ("the reference's compiled SWIG polyiou" if ref_driver._swig() else "the C port"),
                                     "detections": len(f), "seconds": round(dt, 3),
                                     "us_per_detection": round(dt / len(f) * 1e6, 1)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
