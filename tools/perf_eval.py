"""Time the DOTA Task1 evaluation (orientedreppoints_b200.dota.evaluation) on a seeded synthetic set the size of the
DOTA-v1.0 validation split: ~460 images of ~4000^2 px, ~30 000 objects over 15 classes (10 % difficult), ~10^6 Task1
detections (jittered copies of the objects spanning IoU ~0.3-0.9, duplicates, random false positives).

    python tools/perf_eval.py [--images 460] [--objects 65] [--copies 29] [--fp 300] [--reps 5] [--oracle-dets 2000]

Prints one JSON line: the card (name and power limit, read-only nvidia-smi query), the host parse time of the Task1
lines, the device time of the orp_dota_eval_task1 call (CUDA events, after a warm-up, median of --reps) and of the whole
device part (upload, call, the one copy back; host clock after a synchronise), and, for context, the time of the oracle
restatement of the reference's per-detection Python loop (oracle/dota_eval_oracle.py) on a bounded sample of one class.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def synth(images, objects, copies, n_fp, seed=0, extent=4000.0):
    from orientedreppoints_b200.dota.pipeline import DOTA_CLASSES
    rng = np.random.RandomState(seed)

    def quads(cx, cy, w, h, a):
        c, s = np.cos(a)[:, None], np.sin(a)[:, None]
        px = np.array([-0.5, 0.5, 0.5, -0.5])[None] * w[:, None]
        py = np.array([-0.5, -0.5, 0.5, 0.5])[None] * h[:, None]
        x, y = cx[:, None] + c * px - s * py, cy[:, None] + s * px + c * py
        return np.round(np.stack([x, y], 2).reshape(-1, 8), 1)

    gts, per_class = {}, {c: [] for c in DOTA_CLASSES}
    for k in range(images):
        name = "V%04d" % k
        n = rng.poisson(objects)
        cls = rng.randint(0, len(DOTA_CLASSES), n)
        cx, cy = rng.uniform(0, extent, n), rng.uniform(0, extent, n)
        w, h, a = rng.uniform(10, 250, n), rng.uniform(8, 150, n), rng.uniform(-np.pi, np.pi, n)
        gq = quads(cx, cy, w, h, a)
        diff = rng.rand(n) < 0.1
        gts[name] = [{'name': DOTA_CLASSES[c], 'difficult': int(d), 'bbox': [float(v) for v in q]}
                     for c, d, q in zip(cls, diff, gq)]
        # jittered copies: relative jitter j in [0, 0.4] spans IoU ~0.9 down to ~0.3
        rep = np.repeat(np.arange(n), copies)
        j = rng.uniform(0, 0.4, rep.size)
        dq = quads(cx[rep] + rng.normal(0, 1, rep.size) * j * w[rep] / 3, cy[rep] + rng.normal(0, 1, rep.size) * j * h[rep] / 3,
                   w[rep] * (1 + rng.normal(0, 1, rep.size) * j / 3), h[rep] * (1 + rng.normal(0, 1, rep.size) * j / 3),
                   a[rep] + rng.normal(0, 1, rep.size) * j)
        dcls = cls[rep]
        fq = quads(rng.uniform(0, extent, n_fp), rng.uniform(0, extent, n_fp), rng.uniform(10, 250, n_fp),
                   rng.uniform(8, 150, n_fp), rng.uniform(-np.pi, np.pi, n_fp))
        dq = np.concatenate([dq, fq])
        dcls = np.concatenate([dcls, rng.randint(0, len(DOTA_CLASSES), n_fp)])
        for c in range(len(DOTA_CLASSES)):
            per_class[DOTA_CLASSES[c]].append((name, dq[dcls == c]))
    dets = {}
    for c, parts in per_class.items():
        total = sum(len(q) for _, q in parts)
        scores = (rng.permutation(total) + 1) / (total + 1.0)
        lines, i = [], 0
        for name, q in parts:
            for row in q:
                lines.append("%s %r %s" % (name, float(scores[i]), " ".join(repr(float(v)) for v in row)))
                i += 1
        dets[c] = lines
    return gts, dets


def gpu_identity():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [s.strip() for s in out.split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=460)
    ap.add_argument("--objects", type=float, default=65.0, help="mean objects per image")
    ap.add_argument("--copies", type=int, default=29, help="jittered detections per object")
    ap.add_argument("--fp", type=int, default=300, help="random false positives per image")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-dets", type=int, default=2000, help="detections of the oracle sample (0: skip)")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("perf_eval.py measures the GPU evaluation and needs a CUDA device")
    from orientedreppoints_b200.dota import evaluation as ev
    from orientedreppoints_b200.dota.pipeline import DOTA_CLASSES
    name, power = gpu_identity()
    dev = torch.device("cuda", 0)

    gts, dets = synth(args.images, args.objects, args.copies, args.fp)
    nd = sum(len(v) for v in dets.values())
    ng = sum(len(v) for v in gts.values())
    t0 = time.perf_counter()
    arrays, nimg, _ = ev._host_arrays(dets, gts, DOTA_CLASSES)
    host_parse_s = time.perf_counter() - t0

    inputs = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in arrays]
    ev._launch(inputs, len(DOTA_CLASSES), nimg, 0.5, True, dev)       # warm-up
    torch.cuda.synchronize()
    call_ms, device_ms = [], []
    for _ in range(args.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ev._launch(inputs, len(DOTA_CLASSES), nimg, 0.5, True, dev)
        e1.record()
        torch.cuda.synchronize()
        call_ms.append(e0.elapsed_time(e1))
        t0 = time.perf_counter()
        ins = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in arrays]
        buf, _ = ev._launch(ins, len(DOTA_CLASSES), nimg, 0.5, True, dev)
        buf.cpu()
        device_ms.append((time.perf_counter() - t0) * 1e3)
    res = ev.evaluate(dets, gts, DOTA_CLASSES, 0.5, True)

    out = {"gpu": name, "power_limit": power, "images": nimg, "gt_objects": ng, "detections": nd,
           "host_parse_s": round(host_parse_s, 3), "eval_call_ms_median": round(float(np.median(call_ms)), 3),
           "eval_call_ms": [round(v, 3) for v in call_ms],
           "device_part_ms_median": round(float(np.median(device_ms)), 3), "map_07": res["map"]}
    if args.oracle_dets > 0:
        from oracle import dota_eval_oracle as orc
        c = "small-vehicle"
        lines = dets[c][:args.oracle_dets]
        f = [l.split(' ') for l in lines]
        gt = {}
        for img, objs in gts.items():
            sel = [o for o in objs if o['name'] == c]
            gt[img] = (np.array([o['bbox'] for o in sel], np.float64).reshape(-1, 8),
                       np.array([o['difficult'] for o in sel]).astype(bool))
        t0 = time.perf_counter()
        orc.eval_class([x[0] for x in f], np.array([float(x[1]) for x in f]),
                       np.array([[float(v) for v in x[2:]] for x in f]), gt, 0.5, True)
        dt = time.perf_counter() - t0
        from oracle import ref_driver
        out["oracle_sample"] = {"what": "oracle restatement of voc_eval's per-detection Python loop, one class, IoU from %s"
                                        % ("the reference's compiled SWIG polyiou" if ref_driver._swig() else "the C port"),
                                "detections": len(lines), "seconds": round(dt, 3), "us_per_detection": round(dt / len(lines) * 1e6, 1)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
