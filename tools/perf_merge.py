"""Time ResultMerge over packed detections (orp_result_merge, dota.result_merge.merge_packed) followed by the Task1
evaluation, against the text path on the same detections, on a seeded synthetic set the size of the DOTA-v1.0 validation
split: ~460 images of 4000^2 px cut into 1024-px tiles with gap 200 (25 tiles each), objects of 15 classes, and for
every tile that sees an object a few jittered detections of it - so the merge has the cross-tile and in-tile
duplicates to suppress that the real one has.

    python tools/perf_merge.py [--images 460] [--objects 220] [--copies 6] [--cap 256] [--reps 5] [--text-limit 0]

Prints one JSON line: the card (name and power limit, read-only nvidia-smi query); the time of the orp_result_merge
call (CUDA events, after a warm-up, median of --reps; the events bracket merge_packed with the row bound given, so the
window also holds the allocation of the outputs and the read of the survivor count and status - an upper bound of the
library call); the time of merge_packed + evaluate_merged (host
clock after a synchronise); the text path on the same detections, stage by stage (pipeline.task1_lines,
result_merge.merge_lines for the 15 classes, evaluation.evaluate); and both paths' mAP, which must be equal.
--text-limit N bounds the text path to the first N images; both paths are then also compared on that subset.
Needs a CUDA device: there is no fallback.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def _quads(cx, cy, w, h, a):
    c, s = np.cos(a)[:, None], np.sin(a)[:, None]
    px = np.array([-0.5, 0.5, 0.5, -0.5])[None] * w[:, None]
    py = np.array([-0.5, -0.5, 0.5, 0.5])[None] * h[:, None]
    return np.stack([cx[:, None] + c * px - s * py, cy[:, None] + s * px + c * py], 2).reshape(-1, 8)


def synth_packed(images, objects, copies, cap, seed=0, extent=4000, subsize=1024, gap=200, ncls=15):
    """-> (packed fp32 [T, cap + 1, 28], tile_xy int32 [T,2], tile_rate fp64 [T], tile_img int32 [T], gts): per image
    `objects` (Poisson mean) boxes; every tile holds `copies` jittered detections of each object whose centre it
    contains (at most cap, in random order), with scores that rise with the fit.  gts: {image name: objects} as
    evaluation.parse_gt gives them (10 % difficult)."""
    from orientedreppoints_b200.dota.pipeline import DOTA_CLASSES
    from orientedreppoints_b200.dota.split_tiles import tile_origins
    rng = np.random.RandomState(seed)
    origins = np.asarray(tile_origins(extent, extent, subsize, gap), np.int32)
    t_img = len(origins)
    packed = np.zeros((images * t_img, cap + 1, 28), np.float32)
    gts = {}
    for k in range(images):
        n = rng.poisson(objects)
        cls = rng.randint(0, ncls, n)
        cx, cy = rng.uniform(0, extent, n), rng.uniform(0, extent, n)
        w, h, a = rng.uniform(10, 250, n), rng.uniform(8, 150, n), rng.uniform(-np.pi, np.pi, n)
        gq = np.round(_quads(cx, cy, w, h, a), 1)
        gts["V%04d" % k] = [{'name': DOTA_CLASSES[c], 'difficult': int(d), 'bbox': [float(v) for v in q]}
                            for c, d, q in zip(cls, rng.rand(n) < 0.1, gq)]
        for t, (l, u) in enumerate(origins):
            seen = np.flatnonzero((cx >= l) & (cx < l + subsize) & (cy >= u) & (cy < u + subsize))
            rep = rng.permutation(np.repeat(seen, copies))[:cap]
            j = rng.uniform(0, 0.4, rep.size)
            q = _quads(cx[rep] + rng.normal(0, 1, rep.size) * j * w[rep] / 3 - l, cy[rep] + rng.normal(0, 1, rep.size) * j * h[rep] / 3 - u,
                       w[rep] * (1 + rng.normal(0, 1, rep.size) * j / 3), h[rep] * (1 + rng.normal(0, 1, rep.size) * j / 3),
                       a[rep] + rng.normal(0, 1, rep.size) * j)
            slot = packed[k * t_img + t]
            slot[:rep.size, 18:26] = q
            slot[:rep.size, 26] = np.clip(1.0 - j * 2 + rng.normal(0, 0.05, rep.size), 0.01, 1.0)
            slot[:rep.size, 27] = cls[rep]
            slot[cap, 0] = rep.size
    return (packed, np.tile(origins, (images, 1)), np.ones(images * t_img), np.repeat(np.arange(images, dtype=np.int32), t_img),
            gts)


def gpu_identity():
    from perf_eval import gpu_identity as query                    # the same read-only nvidia-smi query
    return query()


def text_path(packed, tile_xy, tile_img, names, gts):
    """the same detections through pipeline.task1_lines -> merge_lines per class -> evaluate, each stage timed"""
    from orientedreppoints_b200.dota import evaluation as ev
    from orientedreppoints_b200.dota.pipeline import DOTA_CLASSES, task1_lines
    from orientedreppoints_b200.dota.result_merge import merge_lines
    cap = packed.shape[1] - 1
    results, tnames = [], []
    for t in range(packed.shape[0]):                                # what rbbox2result hands over: per class [k, 27]
        rows = packed[t, :int(packed[t, cap, 0])]
        results.append([rows[rows[:, 27] == c, :27] for c in range(len(DOTA_CLASSES))])
        tnames.append("%s__1__%d___%d" % (names[tile_img[t]], tile_xy[t, 0], tile_xy[t, 1]))
    t0 = time.perf_counter()
    per_class = task1_lines(results, tnames)
    t1 = time.perf_counter()
    merged = {c: merge_lines(lines) for c, lines in zip(DOTA_CLASSES, per_class)}
    t2 = time.perf_counter()
    res = ev.evaluate(merged, gts)
    t3 = time.perf_counter()
    return merged, res, {"task1_lines_s": round(t1 - t0, 3), "merge_lines_x15_s": round(t2 - t1, 3),
                         "evaluate_s": round(t3 - t2, 3), "total_s": round(t3 - t0, 3),
                         "lines_in": sum(map(len, per_class)), "lines_merged": sum(map(len, merged.values()))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=460)
    ap.add_argument("--objects", type=float, default=220.0, help="mean objects per image")
    ap.add_argument("--copies", type=int, default=6, help="detections of an object per tile that sees it")
    ap.add_argument("--cap", type=int, default=256, help="detection capacity of a tile (max_per_img)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--text-limit", type=int, default=0, help="images of the text path (0: all)")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("perf_merge.py measures the GPU merge and needs a CUDA device")
    from orientedreppoints_b200.dota import evaluation as ev
    from orientedreppoints_b200.dota.pipeline import DOTA_CLASSES
    from orientedreppoints_b200.dota.result_merge import merge_packed
    name, power = gpu_identity()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)

    packed, xy, rate, img, gts = synth_packed(args.images, args.objects, args.copies, args.cap)
    names = list(gts)
    nimg = len(names)
    d_packed = torch.from_numpy(packed).to(dev)
    meta = [torch.arange(packed.shape[0], dtype=torch.int32).to(dev), torch.from_numpy(xy).to(dev),
            torch.from_numpy(rate).to(dev), torch.from_numpy(img).to(dev)]
    rows = int(packed[:, args.cap, 0].sum())

    def device_path(p, m, n, g, nm):
        merged = merge_packed(p, *m, n)
        return merged, ev.evaluate_merged(merged, g, nm)

    device_path(d_packed, meta, nimg, gts, names)                   # warm-up
    torch.cuda.synchronize()
    call_ms, path_ms = [], []
    for _ in range(args.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        merged = merge_packed(d_packed, *meta, nimg, max_rows=rows)  # the bound given: no read before the library call
        e1.record()
        torch.cuda.synchronize()
        call_ms.append(e0.elapsed_time(e1))
        t0 = time.perf_counter()
        merged, res = device_path(d_packed, meta, nimg, gts, names)
        torch.cuda.synchronize()
        path_ms.append((time.perf_counter() - t0) * 1e3)

    out = {"gpu": name, "power_limit": power, "images": nimg, "tiles": int(packed.shape[0]), "rows": rows,
           "survivors": len(merged), "gt_objects": sum(len(v) for v in gts.values()),
           "merge_call_ms_median": round(float(np.median(call_ms)), 3), "merge_call_ms": [round(v, 3) for v in call_ms],
           "merge_plus_evaluate_ms_median": round(float(np.median(path_ms)), 3),
           "merge_plus_evaluate_ms": [round(v, 3) for v in path_ms], "map_07_device": res["map"]}

    lim = nimg if args.text_limit <= 0 else min(args.text_limit, nimg)
    nt = int((img < lim).sum())
    sub_gts = {k: gts[k] for k in names[:lim]}
    lines, text_res, timing = text_path(packed[:nt], xy[:nt], img[:nt], names, sub_gts)
    if lim < nimg:
        sub_meta = [m[:nt] for m in meta]
        device_path(d_packed[:nt], sub_meta, lim, sub_gts, names[:lim])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        merged, res = device_path(d_packed[:nt], sub_meta, lim, sub_gts, names[:lim])
        torch.cuda.synchronize()
        out["device_path_on_text_subset_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
    assert merged.to_lines(names[:lim], DOTA_CLASSES) == lines, "the two paths merged different lines"
    assert res["map"] == text_res["map"] and res["ap"] == text_res["ap"], (res["map"], text_res["map"])
    out["text_path"] = dict(timing, images=lim, map_07=text_res["map"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
