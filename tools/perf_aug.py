"""Time multi-view test-time augmentation (a test pipeline of 2 scales x flip = 4 views) over batches of 1024^2 tiles:
the batched aug_test with the fused post-processing (orp_head_postprocess_aug) against the per-tile eager route it
replaces in the whole-image pipeline, in one process, alternating.

    python tools/perf_aug.py [--batches 1 4 8] [--reps 5] [--window-tiles 16]

R-50, f16x3, seeded uint8 tiles, random weights with score_thr = 0 as bench.py sets it (with random weights nothing
passes 0.05): every view brings its full 80 160 / 77 835 candidates per tile to the cross-view NMS.  The test pipeline
runs once per batch size, outside the timed windows: both routes consume the same device views.  Per batch size, after
a warm-up of every shape, --reps rounds alternate
  (a) eager_per_tile   fused_post off, one aug_test call per tile (batch-1 dense passes, the op-by-op merge, rbbox2result)
  (b) fused_batched    one aug_test call per batch, return_tensors="padded" (no host read)
  (c) post-processing alone on the dense outputs of (b)'s views, held fixed: the op-by-op merge image by image against
      get_bboxes_aug_fused; the two must return identical detections (asserted, bit for bit)
each window CUDA events around enough steps to cover --window-tiles tiles (eight times as many for the two sides of (c),
whose steps are short), ending in a synchronise; medians are reported.
Also per step of one batch: the library's kernel launches (orp_launch_count; the eager route's torch kernels are not in
that count) and the calls torch reports as synchronising the host (torch.cuda.set_sync_debug_mode).
Prints one JSON line with the card's name and power limit (read-only nvidia-smi query).  Needs a CUDA device: there is
no fallback.
"""
import argparse
import json
import os
import sys
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

PIPELINE = [dict(type='LoadImageFromFile'),
            dict(type='MultiScaleFlipAug', img_scale=[(1024, 1024), (960, 960)], flip=True,
                 transforms=[dict(type='RotateResize', keep_ratio=True), dict(type='RotateRandomFlip'),
                             dict(type='Normalize', mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375], to_rgb=True),
                             dict(type='Pad', size_divisor=32), dict(type='ImageToTensor', keys=['img']),
                             dict(type='Collect', keys=['img'])])]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 4, 8])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--window-tiles", type=int, default=16, help="tiles every timed window covers")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("perf_aug.py measures the GPU pipeline and needs a CUDA device")
    from perf_eval import gpu_identity
    from orientedreppoints_b200 import _lib
    from orientedreppoints_b200.core.get_bboxes import get_bboxes_aug_fused
    from orientedreppoints_b200.datasets.pipelines import run_test_pipeline
    from orientedreppoints_b200.detector import STRIDES, OrientedRepPointsDetector
    from orientedreppoints_b200.weights import random_state_dict
    name, power = gpu_identity()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    det = OrientedRepPointsDetector(random_state_dict(50, seed=0, reference_init=True), 50, dev, "f16x3",
                                    test_cfg=dict(score_thr=0.0))

    def timed(fn, steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    def counted(fn):
        """(library launches, torch-reported host synchronisations) of one step"""
        torch.cuda.synchronize()
        _lib.reset_launch_count()
        torch.cuda.set_sync_debug_mode("warn")
        try:
            with warnings.catch_warnings(record=True) as w:
                warnings.simplefilter("always")
                fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        torch.cuda.synchronize()
        return _lib.launch_count(), sum("synchroniz" in str(x.message) for x in w)

    out = {"gpu": name, "power_limit": power, "model": "R-50 f16x3", "views": 4, "tile": 1024, "score_thr": 0.0,
           "reps": args.reps, "window_tiles": args.window_tiles, "batches": {}}
    for nb in args.batches:
        tiles = torch.from_numpy(np.random.RandomState(100 + nb).randint(0, 256, (nb, 1024, 1024, 3)).astype(np.uint8)).to(dev)
        data = run_test_pipeline(PIPELINE, tiles, device=dev)
        views, metas, valids = data['img'], data['img_meta'], data['valid_hw']
        assert len(views) == 4
        per_tile = [([v[k:k + 1] for v in views], [[m[k]] for m in metas], [v[k:k + 1] for v in valids]) for k in range(nb)]

        def eager_per_tile():
            det.fused_post = False
            return [det.aug_test(v, m, True, h) for v, m, h in per_tile]

        def fused_batched():
            det.fused_post = True
            return det.aug_test(views, metas, True, valids, return_tensors="padded")

        # (c): fixed dense outputs of the batched views
        dense = [det.forward_dense(v, h)[0] for v, h in zip(views, valids)]
        cls, ref = [[o[0] for o in outs] for outs in dense], [[o[2] for o in outs] for outs in dense]

        def post_eager():
            return [det._aug_merge_eager([[c[i:i + 1] for c in v] for v in cls], [[p[i:i + 1] for p in v] for v in ref],
                                         [[m[i]] for m in metas], True) for i in range(nb)]

        def post_fused():
            return get_bboxes_aug_fused(cls, ref, STRIDES, metas, det.test_cfg, True)

        dets, labels, counts = post_fused()
        cnt = counts.tolist()
        assert min(cnt) >= 0, "rotated NMS candidate list overflowed"
        for i, (d, l) in enumerate(post_eager()):
            assert cnt[i] == d.shape[0] and torch.equal(dets[i, :cnt[i], 18:], d) and torch.equal(labels[i, :cnt[i]], l), \
                "the fused and the op-by-op merge returned different detections for tile %d" % i

        steps = max(1, -(-args.window_tiles // nb))
        for fn in (eager_per_tile, fused_batched, post_eager, post_fused):    # warm-up: every shape, every route
            fn()
            fn()
        torch.cuda.synchronize()
        ms = {k: [] for k in ("eager_per_tile", "fused_batched", "post_eager", "post_fused")}
        for _ in range(args.reps):
            ms["eager_per_tile"].append(timed(eager_per_tile, steps))
            ms["fused_batched"].append(timed(fused_batched, steps))
            ms["post_eager"].append(timed(post_eager, 8 * steps))
            ms["post_fused"].append(timed(post_fused, 8 * steps))
        row = {"steps_per_window": steps, "post_steps_per_window": 8 * steps, "detections": cnt}
        for k, v in ms.items():
            row[k + "_ms_median"] = round(float(np.median(v)), 3)
            row[k + "_ms"] = [round(x, 3) for x in v]
        for k, fn in (("eager_per_tile", eager_per_tile), ("fused_batched", fused_batched), ("post_eager", post_eager),
                      ("post_fused", post_fused)):
            row[k + "_orp_launches"], row[k + "_torch_syncs"] = counted(fn)
        row["step_speedup"] = round(row["eager_per_tile_ms_median"] / row["fused_batched_ms_median"], 3)
        row["post_speedup"] = round(row["post_eager_ms_median"] / row["post_fused_ms_median"], 3)
        out["batches"][str(nb)] = row
        del dense, cls, ref, views, data, tiles
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
