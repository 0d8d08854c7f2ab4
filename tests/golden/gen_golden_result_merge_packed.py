"""Golden vectors for the merge of packed detections (orp_result_merge): a seeded packed float32 buffer
[S, cap + 1, 28] with its tile metadata, and what the REFERENCE's own DOTA_devkit/ResultMerge_multi_process.py
(mergesingle :182-223 with py_cpu_nms_poly_fast :60-121 over the SWIG polyiou compiled by oracle/build_ref.py from the
reference's polyiou.cpp) makes of the Task1 lines printed from it, class by class.

    python oracle/build_ref.py && python tests/golden/gen_golden_result_merge_packed.py     # needs /root/reference

The set: 3 images and 4 classes of 15; tiles at rates 1 and 0.5 of every image, in a shuffled dataset order and in
shuffled slots; one empty tile; class 2 absent from one image; equal scores across different images; zero-area boxes.
"""
import json
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference/DOTA_devkit"

IMAGES = ("P0007", "P0003", "P0011")
CLASSES = ('plane', 'baseball-diamond', 'bridge', 'ground-track-field', 'small-vehicle', 'large-vehicle', 'ship',
           'tennis-court', 'basketball-court', 'storage-tank', 'soccer-ball-field', 'roundabout', 'harbor', 'swimming-pool',
           'helicopter')
USED = (0, 2, 4, 12)
CAP = 48


def quad_of(cx, cy, w, h, a):
    c, s = np.cos(a), np.sin(a)
    dx = np.array([-w, w, w, -w]) / 2
    dy = np.array([-h, -h, h, h]) / 2
    return np.stack([cx + dx * c - dy * s, cy + dx * s + dy * c], 1).reshape(8)


def make_packed(seed=0):
    rng = np.random.RandomState(seed)
    tiles = []                                                       # (image, left, up, rate)
    for m in range(len(IMAGES)):
        tiles += [(m, l, u, 1.0) for l in (0, 824) for u in (0, 824)] + [(m, 0, 0, 0.5)]
    tiles.append((1, 1024, 1024, 1.0))                               # stays empty
    order = rng.permutation(len(tiles) - 1).tolist() + [len(tiles) - 1]
    order.insert(5, order.pop())                                     # the empty tile in the middle of the dataset
    tiles = [tiles[k] for k in order]
    rows = [[] for _ in tiles]
    for m in range(len(IMAGES)):
        for c in USED:
            if c == 2 and m == 1:
                continue
            for _ in range(14):
                cx, cy = rng.uniform(60, 1788, 2)
                w, h, a = rng.uniform(20, 120), rng.uniform(10, 60), rng.uniform(-np.pi / 2, np.pi / 2)
                for t, (tm, l, u, rate) in enumerate(tiles):
                    if tm != m or t == 5:
                        continue
                    q = quad_of(cx, cy, w, h, a) + rng.normal(0, 1.5, 8)          # every tile sees the object a little differently
                    q = q * rate - np.tile([l, u], 4)
                    if q.min() < 0 or q.max() > 1024 or len(rows[t]) >= CAP - 4:
                        continue
                    rows[t].append((q, rng.uniform(0.05, 1.0), c))
    for t in (0, 3, 8):                                              # zero-area boxes: a point, a segment, a collinear quad
        p = rng.uniform(100, 900, 2)
        rows[t].append((np.tile(p, 4), 0.5, 0))
        rows[t].append((np.concatenate([p, p + 30, p + 30, p]), 0.4, 4))
        rows[t].append((np.concatenate([p, p + 10, p + 20, p + 30]), 0.3, 12))
    packed = np.zeros((len(tiles), CAP + 1, 28), np.float32)
    for t, rs in enumerate(rows):
        for k in rng.permutation(len(rs)).tolist():
            q, s, c = rs[k]
            r = int(packed[t, CAP, 0])
            packed[t, r, :18] = rng.uniform(0, 1024, 18)
            packed[t, r, 18:26] = q
            packed[t, r, 26] = s
            packed[t, r, 27] = c
            packed[t, CAP, 0] = r + 1
    # exactly equal scores across different images, in every used class
    for c in USED:
        hits = [(t, r) for t in range(len(tiles)) for r in range(int(packed[t, CAP, 0])) if packed[t, r, 27] == c]
        by_img = {}
        for t, r in hits:
            by_img.setdefault(tiles[t][0], []).append((t, r))
        imgs = sorted(by_img)
        for a, b in zip(imgs[:-1], imgs[1:]):
            for k in range(3):
                (ta, ra), (tb, rb) = by_img[a][k], by_img[b][k + 3]
                packed[tb, rb, 26] = packed[ta, ra, 26]
    slot = rng.permutation(len(tiles)).astype(np.int32)              # dataset tile i lives in slot[i]
    buf = np.zeros_like(packed)
    buf[slot] = packed
    return buf, slot, tiles


def tile_name(m, l, u, rate):
    return "%s__%s__%d___%d" % (IMAGES[m], "1" if rate == 1.0 else str(rate), l, u)


def lines_of(packed, slot, tiles):
    per_class = [[] for _ in CLASSES]
    for i, (m, l, u, rate) in enumerate(tiles):
        t = int(slot[i])
        for r in range(int(packed[t, CAP, 0])):
            row = packed[t, r]
            per_class[int(row[27])].append(tile_name(m, l, u, rate) + ' ' + str(float(row[26])) + ' ' +
                                           ' '.join(str(float(v)) for v in row[18:26]))
    return per_class


def main():
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    import polyiou                                            # SWIG module built from the reference's polyiou.cpp
    pkg = types.ModuleType("DOTA_devkit")
    pkg.__path__ = []
    utils = types.ModuleType("DOTA_devkit.dota_utils")      # the real one pulls shapely; mergesingle needs one helper
    utils.custombasename = lambda fullname: os.path.basename(os.path.splitext(fullname)[0])
    sys.modules["DOTA_devkit"] = pkg
    sys.modules["DOTA_devkit.dota_utils"] = utils
    sys.modules["DOTA_devkit.polyiou"] = polyiou
    pkg.dota_utils, pkg.polyiou = utils, polyiou
    sys.path.insert(0, REF)
    import ResultMerge_multi_process as R
    packed, slot, tiles = make_packed(0)
    per_class = lines_of(packed, slot, tiles)
    merged = {}
    with tempfile.TemporaryDirectory() as td:
        dst = os.path.join(td, "out")
        os.mkdir(dst)
        for c, lines in zip(CLASSES, per_class):
            if not lines:
                merged[c] = []
                continue
            src = os.path.join(td, "Task1_%s.txt" % c)
            open(src, "w").write("".join(l + "\n" for l in lines))
            R.mergesingle(dst, R.py_cpu_nms_poly_fast, src)
            merged[c] = open(os.path.join(dst, "Task1_%s.txt" % c)).read().splitlines()
    np.savez_compressed(os.path.join(HERE, "result_merge_packed.npz"), packed=packed, tile_slot=slot,
                        tile_xy=np.asarray([(l, u) for _, l, u, _ in tiles], np.int32),
                        tile_rate=np.asarray([r for _, _, _, r in tiles], np.float64),
                        tile_img=np.asarray([m for m, _, _, _ in tiles], np.int32))
    json.dump({"nms_thresh": R.nms_thresh, "images": IMAGES, "classes": CLASSES, "lines": per_class, "merged": merged},
              open(os.path.join(HERE, "result_merge_packed.json"), "w"))
    print("wrote result_merge_packed:", sum(map(len, per_class)), "tile-level lines ->", sum(map(len, merged.values())),
          "merged lines;", {c: len(v) for c, v in merged.items() if v})


if __name__ == "__main__":
    main()
