"""numpy restatement of orp_result_merge (the merge of packed detections), for the tests: the arithmetic of
poly2origpoly in IEEE double, the fp64 CPU-oracle NMS per (class, original image) on the restored doubles, and the order
of the merged Task1 files.  No GPU and no reference tree needed."""
import numpy as np


def packed_rows(packed, tile_slot, tile_xy, tile_rate, tile_img, nimg, ncls):
    """rows of the selected slots in dataset tile order, then in-tile order, rows without a class left out ->
    (quad fp64 [N,8] restored, score fp64 [N], cls int32 [N], img int32 [N])"""
    packed = np.asarray(packed, np.float32).reshape(-1, packed.shape[-2], 28)
    cap = packed.shape[1] - 1
    quad, score, cls, img = [], [], [], []
    for i, slot in enumerate(np.asarray(tile_slot).tolist()):
        if slot < 0:
            continue
        count = int(packed[slot, cap, 0])
        assert 0 <= count <= cap and 0 <= tile_img[i] < nimg and tile_rate[i] > 0
        rows = packed[slot, :count]
        label = rows[:, 27]
        ok = (label >= 0) & (label < ncls) & (label == np.floor(label))
        rows = rows[ok]
        off = np.tile(np.asarray(tile_xy[i], np.float64), 4)
        quad.append((rows[:, 18:26].astype(np.float64) + off) / np.float64(tile_rate[i]))
        score.append(rows[:, 26].astype(np.float64))
        cls.append(rows[:, 27].astype(np.int32))
        img.append(np.full(rows.shape[0], tile_img[i], np.int32))
    if not quad:
        return np.zeros((0, 8)), np.zeros(0), np.zeros(0, np.int32), np.zeros(0, np.int32)
    return np.concatenate(quad), np.concatenate(score), np.concatenate(cls), np.concatenate(img)


def merge_packed_ref(packed, tile_slot, tile_xy, tile_rate, tile_img, nimg, ncls=15, thresh=0.1, plain=False, nms=None):
    """-> dict(cls, img, score, quad, src_row, cls_off) as numpy arrays with the dtypes of MergedDetections.
    nms(dets fp64 [n,9], thresh, fast) returns kept indices in score order (default: oracle.pyoracle.nms_poly_f64)."""
    if nms is None:
        from oracle import pyoracle
        nms = pyoracle.nms_poly_f64
    quad, score, cls, img = packed_rows(packed, tile_slot, tile_xy, tile_rate, tile_img, nimg, ncls)
    rows, cls_off = [], [0]
    for c in range(ncls):
        of_class = np.flatnonzero(cls == c)
        _, first = np.unique(img[of_class], return_index=True)
        for m in img[of_class][np.sort(first)]:                     # original images in first-appearance order
            idx = of_class[img[of_class] == m]
            keep = nms(np.concatenate([quad[idx], score[idx, None]], 1), thresh, fast=not plain)
            rows.extend(idx[np.asarray(keep, np.int64)].tolist())
        cls_off.append(len(rows))
    rows = np.asarray(rows, np.int64)
    return dict(cls=cls[rows].astype(np.int32), img=img[rows].astype(np.int32), score=score[rows], quad=quad[rows].reshape(-1, 8),
                src_row=rows.astype(np.int32), cls_off=np.asarray(cls_off, np.int64))
