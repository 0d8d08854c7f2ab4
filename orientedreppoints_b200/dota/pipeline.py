"""Whole-image inference: tile producer -> detector -> ResultMerge, device resident between the steps.

Composition of the three reference stages that bracket the hot path (SURVEY 8 rows n4, a1-a12, n1):
  DOTA_devkit/SplitOnlyImage_multi_process.py (tiles, gap 200)        -> dota/split_tiles.py
  tools/test.py + OrientedRepPointsDetector.simple_test per tile      -> detector.py
  tools/parse_pkl/parse_pkl_mege_results_for_dota_evaluation.py:93-192 (Task1 lines per class) +
  DOTA_devkit/ResultMerge_multi_process.py:182-262 (coordinates back to the image, per-image poly NMS thr 0.1)
                                                                      -> dota/result_merge.py
The reference goes through PNG tiles, a pickle and per-class text files between these stages; here the tiles never
leave HBM and the per-class result lines are merged in memory (the same `merge_lines` the file-based mirror uses).
`detect_image_tensors` / `detect_images_tensors` are the same composition without the lines: the padded detections are
packed (gather.pack) and merged by one device call (result_merge.merge_packed).
"""
import numpy as np
import torch

from .result_merge import merge_lines, merge_packed
from .split_tiles import split_image

# mmdet/datasets/dota.py:8-12
DOTA_CLASSES = ('plane', 'baseball-diamond', 'bridge', 'ground-track-field', 'small-vehicle', 'large-vehicle', 'ship',
                'tennis-court', 'basketball-court', 'storage-tank', 'soccer-ball-field', 'roundabout', 'harbor',
                'swimming-pool', 'helicopter')


def task1_lines(results, tile_names):
    """rbbox2result lists of every tile -> per-class lists of `tilename score x1 y1 ... x4 y4` (the lines
    parse_pkl_mege_results_for_dota_evaluation.py:150-187 writes: bbox[-1] is the score, bbox[-9:-1] the quadrilateral)"""
    per_class = [[] for _ in DOTA_CLASSES]
    for res, tname in zip(results, tile_names):
        for c, arr in enumerate(res):
            for bbox in arr:
                per_class[c].append(tname + ' ' + str(float(bbox[-1])) + ' ' + ' '.join(str(float(v)) for v in bbox[-9:-1]))
    return per_class


def detect_image(det, img_u8, name="P0000", rate=1, subsize=1024, gap=200, batch=16, merge_thresh=None, test_pipeline=None):
    """det: OrientedRepPointsDetector; img_u8: decoded uint8 HWC image (numpy or tensor).  Returns
    {class name: [`imgname score x1 y1 x2 y2 x3 y3 x4 y4`, ...]} in the Task1 format after ResultMerge.
    test_pipeline: a config's test_pipeline (list of dicts).  When given, every batch of tiles goes through it on the
    device (resize / flip / pad, datasets/pipelines.py) and the detections are mapped back to tile coordinates
    (rescale=True) before ResultMerge, as tools/test.py does.  None (the default) feeds the tiles unchanged."""
    tiles, names, _ = split_image(img_u8, name, rate, subsize, gap, device=det.device)
    results = []
    for i in range(0, tiles.shape[0], batch):
        if test_pipeline is None:
            results.extend(det.simple_test(tiles[i:i + batch]))
            continue
        from ..datasets.pipelines import run_test_pipeline
        data = run_test_pipeline(test_pipeline, tiles[i:i + batch], device=det.device)
        views, metas, valids = data['img'], data['img_meta'], data['valid_hw']
        if len(views) == 1:
            results.extend(det.simple_test(views[0], metas[0], rescale=True, valid_hw=valids[0]))
        else:
            results.extend(_aug_results(det, views, metas, valids))
    per_class = task1_lines(results, names)
    return {cname: merge_lines(lines, merge_thresh) for cname, lines in zip(DOTA_CLASSES, per_class)}


def _aug_results(det, views, metas, valids):
    """one aug_test call for a batch of tiles -> the list of per-tile rbbox2result lists (a batch of one tile comes back
    as that tile's list itself)"""
    res = det.aug_test(views, metas, rescale=True, valid_hws=valids)
    return [res] if views[0].shape[0] == 1 else res


def _pack_rows(per_tile, cap, device):
    """[(dets [k,27], labels [k]) per tile] -> packed [T, cap + 1, 28] (the layout of gather.pack).  The buffer is filled
    where the rows live, so host rows (aug_test's list form) cost one upload per batch"""
    buf = torch.zeros((len(per_tile), cap + 1, 28), dtype=torch.float32, device=per_tile[0][0].device if per_tile else device)
    for t, (d, l) in enumerate(per_tile):
        k = d.shape[0]
        buf[t, :k, :27] = d.to(dtype=torch.float32)
        buf[t, :k, 27] = l.to(dtype=torch.float32)
        buf[t, cap, 0] = k
    return buf.to(device)


def _packed_tiles(det, img_u8, name, rate, subsize, gap, batch, test_pipeline):
    """the tiles of one image at one rate through the detector -> (packed [T, cap + 1, 28], tile origins)"""
    from .. import gather
    tiles, _, origins = split_image(img_u8, name, rate, subsize, gap, device=det.device)
    cap = int(det.test_cfg['max_per_img'])
    parts = []
    for i in range(0, tiles.shape[0], batch):
        if test_pipeline is None:
            out = det.simple_test(tiles[i:i + batch], return_tensors="padded")
        else:
            from ..datasets.pipelines import run_test_pipeline
            data = run_test_pipeline(test_pipeline, tiles[i:i + batch], device=det.device)
            views, metas, valids = data['img'], data['img_meta'], data['valid_hw']
            if len(views) == 1:
                out = det.simple_test(views[0], metas[0], rescale=True, valid_hw=valids[0], return_tensors="padded")
            else:
                out = []
                for res in _aug_results(det, views, metas, valids):
                    # aug_test rows are box(8) | score without the reppoints: right-aligned, as the Task1 writer reads
                    # a row from its end (bbox[-9:-1], bbox[-1])
                    rows = torch.zeros((sum(len(a) for a in res), 27), dtype=torch.float32)
                    width = res[0].shape[1]
                    rows[:, 27 - width:] = torch.from_numpy(np.concatenate([np.asarray(a, np.float32) for a in res]))
                    labels = torch.cat([torch.full((len(a),), c, dtype=torch.int64) for c, a in enumerate(res)])
                    out.append((rows, labels))
        if isinstance(out, tuple):                                   # padded (dets, labels, counts) of the fused head
            parts.append(gather.pack(*out)[0])
        else:                                                        # per-tile (dets, labels): classes kept in row order
            parts.append(_pack_rows(out, cap, det.device))
    return torch.cat(parts), origins


def detect_images_tensors(det, images, rate=1, subsize=1024, gap=200, batch=16, merge_thresh=None, test_pipeline=None,
                          image_ids=None, nimg=None):
    """`detect_image` for a list of (name, uint8 HWC image) with the detections kept on the device: every tile's padded
    detections (simple_test(..., return_tensors="padded")) are packed and ALL images are merged by one device call.
    Returns result_merge.MergedDetections; image i of the list has id i (or image_ids[i], in [0, nimg)), and
    `.to_lines(names, DOTA_CLASSES)` gives what detect_image returns for each image, concatenated per class.
    rate: one rate or a sequence of rates; the tiles of every rate of an image share its id, as the reference's
    multi-scale merge joins them through the tile name.
    No count is read per batch and nothing goes through rbbox2result; the merge reads the host twice (the row total that
    sizes it, then the survivor count with the status - see merge_packed's max_rows).  One exception: a test_pipeline with
    more than one view (multi-scale / flip) makes one batched `aug_test` call per batch of tiles and takes its list form
    (one count read per batch), which is repacked and uploaded once per batch."""
    rates = tuple(rate) if isinstance(rate, (tuple, list)) else (rate,)
    ids = list(range(len(images))) if image_ids is None else [int(i) for i in image_ids]
    nimg = (max(ids) + 1 if ids else 1) if nimg is None else int(nimg)
    parts, xy, tile_rate, tile_img = [], [], [], []
    for (name, img), iid in zip(images, ids):
        for r in rates:
            packed, origins = _packed_tiles(det, img, name, r, subsize, gap, batch, test_pipeline)
            parts.append(packed)
            xy.extend(origins)
            tile_rate.extend([float(str(r))] * len(origins))
            tile_img.extend([iid] * len(origins))
    if not parts:
        parts = [torch.zeros((0, int(det.test_cfg['max_per_img']) + 1, 28), dtype=torch.float32, device=det.device)]
    if len({p.shape[1] for p in parts}) != 1:
        raise ValueError("detect_images_tensors: tiles with different detection capacities")
    packed = torch.cat(parts)
    with torch.cuda.device(det.device):
        return merge_packed(packed, torch.arange(packed.shape[0], dtype=torch.int32), np.asarray(xy, np.int32).reshape(-1, 2),
                            np.asarray(tile_rate, np.float64), np.asarray(tile_img, np.int32), nimg, len(DOTA_CLASSES),
                            merge_thresh)


def detect_image_tensors(det, img_u8, image_id=0, rate=1, subsize=1024, gap=200, batch=16, merge_thresh=None,
                         test_pipeline=None, nimg=None):
    """`detect_image` with tensors out: the same composition (tiles -> detector -> ResultMerge), but the detections stay
    on the device between the steps.  Returns result_merge.MergedDetections whose rows carry `image_id`;
    `.to_lines(names, DOTA_CLASSES)` with names[image_id] = name equals `detect_image(det, img_u8, name, ...)` string for
    string.  See detect_images_tensors for the arguments."""
    return detect_images_tensors(det, [("img", img_u8)], rate, subsize, gap, batch, merge_thresh, test_pipeline,
                                 image_ids=[image_id], nimg=nimg)
