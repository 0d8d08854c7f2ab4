"""Whole-image inference: tile producer -> detector -> ResultMerge, device resident between the steps.

Composition of the three reference stages that bracket the hot path (SURVEY 8 rows n4, a1-a12, n1):
  DOTA_devkit/SplitOnlyImage_multi_process.py (tiles, gap 200)        -> dota/split_tiles.py
  tools/test.py + OrientedRepPointsDetector.simple_test per tile      -> detector.py
  tools/parse_pkl/parse_pkl_mege_results_for_dota_evaluation.py:93-192 (Task1 lines per class) +
  DOTA_devkit/ResultMerge_multi_process.py:182-262 (coordinates back to the image, per-image poly NMS thr 0.1)
                                                                      -> dota/result_merge.py
The reference goes through PNG tiles, a pickle and per-class text files between these stages; here the tiles never
leave HBM and the per-class result lines are merged in memory (the same `merge_lines` the file-based mirror uses).
"""
from .result_merge import merge_lines
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
            results.extend(det.aug_test([v[k:k + 1] for v in views], [[m[k]] for m in metas], rescale=True,
                                        valid_hws=[v[k:k + 1] for v in valids]) for k in range(views[0].shape[0]))
    per_class = task1_lines(results, names)
    return {cname: merge_lines(lines, merge_thresh) for cname, lines in zip(DOTA_CLASSES, per_class)}
