"""Mirror of DOTA_devkit/ResultMerge_multi_process.py (py_cpu_nms_poly[_fast] :23-121, nmsbynamedict
:156-172, poly2origpoly :173-180, mergesingle :182-223, mergebypoly :249-262) and ResultMerge.py:18-41,
with the O(N^2) python/SWIG loop replaced by ONE segmented rotated-NMS launch per result file
(segments = original image), and of the Task1 writer of
tools/parse_pkl/parse_pkl_mege_results_for_dota_evaluation.py:93-192.

Semantics kept: suppression predicate `iou <= thresh` keeps (a NaN IoU suppresses), selection in score
order, output order = first appearance of each original image, then kept detections in score order,
`imgname confidence x1 y1 ... x4 y4` with python float formatting.  Contract difference: the GPU kernel
consumes float32 coordinates (like the reference's own poly_gpu_nms) - of boxes translated, in float64, to their image's own
origin, so the cast costs ~1e-5 px instead of ~1e-3 px at full-image coordinates; text output keeps the doubles.
"""
import os
import re

import numpy as np
import torch

from .. import _lib
from ..ops.nms_wrapper import rnms_indices

nms_thresh = 0.1            # ResultMerge_multi_process.py:21  (ResultMerge.py:15 uses 0.3)

_PAT_XY = re.compile(r'__\d+___\d+')
_PAT_RATE = re.compile(r'__([\d+\.]+)__\d+___')


def _nms_segmented(dets, thresh, segments=None, device=None, union_mode=_lib.ORP_UNION_NAN_SUPPRESSES):
    dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    dets = np.asarray(dets)
    if dets.dtype == np.float64 and dets.shape[0]:
        # full-image coordinates (10^4 px) lose ~1e-3 px in a float32 cast.  IoU is translation invariant, so every segment
        # (original image) is moved to its own origin in float64 first: the float32 the kernel consumes then carries the
        # reference's doubles to ~1e-5 px instead
        seg_ids = np.zeros(dets.shape[0], np.int64) if segments is None else np.asarray(segments, np.int64)
        nseg = int(seg_ids.max()) + 1
        ox = np.full(nseg, np.inf)
        oy = np.full(nseg, np.inf)
        np.minimum.at(ox, seg_ids, dets[:, 0:8:2].min(axis=1))
        np.minimum.at(oy, seg_ids, dets[:, 1:8:2].min(axis=1))
        dets = dets.copy()
        dets[:, 0:8:2] -= np.floor(ox[seg_ids])[:, None]
        dets[:, 1:8:2] -= np.floor(oy[seg_ids])[:, None]
    d = torch.from_numpy(np.ascontiguousarray(dets, dtype=np.float32)).to(dev)
    seg = None if segments is None else torch.from_numpy(np.ascontiguousarray(segments, dtype=np.int32)).to(dev)
    keep = rnms_indices(d, float(thresh), segments=seg, mode="exact64", union_mode=union_mode, order=_lib.ORP_ORDER_SCORE_DESC)
    return keep.cpu().numpy()


def py_cpu_nms_poly(dets, thresh):
    """ResultMerge.py:18-41.  dets: ndarray [N,9] (x1..y4, score) -> list of kept indices in score-descending selection
    order.  Every pair is compared, so two zero-area boxes (union 0, NaN IoU) suppress each other wherever they are."""
    dets = np.asarray(dets)
    if dets.shape[0] == 0:
        return []
    return [int(i) for i in _nms_segmented(dets, thresh, union_mode=_lib.ORP_UNION_NAN_SUPPRESSES_ALL)]


def py_cpu_nms_poly_fast(dets, thresh):
    """ResultMerge_multi_process.py:60-121: as py_cpu_nms_poly, but a pair is only compared when the axis-aligned hulls
    overlap with positive area (the kernel's sweep prefilter), so zero-area boxes apart from each other are all kept."""
    dets = np.asarray(dets)
    if dets.shape[0] == 0:
        return []
    return [int(i) for i in _nms_segmented(dets, thresh)]


def poly2origpoly(poly, x, y, rate):
    origpoly = []
    for i in range(int(len(poly) / 2)):
        origpoly.append(float(poly[i * 2] + x) / float(rate))
        origpoly.append(float(poly[i * 2 + 1] + y) / float(rate))
    return origpoly


def parse_result_lines(lines):
    """-> (image names in first-appearance order, image id per detection, dets float64 [N,9])"""
    names, name_id, ids, rows = [], {}, [], []
    for line in lines:
        sp = line.strip().split(' ')
        if len(sp) < 10:
            continue
        subname = sp[0]
        oriname = subname.split('__')[0]
        x_y = re.findall(_PAT_XY, subname)
        x_y_2 = re.findall(r'\d+', x_y[0])
        x, y = int(x_y_2[0]), int(x_y_2[1])
        rate = re.findall(_PAT_RATE, subname)[0]
        poly = list(map(float, sp[2:10]))
        det = poly2origpoly(poly, x, y, rate)
        det.append(float(sp[1]))
        if oriname not in name_id:
            name_id[oriname] = len(names)
            names.append(oriname)
        ids.append(name_id[oriname])
        rows.append(det)
    return names, np.asarray(ids, dtype=np.int32), np.asarray(rows, dtype=np.float64).reshape(-1, 9)


def merge_lines(lines, thresh=None):
    """tile-level result lines of one class -> merged lines (strings without newline)"""
    thresh = nms_thresh if thresh is None else thresh
    names, ids, dets = parse_result_lines(lines)
    if dets.shape[0] == 0:
        return []
    keep = _nms_segmented(dets, thresh, segments=ids)          # score order across all images
    out = []
    keep_ids = ids[keep]
    for k, name in enumerate(names):                            # dict order of the reference = first appearance
        for i in keep[keep_ids == k]:
            det = dets[i]
            out.append(name + ' ' + str(float(det[8])) + ' ' + ' '.join(map(str, [float(v) for v in det[:8]])))
    return out


def mergesingle(dstpath, nms, fullname):
    """same signature as the reference (`nms` is accepted for compatibility and ignored)"""
    name = os.path.splitext(os.path.basename(fullname))[0]
    with open(fullname, 'r') as f:
        lines = f.readlines()
    merged = merge_lines(lines)
    with open(os.path.join(dstpath, name + '.txt'), 'w') as f:
        for line in merged:
            f.write(line + '\n')


def mergebypoly(srcpath, dstpath):
    os.makedirs(dstpath, exist_ok=True)
    for root, _, files in os.walk(srcpath):
        for fn in sorted(files):
            mergesingle(dstpath, py_cpu_nms_poly_fast, os.path.join(root, fn))


mergebase_parallel = lambda srcpath, dstpath, nms: mergebypoly(srcpath, dstpath)   # noqa: E731


def write_task1_raw(results, tile_names, class_names, outdir):
    """parse_pkl_mege_results_for_dota_evaluation.py:93-192: per class file `Task1_<class>.txt` with one line
    `tilename score x1 y1 x2 y2 x3 y3 x4 y4` per detection (bbox[-9:-1], bbox[-1])."""
    os.makedirs(outdir, exist_ok=True)
    files = [open(os.path.join(outdir, 'Task1_%s.txt' % c), 'w') for c in class_names]
    try:
        for per_class, tname in zip(results, tile_names):
            for c, arr in enumerate(per_class):
                for bbox in arr:
                    files[c].write(tname + ' ' + str(float(bbox[-1])) + ' ' +
                                   ' '.join(str(float(v)) for v in bbox[-9:-1]) + '\n')
    finally:
        for f in files:
            f.close()
