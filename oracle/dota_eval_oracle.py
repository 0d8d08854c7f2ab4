"""CPU restatement of voc_eval's per-detection matching loop (DOTA_devkit/dota_evaluation_task1.py:156-248) - TEST
INFRASTRUCTURE ONLY, the checker of orientedreppoints_b200.dota.evaluation at sizes no golden file holds.

The loop, per class: detections in descending score order (np.argsort with the given `kind`); for each, the ground
truth of its image whose "+1 pixel" axis-aligned overlap is positive; iou_poly(gt, det) against those; np.max /
np.argmax pick the target; a hit above the threshold on a free non-difficult box is a true positive, on a claimed one a
false positive, on a difficult one neither; a miss is a false positive.  IoU comes from the reference's own compiled
SWIG module when oracle/_ref has it (oracle/build_ref.py), else from the C port pinned to polyiou.cpp (pyoracle).
"""
import numpy as np

from . import pyoracle as po
from . import ref_driver

THRESHOLDS_07 = np.arange(0., 1.1, 0.1)


def _iou_rows(gt_rows, bb):
    """iou_poly(gt, bb) for every row of gt_rows, gt first as :211 passes it"""
    swig = ref_driver._swig()
    if swig is None:
        return po.iou_poly_f64(gt_rows, np.repeat(bb[None, :], gt_rows.shape[0], axis=0))
    q = swig.VectorDouble([float(v) for v in bb])
    return np.array([swig.iou_poly(swig.VectorDouble([float(v) for v in g]), q) for g in gt_rows], np.float64)


def _aabb(q):
    q = np.asarray(q, np.float64).reshape(-1, 8)
    return q[:, 0::2].min(axis=1), q[:, 1::2].min(axis=1), q[:, 0::2].max(axis=1), q[:, 1::2].max(axis=1)


def match(image_ids, scores, quads, gt, ovthresh=0.5, kind="quicksort"):
    """image_ids [nd] (hashable), scores [nd], quads [nd, 8]; gt {image: (quads [k, 8], difficult [k] bool)}.
    Returns (order, tp, fp): the input index of each sorted detection and its 0/1 flags in that order."""
    scores = np.asarray(scores, np.float64)
    quads = np.asarray(quads, np.float64).reshape(-1, 8)
    order = np.argsort(-scores, kind=kind)
    nd = order.size
    tp, fp = np.zeros(nd), np.zeros(nd)
    claimed = {img: np.zeros(len(g[1]), bool) for img, g in gt.items()}
    for r, d in enumerate(order):
        gq, diff = gt[image_ids[d]]
        bb = quads[d]
        best, target = -np.inf, None
        if len(gq):
            gx0, gy0, gx1, gy1 = _aabb(gq)
            bx0, by0, bx1, by1 = (v[0] for v in _aabb(bb))
            iw = np.maximum(np.minimum(gx1, bx1) - np.maximum(gx0, bx0) + 1., 0.)
            ih = np.maximum(np.minimum(gy1, by1) - np.maximum(gy0, by0) + 1., 0.)
            inter = iw * ih
            union = (bx1 - bx0 + 1.) * (by1 - by0 + 1.) + (gx1 - gx0 + 1.) * (gy1 - gy0 + 1.) - inter
            with np.errstate(divide="ignore", invalid="ignore"):
                kept = np.nonzero(inter / union > 0)[0]
            if kept.size:
                ious = _iou_rows(np.asarray(gq, np.float64)[kept], bb)
                best, target = np.max(ious), kept[np.argmax(ious)]
        if not best > ovthresh:
            fp[r] = 1.
        elif not diff[target]:
            if claimed[image_ids[d]][target]:
                fp[r] = 1.
            else:
                tp[r] = 1.
                claimed[image_ids[d]][target] = True
    return order, tp, fp


def rec_prec(tp, fp, npos):
    ctp, cfp = np.cumsum(tp), np.cumsum(fp)
    with np.errstate(divide="ignore", invalid="ignore"):
        rec = ctp / float(npos)
    return rec, ctp / np.maximum(ctp + cfp, np.finfo(np.float64).eps)


def voc_ap(rec, prec, use_07_metric=False):
    rec, prec = np.asarray(rec, np.float64), np.asarray(prec, np.float64)
    if use_07_metric:
        ap = 0.
        for t in THRESHOLDS_07:
            sel = prec[rec >= t]
            ap = ap + (np.max(sel) if sel.size else 0) / 11.
        return ap
    mrec = np.concatenate(([0.], rec, [1.]))
    env = np.maximum.accumulate(np.concatenate(([0.], prec, [0.]))[::-1])[::-1]
    with np.errstate(invalid="ignore"):
        i = np.flatnonzero(mrec[1:] != mrec[:-1])
        return np.sum((mrec[i + 1] - mrec[i]) * env[i + 1])


def eval_class(image_ids, scores, quads, gt, ovthresh=0.5, use_07_metric=False, kind="quicksort"):
    """(order, rec, prec, ap) of one class; npos counts the non-difficult boxes of every image in gt"""
    npos = sum(int(np.count_nonzero(~np.asarray(g[1], bool))) for g in gt.values())
    order, tp, fp = match(image_ids, scores, quads, gt, ovthresh, kind)
    rec, prec = rec_prec(tp, fp, npos)
    return order, rec, prec, voc_ap(rec, prec, use_07_metric)
