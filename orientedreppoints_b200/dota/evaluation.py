"""DOTA Task1 evaluation (mirror of DOTA_devkit/dota_evaluation_task1.py) with the matching on the GPU.

`parse_gt`, `voc_ap` and `voc_eval` keep the reference's names and signatures.  Everything goes through `evaluate`,
which scores every class in one device call (orp_dota_eval_task1: sorts, rotated-IoU matching, precision / recall and
AP on the device, one copy back) instead of a Python loop per detection and class:

    gts = {name: parse_gt('labelTxt/%s.txt' % name) for name in imagenames}
    res = evaluate(detect_image(det, img, name), gts)        # or {class: Task1 lines read from Task1_<class>.txt}
    res['ap']['plane'], res['map']

Differences from the reference (DESIGN.md section 6):
  - detections with equal scores are taken in input order (a stable sort; np.argsort's order is not specified);
  - a class without detections gets empty rec / prec and ap = voc_ap([], []) = 0.0 (the reference raises on an empty
    Task1 file; a missing file still raises FileNotFoundError in voc_eval);
  - nothing is printed per class (the reference prints the tp / fp arrays and npos).

    python -m orientedreppoints_b200.dota.evaluation DETPATH ANNOPATH IMAGESETFILE
prints the per-class AP and the mAP as the reference's main() does (DETPATH e.g. 'Task1_{:s}.txt').
"""
import argparse

import numpy as np
import torch

from .. import _lib
from .pipeline import DOTA_CLASSES

# the recall thresholds of the 11-point metric, exactly as numpy produces them (0.30000000000000004, ...)
THRESHOLDS_07 = np.arange(0., 1.1, 0.1)


def parse_gt(filename):
    """objects of a DOTA label file: [{'name', 'difficult', 'bbox': [x1, y1, ..., x4, y4]}, ...].  Lines are split on
    single spaces; lines with fewer than 9 fields (the imagesource: / gsd: headers) are skipped; field 10, when present,
    is the difficult flag (0 when absent)."""
    objects = []
    with open(filename, 'r') as f:
        for line in f:
            fields = line.strip().split(' ')
            if len(fields) < 9:
                continue
            objects.append({'name': fields[8], 'difficult': int(fields[9]) if len(fields) > 9 else 0,
                            'bbox': [float(v) for v in fields[:8]]})
    return objects


def voc_ap(rec, prec, use_07_metric=False):
    """VOC AP of a precision / recall curve: the 11-point metric (VOC07) or the area under the precision envelope."""
    rec, prec = np.asarray(rec, np.float64), np.asarray(prec, np.float64)
    if use_07_metric:
        ap = 0.
        for t in THRESHOLDS_07:
            sel = prec[rec >= t]
            ap = ap + (np.max(sel) if sel.size else 0) / 11.
        return ap
    mrec = np.concatenate(([0.], rec, [1.]))
    envelope = np.maximum.accumulate(np.concatenate(([0.], prec, [0.]))[::-1])[::-1]
    with np.errstate(invalid='ignore'):
        steps = np.flatnonzero(mrec[1:] != mrec[:-1])
        return np.sum((mrec[steps + 1] - mrec[steps]) * envelope[steps + 1])


def _parse_detections(lines, index):
    """Task1 lines `imagename score x1 y1 ... x4 y4` -> (image ids, scores, quads); an image outside `index` is a
    KeyError as in the reference"""
    fields = [line.strip().split(' ') for line in lines]
    img = np.fromiter((index[f[0]] for f in fields), np.int32, len(fields))
    nums = np.array([f[1:] for f in fields], dtype=np.float64).reshape(len(fields), -1)
    if nums.shape[1] != 9:
        raise ValueError("a Task1 line holds an image name, a score and 8 coordinates")
    return img, nums[:, 0], nums[:, 1:]


def _host_arrays(dets, gts, classnames):
    """the inputs of orp_dota_eval_task1 as numpy arrays: (arrays, number of images, index of each class's first
    detection)"""
    cls_index = {c: i for i, c in enumerate(classnames)}
    img_index = {name: i for i, name in enumerate(gts)}
    g_cls, g_img, g_quad, g_diff = [], [], [], []
    for name, objects in gts.items():
        for obj in objects:
            c = cls_index.get(obj['name'])
            if c is None:
                continue
            g_cls.append(c)
            g_img.append(img_index[name])
            g_quad.append(obj['bbox'])
            g_diff.append(int(obj['difficult']) != 0)
    d_cls, d_img, d_score, d_quad, first = [], [], [], [], []
    nd = 0
    for c, cname in enumerate(classnames):
        lines = dets.get(cname, ())
        first.append(nd)
        if len(lines) == 0:
            continue
        img, score, quad = _parse_detections(lines, img_index)
        d_cls.append(np.full(len(img), c, np.int32))
        d_img.append(img)
        d_score.append(score)
        d_quad.append(quad)
        nd += len(img)

    def cat(parts, dtype, width=None):
        return np.concatenate(parts).astype(dtype) if parts else np.zeros((0,) if width is None else (0, width), dtype)

    arrays = [cat(d_cls, np.int32), cat(d_img, np.int32), cat(d_score, np.float64), cat(d_quad, np.float64, 8),
              np.asarray(g_cls, np.int32), np.asarray(g_img, np.int32),
              np.asarray(g_quad, np.float64).reshape(len(g_cls), 8), np.asarray(g_diff, np.uint8)]
    return arrays, len(img_index), first


# output sections of the result buffer: npos, cls_off, rec, prec, ap, order (the 4-byte one last keeps the rest aligned)
_OUT_DTYPES = (np.int64, np.int64, np.float64, np.float64, np.float64, np.int32)
_ABI_ORDER = (0, 1, 5, 2, 3, 4)   # the sections in the argument order of orp_dota_eval_task1


def _launch(inputs, ncls, nimg, ovthresh, use_07_metric, dev):
    """enqueue orp_dota_eval_task1 on the current stream over device inputs (the _host_arrays order); every output
    lands in one byte buffer, returned with its section offsets"""
    dc, di, ds, dq, gc, gi, gq, gd = inputs
    nd, ng = dc.shape[0], gc.shape[0]
    sizes = [np.dtype(t).itemsize * n for t, n in zip(_OUT_DTYPES, (ncls, ncls + 1, nd, nd, ncls, nd))]
    offs = np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)
    buf = torch.empty(max(int(offs[-1]), 8), dtype=torch.uint8, device=dev)
    thr = np.ascontiguousarray(THRESHOLDS_07, np.float64)
    with torch.cuda.device(dev):
        rc = _lib.lib().orp_dota_eval_task1(
            _lib.ptr(dc), _lib.ptr(di), _lib.ptr(ds), _lib.ptr(dq), nd, _lib.ptr(gc), _lib.ptr(gi), _lib.ptr(gq),
            _lib.ptr(gd), ng, ncls, nimg, float(ovthresh), int(bool(use_07_metric)), thr.ctypes.data_as(_lib._vp),
            *(_lib.ptr(buf[offs[k]:offs[k + 1]]) for k in _ABI_ORDER), _lib.current_stream_ptr())
    _lib.check(rc, "orp_dota_eval_task1")
    return buf, offs


def evaluate(dets, gts, classnames=DOTA_CLASSES, ovthresh=0.5, use_07_metric=True, device=None):
    """Task1 evaluation of every class in one device call.
      dets  {class name: Task1 lines} (what detect_image returns, or the lines of Task1_<class>.txt); a class that is
            absent or empty has no detections
      gts   {image name: parse_gt(...) objects}: the image set; objects of other classes are ignored
    Returns {'rec': {class: fp64 array}, 'prec': {...}, 'ap': {class: float}, 'npos': {class: int},
             'order': {class: index of each ranked detection in that class's lines}, 'map': float}, with rec / prec / ap as
    voc_eval(ovthresh, use_07_metric) computes them and map = the sum of the class APs in class order over their count
    (the reference's main())."""
    classnames = tuple(classnames)
    arrays, nimg, first = _host_arrays(dets, gts, classnames)
    dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    inputs = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in arrays]
    buf, offs = _launch(inputs, len(classnames), nimg, ovthresh, use_07_metric, dev)
    out = buf.cpu().numpy()                                                           # the one copy back
    npos, cls_off, rec, prec, ap, order = (out[offs[k]:offs[k + 1]].view(t) for k, t in enumerate(_OUT_DTYPES))
    res = {'rec': {}, 'prec': {}, 'ap': {}, 'npos': {}, 'order': {}}
    total = 0
    for c, cname in enumerate(classnames):
        sl = slice(int(cls_off[c]), int(cls_off[c + 1]))
        res['rec'][cname] = rec[sl].copy()
        res['prec'][cname] = prec[sl].copy()
        res['ap'][cname] = float(ap[c])
        res['npos'][cname] = int(npos[c])
        res['order'][cname] = order[sl].astype(np.int64) - first[c]
        total = total + res['ap'][cname]
    res['map'] = total / len(classnames) if classnames else float('nan')
    return res


def _merged_inputs(merged, gts, image_names, classnames, who):
    """the device inputs of the evaluation calls (the _host_arrays order) from result_merge.MergedDetections: the merge's
    tensors as they are, image ids mapped to positions in `gts` on the device -> (inputs, number of images, device).  An
    image that carries a detection and is not a key of `gts` is a KeyError."""
    if len(classnames) != merged.ncls or len(image_names) != merged.nimg:
        raise ValueError("%s: %d class names and %d image names expected" % (who, merged.ncls, merged.nimg))
    arrays, nimg, _ = _host_arrays({}, gts, classnames)
    img_index = {name: i for i, name in enumerate(gts)}
    dev = merged.cls.device
    missing = [i for i, name in enumerate(image_names) if name not in img_index]
    if missing and len(merged):
        hit = torch.isin(merged.img, torch.tensor(missing, dtype=torch.int32, device=dev)).nonzero()
        if hit.numel():
            raise KeyError(image_names[int(merged.img[hit[0, 0]])])
    lut = torch.tensor([img_index.get(name, -1) for name in image_names], dtype=torch.int32).to(dev)
    inputs = [merged.cls.contiguous(), lut[merged.img.long()].contiguous(), merged.score.contiguous(),
              merged.quad.contiguous()] + [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in arrays[4:]]
    return inputs, nimg, dev


def evaluate_merged(merged, gts, image_names, classnames=DOTA_CLASSES, ovthresh=0.5, use_07_metric=True):
    """`evaluate` over result_merge.MergedDetections (merge_packed, detect_image_tensors): the same dict, with nothing
    parsed and no detection uploaded - the merge's tensors go to orp_dota_eval_task1 as they are.
      image_names  name of every image id of the merge.  The ids are mapped to the positions in `gts` on the device; an
                   image that carries a detection must be a key of `gts` (KeyError, as for a detection line of an unknown
                   image), one without detections need not be
      classnames   the merge's classes, in its class order
    'order' indexes each class's merged rows, i.e. the lines of `merged.to_lines(image_names, classnames)`."""
    classnames = tuple(classnames)
    inputs, nimg, dev = _merged_inputs(merged, gts, image_names, classnames, "evaluate_merged")
    buf, offs = _launch(inputs, len(classnames), nimg, ovthresh, use_07_metric, dev)
    out = buf.cpu().numpy()                                                           # the one copy back
    npos, cls_off, rec, prec, ap, order = (out[offs[k]:offs[k + 1]].view(t) for k, t in enumerate(_OUT_DTYPES))
    res = {'rec': {}, 'prec': {}, 'ap': {}, 'npos': {}, 'order': {}}
    total = 0
    for c, cname in enumerate(classnames):
        sl = slice(int(cls_off[c]), int(cls_off[c + 1]))
        res['rec'][cname] = rec[sl].copy()
        res['prec'][cname] = prec[sl].copy()
        res['ap'][cname] = float(ap[c])
        res['npos'][cname] = int(npos[c])
        res['order'][cname] = order[sl].astype(np.int64) - sl.start     # the merge is sorted by class: a class's rows start at cls_off
        total = total + res['ap'][cname]
    res['map'] = total / len(classnames)
    return res


def voc_eval(detpath, annopath, imagesetfile, classname, ovthresh=0.5, use_07_metric=False):
    """rec, prec, ap of one class from files: detpath.format(classname) holds its Task1 lines, annopath.format(name)
    the label file of every image listed in imagesetfile"""
    with open(imagesetfile, 'r') as f:
        imagenames = [x.strip() for x in f.readlines()]
    gts = {name: parse_gt(annopath.format(name)) for name in imagenames}
    with open(detpath.format(classname), 'r') as f:
        lines = f.readlines()
    res = evaluate({classname: lines}, gts, (classname,), ovthresh, use_07_metric)
    return res['rec'][classname], res['prec'][classname], res['ap'][classname]


def main(argv=None):
    ap = argparse.ArgumentParser(description="DOTA Task1 mAP (11-point metric, IoU 0.5) of Task1_<class>.txt files")
    ap.add_argument("detpath", help="detection files, e.g. 'results/Task1_{:s}.txt'")
    ap.add_argument("annopath", help="label files, e.g. 'val/labelTxt/{:s}.txt'")
    ap.add_argument("imagesetfile", help="text file with one image name per line")
    args = ap.parse_args(argv)
    with open(args.imagesetfile, 'r') as f:
        imagenames = [x.strip() for x in f.readlines()]
    gts = {name: parse_gt(args.annopath.format(name)) for name in imagenames}
    dets = {}
    for cname in DOTA_CLASSES:
        with open(args.detpath.format(cname), 'r') as f:
            dets[cname] = f.readlines()
    res = evaluate(dets, gts, DOTA_CLASSES, ovthresh=0.5, use_07_metric=True)
    for cname in DOTA_CLASSES:
        print('classname:', cname)
        print('ap: ', res['ap'][cname])
    print('map:', res['map'])
    print('classaps: ', 100 * np.array([res['ap'][c] for c in DOTA_CLASSES]))


if __name__ == '__main__':
    main()
