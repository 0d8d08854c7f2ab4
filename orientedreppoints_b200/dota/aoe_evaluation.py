"""DOTA mAOE, the mean absolute orientation error (mirror of DOTA_devkit/mAOE_evaluation.py), with the matching and the
angles on the GPU.

`aoe_eval` keeps the reference's name and signature.  Everything goes through `evaluate_aoe`, which scores every class
in one device call (orp_dota_eval_aoe: the sorts and the rotated-IoU matching of the Task1 evaluation, then
poly2rbox_single_v3 angles and the per-class sums on the device, one copy back):

    gts = {name: parse_gt('labelTxt/%s.txt' % name) for name in imagenames}
    res = evaluate_aoe(dets, gts)                  # dets: {class: Task1 lines}, as for evaluation.evaluate
    res['aoe']['plane'], res['maoe']

A detection counts when the best iou_poly over ALL boxes of its image and class (difficult ones included, no claims)
exceeds ovthresh; its error is abs(v3(det) - v3(gt)) * 57.32 degrees.  Differences from the reference (DESIGN.md
section 2, deviation 11): a class without a matched detection gets aoe = nan and n = 0, and the mAOE is then nan (the
reference raises ZeroDivisionError); detections with equal scores are ranked in input order; |angle1| against |angle2|
within ~45 ulp in poly2rbox_single_v3 is decided by the exact angles.

    python -m orientedreppoints_b200.dota.aoe_evaluation DETPATH ANNOPATH IMAGESETFILE
prints the per-class AOE and the mAOE at ovthresh 0.7 as the reference's main() does (DETPATH e.g. 'Task1_{:s}.txt').
"""
import argparse

import numpy as np
import torch

from .. import _lib
from .evaluation import _host_arrays, _merged_inputs, parse_gt
from .pipeline import DOTA_CLASSES

# output sections of the result buffer: cls_off, count, aoe, angle_dif, order (the 4-byte one last keeps the rest aligned)
_OUT_DTYPES = (np.int64, np.int64, np.float64, np.float64, np.int32)
_ABI_ORDER = (0, 4, 3, 1, 2)   # the sections in the argument order of orp_dota_eval_aoe


def _launch(inputs, ncls, nimg, ovthresh, dev):
    """enqueue orp_dota_eval_aoe on the current stream over device inputs (the _host_arrays order, without the difficult
    flags); every output lands in one byte buffer, returned with its section offsets"""
    dc, di, ds, dq, gc, gi, gq = inputs[:7]
    nd, ng = dc.shape[0], gc.shape[0]
    sizes = [np.dtype(t).itemsize * n for t, n in zip(_OUT_DTYPES, (ncls + 1, ncls, ncls, nd, nd))]
    offs = np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)
    buf = torch.empty(max(int(offs[-1]), 8), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        rc = _lib.lib().orp_dota_eval_aoe(
            _lib.ptr(dc), _lib.ptr(di), _lib.ptr(ds), _lib.ptr(dq), nd, _lib.ptr(gc), _lib.ptr(gi), _lib.ptr(gq), ng, ncls,
            nimg, float(ovthresh), *(_lib.ptr(buf[offs[k]:offs[k + 1]]) for k in _ABI_ORDER), _lib.current_stream_ptr())
    _lib.check(rc, "orp_dota_eval_aoe")
    return buf, offs


def _result(buf, offs, classnames, first):
    out = buf.cpu().numpy()                                                           # the one copy back
    cls_off, count, aoe, angle_dif, order = (out[offs[k]:offs[k + 1]].view(t) for k, t in enumerate(_OUT_DTYPES))
    res = {'angle_dif': {}, 'order': {}, 'n': {}, 'aoe': {}}
    total = 0
    for c, cname in enumerate(classnames):
        sl = slice(int(cls_off[c]), int(cls_off[c + 1]))
        res['angle_dif'][cname] = angle_dif[sl].copy()
        res['order'][cname] = order[sl].astype(np.int64) - (sl.start if first is None else first[c])
        res['n'][cname] = int(count[c])
        res['aoe'][cname] = float(aoe[c])
        total = total + res['aoe'][cname]          # main()'s running sum (Python's sum() compensates since 3.12)
    res['maoe'] = total / len(classnames) if classnames else float('nan')
    return res


def evaluate_aoe(dets, gts, classnames=DOTA_CLASSES, ovthresh=0.7, device=None):
    """mAOE of every class in one device call.
      dets  {class name: Task1 lines} (what detect_image returns, or the lines of Task1_<class>.txt); a class that is
            absent or empty has no detections
      gts   {image name: parse_gt(...) objects}: the image set; objects of other classes are ignored, difficult ones are
            ground truth like any other
    Returns {'angle_dif': {class: fp64 array, per ranked detection its error in degrees, nan when unmatched},
             'order': {class: index of each ranked detection in that class's lines}, 'n': {class: matched detections},
             'aoe': {class: float}, 'maoe': float}.  The matched entries of angle_dif in rank order are aoe_eval's
    angle_dif_list; aoe = their left-to-right sum / n and maoe = the sum of the class aoe in class order over their count
    (the reference's main())."""
    classnames = tuple(classnames)
    arrays, nimg, first = _host_arrays(dets, gts, classnames)
    dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    inputs = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in arrays[:7]]
    buf, offs = _launch(inputs, len(classnames), nimg, ovthresh, dev)
    return _result(buf, offs, classnames, first)


def evaluate_aoe_merged(merged, gts, image_names, classnames=DOTA_CLASSES, ovthresh=0.7):
    """`evaluate_aoe` over result_merge.MergedDetections (merge_packed, detect_image_tensors): the same dict, with nothing
    parsed and no detection uploaded, as evaluation.evaluate_merged does for Task1 (the same KeyError for a detection of
    an image outside `gts`).  'order' indexes each class's merged rows, i.e. the lines of
    `merged.to_lines(image_names, classnames)`."""
    classnames = tuple(classnames)
    inputs, nimg, dev = _merged_inputs(merged, gts, image_names, classnames, "evaluate_aoe_merged")
    buf, offs = _launch(inputs, len(classnames), nimg, ovthresh, dev)
    return _result(buf, offs, classnames, None)


def aoe_eval(detpath, annopath, imagesetfile, classname, ovthresh=0.5):
    """angle_dif_list of one class from files: the error in degrees of every matched detection in descending score
    order.  detpath.format(classname) holds its Task1 lines, annopath.format(name) the label file of every image listed
    in imagesetfile"""
    with open(imagesetfile, 'r') as f:
        imagenames = [x.strip() for x in f.readlines()]
    gts = {name: parse_gt(annopath.format(name)) for name in imagenames}
    with open(detpath.format(classname), 'r') as f:
        lines = f.readlines()
    a = evaluate_aoe({classname: lines}, gts, (classname,), ovthresh)['angle_dif'][classname]
    return [float(v) for v in a[~np.isnan(a)]]


def main(argv=None):
    ap = argparse.ArgumentParser(description="DOTA mAOE (IoU 0.7) of Task1_<class>.txt files")
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
    res = evaluate_aoe(dets, gts, DOTA_CLASSES, ovthresh=0.7)
    for cname in DOTA_CLASSES:
        print('classname:', cname)
        print('angle_dif_ave: ', res['aoe'][cname])
    print('mAOE: ', res['maoe'])


if __name__ == '__main__':
    main()
