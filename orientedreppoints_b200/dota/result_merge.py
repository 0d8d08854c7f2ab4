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


# --------------------------------------------------------------------------------------------------------------------
# The same merge over the packed detection buffer (gather.pack / gather.all_gather_detections), without the text
# --------------------------------------------------------------------------------------------------------------------

class MergedDetections:
    """Survivors of `merge_packed`, device resident and trimmed to their count, in the order of the merged Task1 files
    (class ascending; original image by first appearance among the class's rows; score descending, ties in row order):
      cls, img  int32 [n]    class and original-image id
      score     fp64 [n]     the fp32 score widened
      quad      fp64 [n, 8]  x1 y1 ... x4 y4 in original-image coordinates (the doubles poly2origpoly gives)
      src_row   int32 [n]    row number before the merge (dataset tile order, then in-tile order; unlabelled rows left out)
      cls_off   int64 [ncls + 1] range of every class
    These are the detection arrays orp_dota_eval_task1 reads (`evaluation.evaluate_merged`)."""

    def __init__(self, cls, img, score, quad, src_row, cls_off, nimg):
        self.cls, self.img, self.score, self.quad, self.src_row, self.cls_off = cls, img, score, quad, src_row, cls_off
        self.nimg, self.ncls = int(nimg), int(cls_off.shape[0]) - 1

    def __len__(self):
        return int(self.cls.shape[0])

    def to_lines(self, image_names, class_names):
        """{class name: [`imgname score x1 y1 x2 y2 x3 y3 x4 y4`, ...]}: string for string what `merge_lines` returns for
        the same detections (python float formatting of the doubles); image_names[i] is the name of image id i"""
        if len(image_names) != self.nimg or len(class_names) != self.ncls:
            raise ValueError("to_lines: %d image names and %d class names expected" % (self.nimg, self.ncls))
        off = self.cls_off.tolist()
        img, score, quad = self.img.tolist(), self.score.tolist(), self.quad.tolist()
        return {cname: [image_names[img[k]] + ' ' + str(score[k]) + ' ' + ' '.join(map(str, quad[k]))
                        for k in range(off[c], off[c + 1])] for c, cname in enumerate(class_names)}

    def write_task1(self, outdir, image_names, class_names):
        """the merged submission files `Task1_<class>.txt` (what mergebypoly writes), one per class, empty ones included"""
        os.makedirs(outdir, exist_ok=True)
        for cname, lines in self.to_lines(image_names, class_names).items():
            with open(os.path.join(outdir, 'Task1_%s.txt' % cname), 'w') as f:
                for line in lines:
                    f.write(line + '\n')


def merge_packed(packed, tile_slot, tile_xy, tile_rate, tile_img, nimg, ncls=15, thresh=None, plain=False, max_rows=None):
    """ResultMerge of packed detections in one device call (orp_result_merge) -> MergedDetections.
      packed     device fp32 [S, cap + 1, 28] from gather.pack, or the all-gather's [world, T, cap + 1, 28] as
                 gather.all_gather_detections(buf, packed=True) returns it.  The LAST row of every slot must be its count row:
                 the (all_buf, all_counts) pair that all_gather_detections returns by default has it cut off and is not an
                 input of this call (a count row with anything but zeros after the count is refused)
      tile_slot  int32 [Tn]: slot of `packed` (flattened over world, T) holding dataset tile i, negative to skip it
                 (gather.dataset_slots for the all-gather's layout, arange for a dataset-order buffer)
      tile_xy    int32 [Tn, 2] (left, up); tile_rate fp64 [Tn]; tile_img int32 [Tn] original image in [0, nimg)
                 (tiles of several rates of one image share its id); tensors or array-likes, uploaded when on the host
      plain      py_cpu_nms_poly (every pair compared) instead of py_cpu_nms_poly_fast, which mergesingle uses
      max_rows   bound on the rows to merge.  None reads the sum of the selected counts (one scalar) to size the call;
                 the trimmed result costs one more read of the survivor count and status: two host reads in all.  A
                 caller that passes a bound (Tn * cap always is one) saves the first, but the NMS is then planned, and its
                 scratch allocated, for the bound, so a loose one costs more than the read.
    A slot whose count is the NMS-overflow mark of orp_head_postprocess (-1), a slot outside the buffer, a rate <= 0 or an
    image id outside [0, nimg) raise OrpError: such a tile is never merged as an empty one."""
    if packed.dim() == 4:
        packed = packed.reshape(-1, packed.shape[2], packed.shape[3])
    if not packed.is_cuda or packed.dtype != torch.float32 or packed.dim() != 3 or packed.shape[2] != 28 or packed.shape[1] < 2:
        raise ValueError("merge_packed: a CUDA float32 [S, cap + 1, 28] buffer expected")
    dev = packed.device
    packed = packed.contiguous()
    s, cap = int(packed.shape[0]), int(packed.shape[1]) - 1
    slot = torch.as_tensor(tile_slot, dtype=torch.int32).reshape(-1).to(dev).contiguous()
    tn = int(slot.shape[0])
    xy = torch.as_tensor(tile_xy, dtype=torch.int32).reshape(tn, 2).to(dev).contiguous()
    rate = torch.as_tensor(tile_rate, dtype=torch.float64).reshape(tn).to(dev).contiguous()
    img = torch.as_tensor(tile_img, dtype=torch.int32).reshape(tn).to(dev).contiguous()
    if max_rows is None:
        sel = slot[(slot >= 0) & (slot < s)].long()
        max_rows = int(packed[sel, cap, 0].nan_to_num(0.0).clamp(0, cap).sum(dtype=torch.float64).item()) if tn else 0
    max_rows = int(max_rows)
    head = torch.empty(2, dtype=torch.int32, device=dev)                      # survivor count, status
    cls_off = torch.empty(ncls + 1, dtype=torch.int64, device=dev)
    o_cls, o_img, o_row = (torch.empty(max_rows, dtype=torch.int32, device=dev) for _ in range(3))
    o_score = torch.empty(max_rows, dtype=torch.float64, device=dev)
    o_quad = torch.empty((max_rows, 8), dtype=torch.float64, device=dev)
    mode = _lib.ORP_UNION_NAN_SUPPRESSES_ALL if plain else _lib.ORP_UNION_NAN_SUPPRESSES
    with torch.cuda.device(dev):
        rc = _lib.lib().orp_result_merge(
            _lib.ptr(packed), s, cap, _lib.ptr(slot), _lib.ptr(xy), _lib.ptr(rate), _lib.ptr(img), tn, int(ncls), int(nimg),
            float(nms_thresh if thresh is None else thresh), mode, max_rows, _lib.ptr(head[0:1]), _lib.ptr(cls_off),
            _lib.ptr(o_cls), _lib.ptr(o_img), _lib.ptr(o_score), _lib.ptr(o_quad), _lib.ptr(o_row), _lib.ptr(head[1:2]),
            _lib.current_stream_ptr())
    _lib.check(rc, "orp_result_merge")
    n, status = head.tolist()
    if status:
        why = [text for bit, text in ((_lib.ORP_MERGE_BAD_COUNT, "a tile's count is not in [0, cap] (-1: its NMS overflowed)"),
                                      (_lib.ORP_MERGE_BAD_TILE, "a tile's slot, rate or image id is out of range"),
                                      (_lib.ORP_MERGE_ROWS_OVERFLOW, "more rows than max_rows")) if status & bit]
        raise _lib.OrpError("orp_result_merge refused its input: " + "; ".join(why))
    return MergedDetections(o_cls[:n], o_img[:n], o_score[:n], o_quad[:n], o_row[:n], cls_off, nimg)
