"""Mirror of OrientedRepPointsHead.get_bboxes / get_bboxes_single
(mmdet/models/anchor_heads/orientedreppoints_head.py:673-779) on NHWC head outputs.

Per level: sigmoid, max-over-class top-k(nms_pre), (dy,dx)->(x,y), minaerarect with the
`*stride + centre` affine fused into the kernel, reppoints likewise; levels concatenated; multiclass_rnms.
"""
import torch

from ..ops import minaerarect
from .bbox_nms import multiclass_rnms


def grid_points(h, w, stride, device):
    """PointGenerator.grid_points (mmdet/core/anchor/point_generator.py:14-22): (x*s, y*s), x fastest."""
    xs = torch.arange(0, w, device=device, dtype=torch.float32) * stride
    ys = torch.arange(0, h, device=device, dtype=torch.float32) * stride
    return torch.stack([xs.repeat(h), ys.view(-1, 1).repeat(1, w).view(-1)], dim=1)


def get_bboxes_single(cls_scores, points_preds, strides, scale_factor, cfg, rescale=False, nms=True):
    """cls_scores[l]: [H,W,15] logits, points_preds[l]: [H,W,18] (dy,dx interleaved, stride units) of ONE image."""
    mlvl_bboxes, mlvl_scores, mlvl_reppoints = [], [], []
    nms_pre = cfg.get('nms_pre', -1)
    for cls_score, points_pred, stride in zip(cls_scores, points_preds, strides):
        h, w, c = cls_score.shape
        scores = cls_score.reshape(-1, c).sigmoid()
        points_pred = points_pred.reshape(-1, 18)
        points = grid_points(h, w, stride, cls_score.device)
        if nms_pre > 0 and scores.shape[0] > nms_pre:
            max_scores, _ = scores.max(dim=1)
            # torch.topk in the reference; ties (implementation-defined there) -> lower index first
            _, order = max_scores.sort(descending=True, stable=True)
            topk_inds = order[:nms_pre]
            points = points[topk_inds, :]
            points_pred = points_pred[topk_inds, :]
            scores = scores[topk_inds, :]
        pts = points_pred.reshape(-1, 9, 2)
        pts_xy = torch.cat([pts[:, :, 1:2], pts[:, :, 0:1]], dim=2).reshape(-1, 18).contiguous()
        bboxes = minaerarect(pts_xy, scale=float(stride), center=points)         # rect*stride + centre (:748-749)
        reppoints = pts_xy * stride + points.repeat(1, 9)                         # :754-760
        mlvl_bboxes.append(bboxes)
        mlvl_scores.append(scores)
        mlvl_reppoints.append(reppoints)
    mlvl_bboxes = torch.cat(mlvl_bboxes)
    mlvl_reppoints = torch.cat(mlvl_reppoints)
    if rescale:
        mlvl_bboxes = mlvl_bboxes / mlvl_bboxes.new_tensor(scale_factor)
        mlvl_reppoints = mlvl_reppoints / mlvl_reppoints.new_tensor(scale_factor)
    mlvl_scores = torch.cat(mlvl_scores)
    padding = mlvl_scores.new_zeros(mlvl_scores.shape[0], 1)
    mlvl_scores = torch.cat([padding, mlvl_scores], dim=1)
    if nms:
        return multiclass_rnms(mlvl_bboxes, mlvl_scores, cfg['score_thr'], cfg['nms'], cfg['max_per_img'],
                               multi_reppoints=mlvl_reppoints)
    return mlvl_bboxes, mlvl_scores


def scalar_scale_factor(sf):
    """img_meta['scale_factor'] as one number.  mmdet's Resize writes a float with keep_ratio=True (every config of this path)
    and a 4-vector (w, h, w, h) otherwise; the head divides its 8 box / 18 point coordinates by it (:766-768), which only
    broadcasts for a scalar - a vector is accepted here when all its entries agree"""
    import numpy as np
    a = np.asarray(sf, dtype=np.float64).reshape(-1)
    if a.size == 0 or not np.all(a == a[0]):
        raise ValueError("scale_factor %r: the rotated-box head needs one scale for x and y (keep_ratio=True)" % (sf,))
    return float(a[0])


def get_bboxes_fused(cls_scores, pts_preds_refine, strides, img_metas, cfg, rescale=False):
    """The same computation as get_bboxes() as ONE device-resident pipeline (orp_head_postprocess): returns
    padded (dets [B,max_per_img,27], labels [B,max_per_img], counts [B]) device tensors, no host sync."""
    import ctypes

    from .. import _lib
    n = len(cls_scores)
    b = cls_scores[0].shape[0]
    dev = cls_scores[0].device
    cls_c = [c.contiguous() for c in cls_scores]
    ref_c = [p.contiguous() for p in pts_preds_refine]
    pa = (ctypes.c_void_p * n)(*[c.data_ptr() for c in cls_c])
    pr = (ctypes.c_void_p * n)(*[p.data_ptr() for p in ref_c])
    hs = (ctypes.c_int * n)(*[c.shape[1] for c in cls_c])
    ws = (ctypes.c_int * n)(*[c.shape[2] for c in cls_c])
    ss = (ctypes.c_int * n)(*[int(s) for s in strides])
    cap = int(cfg['max_per_img'])
    dets = torch.empty((b, cap, 27), dtype=torch.float32, device=dev)
    labels = torch.empty((b, cap), dtype=torch.int64, device=dev)
    counts = torch.empty((b,), dtype=torch.int32, device=dev)
    sf = None
    if rescale:
        sf = torch.tensor([scalar_scale_factor(m['scale_factor']) for m in img_metas], dtype=torch.float32).to(dev, non_blocking=True)
    nms_cfg = cfg['nms']
    if nms_cfg.get('type', 'rnms') != 'rnms' or nms_cfg.get('mode', 'exact64') != 'exact64':
        raise ValueError("get_bboxes_fused serves nms type 'rnms' in the default arithmetic; use get_bboxes() for %r" % (nms_cfg,))
    with torch.cuda.device(dev):
        rc = _lib.lib().orp_head_postprocess(n, pa, pr, hs, ws, ss, b, cls_c[0].shape[3], int(cfg.get('nms_pre', -1)),
                                             float(cfg['score_thr']), float(nms_cfg['iou_thr']), cap, _lib.ptr(sf),
                                             _lib.ptr(dets), _lib.ptr(labels), _lib.ptr(counts), _lib.current_stream_ptr())
    _lib.check(rc, "orp_head_postprocess")
    return dets, labels, counts


def aug_meta_table(img_metas, rescale):
    """The host side of orp_head_postprocess_aug's two small inputs as ONE fp32 array [V*B*3 + B]: per (view, image)
    flip (0 / 1), img_shape width, scale_factor, then per image the factor the result is multiplied by - the first view's
    scale_factor when rescale is False (orientedreppoints_detector.py:139-141), 1 otherwise.  img_metas[v] is the list of
    the B images' dicts of view v.  Only horizontal flips and one scale for x and y exist on this path."""
    import numpy as np
    nv, b = len(img_metas), len(img_metas[0])
    if nv < 1 or b < 1 or any(len(m) != b for m in img_metas):
        raise ValueError("aug_meta_table: every view needs the metas of the same %d images" % b)
    t = np.empty((nv * b * 3 + b,), np.float32)
    view = t[:nv * b * 3].reshape(nv, b, 3)
    for v, metas in enumerate(img_metas):
        for i, m in enumerate(metas):
            flip = bool(m.get('flip', False))
            if flip and m.get('flip_direction', 'horizontal') != 'horizontal':
                raise ValueError("aug_test maps back horizontal flips only, got flip_direction=%r" % (m['flip_direction'],))
            view[v, i] = (float(flip), float(m['img_shape'][1]) if flip else 0.0, scalar_scale_factor(m['scale_factor']))
    t[nv * b * 3:] = 1.0 if rescale else view[0, :, 2]
    return t


def get_bboxes_aug_fused(cls_scores, pts_preds_refine, strides, img_metas, cfg, rescale=False):
    """aug_test's post-processing (get_bboxes(nms=False) per view, flip / scale map-back, ONE multiclass_rnms across the
    views) as one device-resident pipeline (orp_head_postprocess_aug).  cls_scores[v][l]: [B,H,W,C] of view v;
    img_metas[v]: the B dicts of view v.  Returns padded (dets [B,max_per_img,27] with box | score in columns 18..26 and
    zero reppoint columns, labels [B,max_per_img], counts [B]) device tensors, no host sync."""
    import ctypes

    from .. import _lib
    nv, nl = len(cls_scores), len(strides)
    if any(len(c) != nl for c in cls_scores) or any(len(p) != nl for p in pts_preds_refine) or len(pts_preds_refine) != nv:
        raise ValueError("get_bboxes_aug_fused: every view needs %d levels of scores and points" % nl)
    nms_cfg = cfg['nms']
    if nms_cfg.get('type', 'rnms') != 'rnms' or nms_cfg.get('mode', 'exact64') != 'exact64':
        raise ValueError("get_bboxes_aug_fused serves nms type 'rnms' in the default arithmetic, got %r" % (nms_cfg,))
    b = cls_scores[0][0].shape[0]
    dev = cls_scores[0][0].device
    cls_c = [c.contiguous() for view in cls_scores for c in view]
    ref_c = [p.contiguous() for view in pts_preds_refine for p in view]
    n = nv * nl
    pa = (ctypes.c_void_p * n)(*[c.data_ptr() for c in cls_c])
    pr = (ctypes.c_void_p * n)(*[p.data_ptr() for p in ref_c])
    hs = (ctypes.c_int * n)(*[c.shape[1] for c in cls_c])
    ws = (ctypes.c_int * n)(*[c.shape[2] for c in cls_c])
    ss = (ctypes.c_int * n)(*[int(s) for s in strides] * nv)
    cap = int(cfg['max_per_img'])
    dets = torch.empty((b, cap, 27), dtype=torch.float32, device=dev)
    labels = torch.empty((b, cap), dtype=torch.int64, device=dev)
    counts = torch.empty((b,), dtype=torch.int32, device=dev)
    table = torch.from_numpy(aug_meta_table(img_metas, rescale)).to(dev, non_blocking=True)
    meta, out_scale = table[:nv * b * 3], (None if rescale else table[nv * b * 3:])
    with torch.cuda.device(dev):
        rc = _lib.lib().orp_head_postprocess_aug(nv, nl, pa, pr, hs, ws, ss, b, cls_c[0].shape[3], int(cfg.get('nms_pre', -1)),
                                                 float(cfg['score_thr']), float(nms_cfg['iou_thr']), cap, _lib.ptr(meta),
                                                 _lib.ptr(out_scale), _lib.ptr(dets), _lib.ptr(labels), _lib.ptr(counts),
                                                 _lib.current_stream_ptr())
    _lib.check(rc, "orp_head_postprocess_aug")
    return dets, labels, counts


def get_bboxes(cls_scores, pts_preds_refine, strides, img_metas, cfg, rescale=False, nms=True):
    """cls_scores[l]: [N,H,W,15]; pts_preds_refine[l]: [N,H,W,18] -> list of (dets [k,27], labels [k])"""
    out = []
    for img_id in range(cls_scores[0].shape[0]):
        out.append(get_bboxes_single([c[img_id] for c in cls_scores], [p[img_id] for p in pts_preds_refine], strides,
                                     img_metas[img_id]['scale_factor'], cfg, rescale, nms))
    return out
