"""numpy restatement of the mAOE (DOTA_devkit/mAOE_evaluation.py aoe_eval) and of poly2rbox_single_v3
(dota_poly2rbox.py:128-190), for the tests: the reference's float32 / float64 arithmetic with numpy scalars, the
matching loop of aoe_eval over the oracle's iou_poly (oracle/dota_eval_oracle.py), and the one rule of orp_poly2rbox_v3
that is not numpy's: |angle1| against |angle2| within a band of ~45 ulp is decided by the exact angles.  No GPU and no
reference tree needed."""
import numpy as np

BAND = 1e-14        # the band of abs_angle_greater in csrc/evaluation.cu


def norm_angle(a):
    return (a - (-np.pi / 4)) % np.pi + (-np.pi / 4)


def _fold(x, y):
    """the direction (x, y) (float32) as a vector of angle |norm_angle(atan2(y, x))| in [0, 3pi/4)"""
    if not (x > -y or (x == -y and x > 0)):
        x, y = -x, -y
    return float(x), abs(float(y))


def abs_angle_greater(a1, a2, d1, d2):
    """abs(a1) > abs(a2), the exact angles of the float32 directions d1, d2 deciding within BAND"""
    d = abs(a1) - abs(a2)
    if not abs(d) <= BAND:
        return bool(d > 0)
    if d2[0] == 0 and d2[1] == 0:
        return _fold(*d1)[1] > 0
    (u1, v1), (u2, v2) = _fold(*d1), _fold(*d2)
    return u2 * v1 > v2 * u1            # products of float32 values: exact in float64


def poly2rbox_v3(poly):
    """(x_ctr, y_ctr, w, h, angle, branch): branch 1 / 2 is the edge whose angle was taken (0: a NaN edge)"""
    p = np.array(poly[:8], dtype=np.float32)
    pt1, pt2, pt3, pt4 = (p[0], p[1]), (p[2], p[3]), (p[4], p[5]), (p[6], p[7])
    with np.errstate(all="ignore"):
        edge1 = np.sqrt((pt1[0] - pt2[0]) * (pt1[0] - pt2[0]) + (pt1[1] - pt2[1]) * (pt1[1] - pt2[1]))
        edge2 = np.sqrt((pt2[0] - pt3[0]) * (pt2[0] - pt3[0]) + (pt2[1] - pt3[1]) * (pt2[1] - pt3[1]))
        max_edge, min_edge = max(edge1, edge2), min(edge1, edge2)
        ratio = max_edge / min_edge
        d1 = (pt2[0] - pt1[0], pt2[1] - pt1[1])
        d2 = (pt4[0] - pt1[0], pt4[1] - pt1[1])
        if ratio < np.float32(1.15):
            width, height = max_edge, min_edge
            a1 = norm_angle(np.arctan2(float(d1[1]), float(d1[0])))
            a2 = norm_angle(np.arctan2(float(d2[1]), float(d2[0])))
            angle, branch = (a2, 2) if abs_angle_greater(a1, a2, d1, d2) else (a1, 1)
        elif edge1 > edge2:
            width, height, branch = edge1, edge2, 1
            angle = norm_angle(np.arctan2(float(d1[1]), float(d1[0])))
        elif edge2 >= edge1:
            width, height, branch = edge2, edge1, 2
            angle = norm_angle(np.arctan2(float(d2[1]), float(d2[0])))
        else:
            width, height, branch, angle = 0, 0, 0, norm_angle(0)
        x_ctr = float(pt1[0] + pt3[0]) / 2
        y_ctr = float(pt1[1] + pt3[1]) / 2
    return float(x_ctr), float(y_ctr), float(width), float(height), float(angle), branch


def aoe_class(image_ids, scores, quads, gt, ovthresh=0.7, kind="quicksort"):
    """aoe_eval's loop for one class.  image_ids [nd], scores [nd], quads [nd, 8]; gt {image: quads [k, 8]} (every box of
    the class, difficult ones included).  Returns (order, angle_dif): the input index of each ranked detection and its
    error in degrees, nan when unmatched."""
    from oracle.dota_eval_oracle import _aabb, _iou_rows
    quads = np.asarray(quads, np.float64).reshape(-1, 8)
    order = np.argsort(-np.asarray(scores, np.float64), kind=kind)
    out = np.full(order.size, np.nan)
    for r, d in enumerate(order):
        gq = np.asarray(gt[image_ids[d]], np.float64).reshape(-1, 8)
        bb = quads[d]
        if not len(gq):
            continue
        gx0, gy0, gx1, gy1 = _aabb(gq)
        bx0, by0, bx1, by1 = (v[0] for v in _aabb(bb))
        with np.errstate(all="ignore"):
            iw = np.maximum(np.minimum(gx1, bx1) - np.maximum(gx0, bx0) + 1., 0.)
            ih = np.maximum(np.minimum(gy1, by1) - np.maximum(gy0, by0) + 1., 0.)
            inter = iw * ih
            uni = (bx1 - bx0 + 1.) * (by1 - by0 + 1.) + (gx1 - gx0 + 1.) * (gy1 - gy0 + 1.) - inter
            keep = gq[inter / uni > 0]
        if not len(keep):
            continue
        ious = _iou_rows(keep, bb)
        if np.max(ious) > ovthresh:
            g = keep[np.argmax(ious)]
            out[r] = abs(poly2rbox_v3(bb)[4] - poly2rbox_v3(g)[4]) * 57.32
    return order, out


def running_mean(values):
    """the reference main()'s plain running sum over the list, divided by its length (nan for an empty list)"""
    total = 0.0
    for v in values:
        total = total + v
    return total / len(values) if len(values) else float("nan")
