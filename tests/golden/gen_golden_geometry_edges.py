"""Mint tests/golden/geometry_edges.npz: the rotated-geometry operators on small sets of edge cases, answered by the
reference's own code as oracle/build_ref.py compiles it:
    ref_box_iou_rotated.so     mmdet/ops/box_iou_rotated/src/box_iou_rotated_cpu.cpp (unmodified)
    ref_poly_overlaps_dev.so   DOTA_devkit/poly_nms_gpu/poly_overlaps_kernel.cu  (RotBox2Poly, devPolyIoU)
    ref_minarearect_dev.so     mmdet/ops/minarearect/src/minarearect_kernel.cu   (Findminbox, Jarvis_and_index)
    ref_convex_iou_dev.so      mmdet/ops/iou/src/convex_iou_kernel.cu            (devrIoU)

Every input is finite: the reference's gift wrapping never ends on NaN (the CPU oracle, whose loops are bounded, is the
reference for non-finite input).  Authoring machine only (needs the reference's source tree):

    python oracle/build_ref.py && python tests/golden/gen_golden_geometry_edges.py
"""
import ctypes
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import build_ref, pyoracle as po                                          # noqa: E402

F = np.float32
PI = float(np.pi)


def P(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def area_threshold_sides():
    """(w, h) with float(w) * float(h) == float(1e-14) exactly, and (w, h2) whose product is the next float above it"""
    w = h = F(1e-7)
    assert w * h == F(1e-14)
    target = np.nextafter(F(1e-14), F(1))
    h2 = h
    while w * h2 < target:
        h2 = np.nextafter(h2, F(1))
    assert w * h2 == target
    return w, h, h2


def rotated_boxes():
    """(cx, cy, w, h, theta) rows in two lists; `kind` marks each row: 0 ordinary, 1 far from the origin, thin or
    tiny (the reference's fp32 evaluation loses digits there), 2 zero or below-threshold area"""
    w7, h7, h7up = area_threshold_sides()
    a, b, kind = [], [], []

    def pair(r1, r2, k=0):
        a.append(r1)
        b.append(r2)
        kind.append(k)
    pair((10, 20, 8, 4, 0.3), (10, 20, 8, 4, 0.3))                                    # identical
    pair((0, 0, 10, 10, 0), (1, 1, 2, 3, 0.5))                                        # one inside the other
    pair((0, 0, 2, 2, 0), (2, 0, 2, 2, 0))                                            # shared edge
    pair((0, 0, 2, 2, 0), (2, 2, 2, 2, 0))                                            # shared corner
    pair((0, 0, 2, 2, PI / 4), (0, 2 * np.sqrt(2), 2, 2, PI / 4))                    # shared corner, rotated
    pair((0, 0, 2, 2, 0), (10, 10, 2, 2, 1))                                          # disjoint
    for t in (0.0, PI / 2, -PI / 2, PI, -PI, 2 * PI, 1e3):                            # angle conventions
        pair((5, 5, 6, 2, t), (5.5, 5, 6, 2, 0.2))
    pair((0, 0, 0, 2, 0), (0, 0, 2, 2, 0), 2)                                         # w = 0
    pair((0, 0, 2, 0, 0), (0, 0, 2, 2, 0), 2)                                         # h = 0
    pair((0, 0, -2, 2, 0), (0, 0, 2, 2, 0), 2)                                        # w < 0
    pair((0, 0, 2, -2, 0.4), (0, 0, 2, 2, 0), 2)                                      # h < 0
    pair((0, 0, -4, -2, 0.1), (0.5, 0, 4, 2, 0.1))                                    # both < 0: positive area
    pair((0, 0, w7, h7, 0), (0, 0, w7, h7, 0), 2)                                     # area exactly float(1e-14)
    pair((0, 0, w7, h7up, 0), (0, 0, w7, h7up, 0), 1)                                 # the next float above it
    for cx, cy in ((16000, 16000), (-16000, 16000), (16000.3, -16000.7)):             # small boxes far out
        pair((cx, cy, 3, 2, 0.4), (cx + 0.8, cy + 0.5, 3, 2, 0.9), 1)
        pair((cx, cy, 3, 2, 0.0), (cx + 1.5, cy, 3, 2, 0.0), 1)
    for d in (0.0, 0.2, 0.5):                                                         # aspect ratio 1e3 at 45 degrees
        pair((100, 100, 1000, 1, PI / 4), (100 + d, 100, 1000, 1, PI / 4 + 1e-3), 1)
    pair((100, 100, 1000, 1, PI / 4), (100, 100, 1, 1000, PI / 4), 1)                # crossing at right angles
    return np.array(a, F), np.array(b, F), np.array(kind, np.int32)


def point_sets():
    """[n, 18] nine-point sets where the hull and the min-area search go wrong"""
    rng = np.random.RandomState(11)
    s = []
    for v in (0.0, 3.5, -1000.0):                                                     # all nine points equal
        s.append(np.full(18, v, F))
    for p, q, k in (((0, 0), (1, 0), 4), ((2, 3), (2, 7), 5), ((-1, 5), (3, 1), 1), ((0.5, 0.25), (-7, 9), 8)):
        pts = [q if i % (k + 1) == k else p for i in range(9)]                        # two distinct points
        s.append(np.array(pts, F).reshape(18))
    for dx, dy in ((1, 0), (0, 1), (1, 1), (3, -2), (0.1, 0.7)):                      # nine collinear points
        t = rng.permutation(9).astype(F)
        s.append(np.stack([2 + t * F(dx), -1 + t * F(dy)], 1).astype(F).reshape(18))
    g = np.stack(np.meshgrid(np.arange(3), np.arange(3)), -1).reshape(9, 2).astype(F)
    for sc, perm in ((1, False), (4, False), (1, True), (3, True)):                   # integer grids
        pts = g * F(sc) + F(rng.randint(-5, 5))
        s.append((pts[rng.permutation(9)] if perm else pts).reshape(18))
    for off in ((1e3, 1e3), (-1e3, 1e3), (1e3, -1e3), (-1e3, -1e3)):                  # reppoints far out, in stride units
        s.append((rng.normal(0, 2, (9, 2)) + np.array(off)).astype(F).reshape(18))
        s.append((np.round(rng.normal(0, 2, (9, 2))) + np.array(off)).astype(F).reshape(18))
    # exact ties of the min-area argmin: shapes symmetric under a reflection that maps edge angle t to 90 - t
    for a, c in ((2, 1), (3, 1), (5, 2), (1, 1)):
        pts = np.array([(a, 0), (0, c), (-a, 0), (0, -c), (0, 0), (a / 2, 0), (0, c / 2), (-a / 2, 0), (0, -c / 2)], F)
        s.append(pts.reshape(18))
    oct_ = np.array([(2, 1), (1, 2), (-1, 2), (-2, 1), (-2, -1), (-1, -2), (1, -2), (2, -1), (0, 0)], F)
    s.append(oct_.reshape(18))
    s.append(oct_[::-1].copy().reshape(18))
    s.append((np.array([(0, 0), (4, 0), (4, 4), (0, 4), (1, 1), (2, 2), (3, 1), (1, 3), (2, 0)], F)).reshape(18))
    return np.stack(s).astype(F)


def quads():
    """[k, 8]: convex quadrilaterals in both orders, zero-area ones"""
    q = [(0, 0, 4, 0, 4, 3, 0, 3), (0, 0, 0, 3, 4, 3, 4, 0),                           # counter-clockwise, clockwise
         (-2, -1, 2, -1, 2, 1, -2, 1), (-2, 1, 2, 1, 2, -1, -2, -1),
         (1, -3, 4, 0, 1, 3, -2, 0), (1, -3, -2, 0, 1, 3, 4, 0),
         (1e3 - 3, 1e3 - 3, 1e3 + 3, 1e3 - 3, 1e3 + 3, 1e3 + 3, 1e3 - 3, 1e3 + 3),
         (0, 0, 1, 1, 2, 2, 3, 3),                                                     # zero area: collinear corners
         (1, 1, 1, 1, 1, 1, 1, 1),                                                     # zero area: one point
         (0, 0, 4, 0, 4, 0, 0, 0)]                                                     # zero area: a segment, doubled
    return np.array(q, F)


def main():
    build_ref.build(verbose=False)
    import torch  # noqa: F401  (ref_box_iou_rotated.so links libtorch)
    rb = ctypes.CDLL(os.path.join(po.REF_DIR, "ref_box_iou_rotated.so"))
    ro = ctypes.CDLL(os.path.join(po.REF_DIR, "ref_poly_overlaps_dev.so"))
    rm = ctypes.CDLL(os.path.join(po.REF_DIR, "ref_minarearect_dev.so"))
    rc = ctypes.CDLL(os.path.join(po.REF_DIR, "ref_convex_iou_dev.so"))

    b1, b2, kind = rotated_boxes()
    bir = np.zeros((len(b1), len(b2)), F)
    rb.ref_box_iou_rotated(P(b1), len(b1), P(b2), len(b2), P(bir))
    pov = np.zeros((len(b1), len(b2)), F)
    ro.ref_poly_overlaps(P(b1), len(b1), P(b2), len(b2), P(pov))
    poq = np.zeros((len(b1), 8), F)
    ro.ref_rotbox2poly(P(b1), len(b1), P(poq))

    pts = point_sets()
    boxes = np.zeros((len(pts), 8), F)
    rm.ref_minarearect(P(pts), len(pts), P(boxes))
    maps = np.full((len(pts), 9), -1, np.int32)
    hull_n = np.zeros(len(pts), np.int32)
    for i in range(len(pts)):
        hull_n[i] = rm.ref_hull_index_map(P(pts[i]), P(maps[i]))

    q = quads()
    cx = np.zeros((len(pts), len(q)), F)
    rc.ref_convex_iou(P(pts), len(pts), P(q), len(q), P(cx))

    np.savez_compressed(os.path.join(HERE, "geometry_edges.npz"),
                        bir_b1=b1, bir_b2=b2, bir_kind=kind, bir_iou=bir, po_quads=poq, po_iou=pov,
                        mar_pts=pts, mar_boxes=boxes, mar_map=maps, mar_hull_n=hull_n, cx_quads=q, cx_iou=cx)
    print("geometry_edges.npz: %d x %d rotated boxes, %d point sets, %d quadrilaterals" % (len(b1), len(b2), len(pts), len(q)))


if __name__ == "__main__":
    main()
