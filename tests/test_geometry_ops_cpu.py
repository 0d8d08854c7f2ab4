"""CPU: the oracle of the rotated-geometry operators against tests/golden/geometry_edges.npz (edge cases answered by the
reference's own code, tests/golden/gen_golden_geometry_edges.py), the case table of tests/test_geometry_ops_gpu.py against
the geometry entry points of include/orp_b200.h, and the row-shape checks of the Python wrappers."""
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gen():
    import importlib.util
    spec = importlib.util.spec_from_file_location("gen_golden_geometry_edges",
                                                  os.path.join(ROOT, "tests", "golden", "gen_golden_geometry_edges.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _quad_area(b):
    b = b.reshape(-1, 4, 2).astype(np.float64)
    x, y = b[:, :, 0], b[:, :, 1]
    return 0.5 * np.abs((x * np.roll(y, -1, 1) - y * np.roll(x, -1, 1)).sum(1))


def test_golden_inputs_are_the_generators(golden):
    """the stored inputs are what gen_golden_geometry_edges.py builds (its input half needs no reference)"""
    g, gen = golden("geometry_edges.npz"), _gen()
    b1, b2, kind = gen.rotated_boxes()
    assert np.array_equal(g["bir_b1"], b1) and np.array_equal(g["bir_b2"], b2) and np.array_equal(g["bir_kind"], kind)
    assert np.array_equal(g["mar_pts"], gen.point_sets()) and np.array_equal(g["cx_quads"], gen.quads())
    assert np.isfinite(g["bir_b1"]).all() and np.isfinite(g["mar_pts"]).all()


def test_minarearect_oracle_reproduces_edges(po, golden):
    """equal, two-point, collinear, grid, far (+-1e3) and tied sets: hull index maps identical to the reference's
    Jarvis_and_index; boxes identical, or within 2e-6 (the reference calls cosf, the oracle rounds a double cos: DESIGN
    deviation 3), or - at an exact tie of the min-area search - the other rectangle of the same area"""
    g = golden("geometry_edges.npz")
    boxes, maps, hull_n = po.minarearect(g["mar_pts"])
    assert np.array_equal(hull_n, g["mar_hull_n"])
    for i in range(len(hull_n)):
        assert np.array_equal(maps[i][:hull_n[i]], g["mar_map"][i][:hull_n[i]]), i
    d = np.abs(boxes - g["mar_boxes"]).max(1)
    scale = np.maximum(1.0, np.abs(g["mar_boxes"]).max(1))
    ties = np.nonzero(d > 2e-6 * scale)[0]
    a_ref, a_mine = _quad_area(g["mar_boxes"][ties]), _quad_area(boxes[ties])
    assert np.all(np.abs(a_ref - a_mine) <= 1e-6 * np.maximum(a_ref, 1e-12)), ties
    assert (hull_n <= 2).sum() >= 7                                   # the degenerate sets are in


def test_convex_iou_oracle_reproduces_edges(po, golden):
    """degenerate point sets against clockwise, counter-clockwise and zero-area quadrilaterals: every value, NaN (0 / 0)
    where the reference has NaN"""
    g = golden("geometry_edges.npz")
    out = po.convex_iou(g["mar_pts"], g["cx_quads"])
    ref = g["cx_iou"]
    assert np.array_equal(np.isnan(out), np.isnan(ref))
    ok = ~np.isnan(ref)
    assert np.array_equal(out[ok].view(np.uint32), ref[ok].view(np.uint32))
    assert np.isnan(ref).any() and (ref > 0.05).any()


def test_poly_overlaps_oracle_reproduces_edges(po, golden):
    """RotBox2Poly and devPolyIoU of poly_overlaps_kernel.cu on the rotated-box edge cases, bit for bit"""
    g = golden("geometry_edges.npz")
    assert np.array_equal(po.rotbox_to_quad_f32(g["bir_b1"]).view(np.uint32), g["po_quads"].view(np.uint32))
    ov = po.poly_overlaps_f32(g["bir_b1"], g["bir_b2"])
    assert np.array_equal(np.isnan(ov), np.isnan(g["po_iou"]))
    ok = ~np.isnan(ov)
    assert np.array_equal(ov[ok].view(np.uint32), g["po_iou"][ok].view(np.uint32))


def test_every_geometry_entry_point_has_gpu_cases():
    """each function the header declares under "Pairwise rotated IoU" and "minaerarect" names at least one existing case
    of tests/test_geometry_ops_gpu.py"""
    import test_geometry_ops_gpu as t
    hdr = open(os.path.join(ROOT, "include", "orp_b200.h")).read()
    start, end = hdr.index("Pairwise rotated IoU"), hdr.index("Head post-processing")
    names = set(re.findall(r"^int (orp_\w+)\(", hdr[start:end], re.M))
    assert names == {"orp_poly_overlaps_host", "orp_poly_overlaps", "orp_quad_iou_matrix", "orp_iou_poly_f64_pairs",
                     "orp_convex_iou", "orp_box_iou_rotated", "orp_minarearect"}
    assert set(t.ENTRY_POINTS) == names
    for name, cases in t.ENTRY_POINTS.items():
        assert cases, name
        for c in cases:
            assert callable(getattr(t, c, None)), (name, c)


@pytest.mark.parametrize("shape", [(3, 4), (3, 6), (5,), (2, 5, 1)])
def test_box_iou_rotated_rejects_wrong_rows(shape):
    """a [N, 4] tensor would make the kernel read 5 floats per row past its buffer"""
    from orientedreppoints_b200.ops import box_iou_rotated
    ok = torch.zeros(2, 5)
    with pytest.raises(ValueError, match=r"\[N, 5\]"):
        box_iou_rotated(torch.zeros(shape), ok)
    with pytest.raises(ValueError, match=r"\[N, 5\]"):
        box_iou_rotated(ok, torch.zeros(shape))


@pytest.mark.parametrize("shape", [(3, 5), (3, 9), (8,), (2, 4, 2)])
def test_quad_iou_matrix_rejects_wrong_rows(shape):
    from orientedreppoints_b200.ops import quad_iou_matrix
    ok = torch.zeros(2, 8)
    with pytest.raises(ValueError, match=r"\[N, 8\]"):
        quad_iou_matrix(torch.zeros(shape), ok)
    with pytest.raises(ValueError, match=r"\[N, 8\]"):
        quad_iou_matrix(ok, torch.zeros(shape))
