"""GPU: the rotated-geometry entry points (csrc/minarearect.cu + minrect.cuh, csrc/overlaps.cu, csrc/convex_iou.cu and the
decode step of csrc/head_post.cu) at their launch edges and on degenerate input.

Every case calls the C entry point through _lib into outputs carved out of guard regions (Guarded, test_conv_plans_gpu.py)
and launches twice, into outputs pre-filled with two different NaN patterns: the results must be bitwise equal (every
output element written) and the guards untouched (nothing written outside).  References, by operator:
- minarearect: the hull maps of the reference's own device code (tests/golden/minarearect_ref.npz, geometry_edges.npz), the
  boxes of the CPU oracle bit for bit (it evaluates cos / atan2 in double and rounds, as the kernel does);
- box_iou_rotated: the reference's box_iou_rotated_cpu.cpp (box_iou_rotated.npz, geometry_edges.npz), and fp64 where the
  reference's fp32 evaluation loses digits (far from the origin, thin, tiny);
- quad_iou_matrix / poly_overlaps: fp64 (EXACT64), the oracle's fp32 rnms arithmetic bit for bit (COMPAT32);
- iou_poly_f64_pairs, convex_iou: the oracle bit for bit, and the reference's own devrIoU (device_ops_ref.npz).
ENTRY_POINTS names the cases of each entry point; tests/test_geometry_ops_cpu.py checks that it covers every geometry entry
point of include/orp_b200.h."""
import ctypes

import numpy as np
import pytest
import torch

from orientedreppoints_b200 import _lib

from test_conv_plans_gpu import PATTERNS, Guarded

pytestmark = pytest.mark.gpu

ENTRY_POINTS = {
    "orp_minarearect": ("test_minarearect_reference_sets", "test_minarearect_launch_edges", "test_minarearect_nonfinite",
                        "test_errors_and_empty_launches"),
    "orp_box_iou_rotated": ("test_box_iou_rotated_edges", "test_box_iou_rotated_ragged", "test_large_row_counts",
                            "test_errors_and_empty_launches"),
    "orp_quad_iou_matrix": ("test_quad_iou_zero_area_union_modes", "test_quad_iou_concave_and_compat32",
                            "test_quad_iou_and_poly_overlaps_ragged", "test_large_row_counts", "test_errors_and_empty_launches"),
    "orp_poly_overlaps": ("test_poly_overlaps_reference_boxes", "test_quad_iou_and_poly_overlaps_ragged", "test_large_row_counts",
                          "test_errors_and_empty_launches"),
    "orp_poly_overlaps_host": ("test_quad_iou_and_poly_overlaps_ragged", "test_errors_and_empty_launches"),
    "orp_iou_poly_f64_pairs": ("test_iou_poly_f64_pairs", "test_errors_and_empty_launches"),
    "orp_convex_iou": ("test_convex_iou_reference_sets", "test_convex_iou_past_the_grid_cap", "test_errors_and_empty_launches"),
}

SIZES = (1, 31, 32, 33, 65)


# ------------------------------------------------------------------------------------------------------------- helpers
def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _stream():
    return _lib.current_stream_ptr()


def _twice(dev, specs, launch, what):
    """run launch(*outputs) into Guarded outputs of specs [(shape, dtype)] once per NaN fill; returns the outputs (numpy)"""
    outs = [Guarded(shape, dtype, dev) for shape, dtype in specs]
    bits = []
    for pat in PATTERNS:
        for o in outs:
            o.fill(pat)
        _lib.check(launch(*[o.t for o in outs]), what)
        torch.cuda.synchronize()
        for o in outs:
            assert o.guards_intact(pat), "%s: a store landed outside the output" % what
        bits.append([o.bits() for o in outs])
    for i, (a, b) in enumerate(zip(*bits)):
        assert torch.equal(a, b), "%s: output %d differs between launches (an element was not written)" % (what, i)
    return [o.t.cpu().numpy() for o in outs]


def _same(a, b):
    """equal values, NaN where the other is NaN (the sign of a NaN is not part of the contract)"""
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


def _minarearect(dev, pts, scale=1.0, center=None):
    """orp_minarearect on a device tensor [n, 18] (any storage offset) -> (boxes, hull_map)"""
    n = pts.shape[0]
    L = _lib.lib()
    return _twice(dev, [((n, 8), torch.float32), ((n, 9), torch.int32)],
                  lambda o, m: L.orp_minarearect(_lib.ptr(pts), n, _lib.ptr(o), _lib.ptr(m), float(scale), _lib.ptr(center),
                                                 _stream()), "orp_minarearect")


def _box_iou(dev, b1, b2):
    L = _lib.lib()
    x, y = _t(b1.astype(np.float32), dev), _t(b2.astype(np.float32), dev)
    return _twice(dev, [((len(b1), len(b2)), torch.float32)],
                  lambda o: L.orp_box_iou_rotated(_lib.ptr(x), len(b1), _lib.ptr(y), len(b2), _lib.ptr(o), _stream()),
                  "orp_box_iou_rotated")[0]


def _quad_iou(dev, qa, qb, mode=_lib.ORP_NMS_EXACT64, union=_lib.ORP_UNION_NAN_KEEPS):
    L = _lib.lib()
    x, y = _t(qa.astype(np.float32), dev), _t(qb.astype(np.float32), dev)
    return _twice(dev, [((len(qa), len(qb)), torch.float32)],
                  lambda o: L.orp_quad_iou_matrix(_lib.ptr(x), len(qa), _lib.ptr(y), len(qb), mode, union, _lib.ptr(o),
                                                  _stream()), "orp_quad_iou_matrix")[0]


def _poly_overlaps(dev, b, q):
    L = _lib.lib()
    x, y = _t(b.astype(np.float32), dev), _t(q.astype(np.float32), dev)
    return _twice(dev, [((len(b), len(q)), torch.float32)],
                  lambda o: L.orp_poly_overlaps(_lib.ptr(x), len(b), _lib.ptr(y), len(q), _lib.ptr(o), _stream()),
                  "orp_poly_overlaps")[0]


def _convex_iou(dev, pts, quads):
    L = _lib.lib()
    x, y = _t(pts.astype(np.float32), dev), _t(quads.astype(np.float32), dev)
    return _twice(dev, [((len(pts), len(quads)), torch.float32)],
                  lambda o: L.orp_convex_iou(_lib.ptr(x), len(pts), _lib.ptr(y), len(quads), _lib.ptr(o), _stream()),
                  "orp_convex_iou")[0]


def _rotbox_vertices_f64(b):
    """corners of (cx, cy, w, h, theta) boxes in double from the fp32 inputs, as a ring"""
    b = np.asarray(b, np.float32).astype(np.float64)
    c, s = np.cos(b[:, 4]), np.sin(b[:, 4])
    out = np.empty((len(b), 8))
    for k, (u, v) in enumerate(((-0.5, -0.5), (0.5, -0.5), (0.5, 0.5), (-0.5, 0.5))):
        dx, dy = u * b[:, 2], v * b[:, 3]
        out[:, 2 * k] = b[:, 0] + c * dx - s * dy
        out[:, 2 * k + 1] = b[:, 1] + s * dx + c * dy
    return out


def _box_iou_f64(b1, b2):
    """[N, M] IoU in fp64 of the fp32 boxes, with the reference's rule that a float area below 1e-14 gives 0.  Each pair is
    moved to its centre and scaled to unit extent first (IoU does not change; the fp64 clip's absolute tolerances would
    not hold for 1e-7 boxes).  Also returns, per pair, the largest centre-shifted vertex coordinate in float"""
    va, vb = _rotbox_vertices_f64(b1), _rotbox_vertices_f64(b2)
    n, m = len(b1), len(b2)
    p, q = np.repeat(va, m, 0), np.tile(vb, (n, 1))
    ctr = np.concatenate([p, q], 1).reshape(-1, 8, 2)
    ctr = 0.5 * (ctr.max(1) + ctr.min(1))
    p, q = (p.reshape(-1, 4, 2) - ctr[:, None]).reshape(-1, 8), (q.reshape(-1, 4, 2) - ctr[:, None]).reshape(-1, 8)
    ext = np.maximum(np.abs(p).max(1), np.abs(q).max(1))
    sx = 0.5 * (np.repeat(b1[:, 0], m).astype(np.float32) + np.tile(b2[:, 0], n).astype(np.float32))
    sy = 0.5 * (np.repeat(b1[:, 1], m).astype(np.float32) + np.tile(b2[:, 1], n).astype(np.float32))
    shifted = np.maximum(np.abs(np.concatenate([va[:, 0::2].repeat(m, 0), np.tile(vb[:, 0::2], (n, 1))], 1) - sx[:, None]).max(1),
                         np.abs(np.concatenate([va[:, 1::2].repeat(m, 0), np.tile(vb[:, 1::2], (n, 1))], 1) - sy[:, None]).max(1))
    scale = np.where(ext > 0, ext, 1.0)[:, None]
    iou = np.asarray(_po().iou_poly_f64(p / scale, q / scale)).reshape(n, m)
    a1 = (b1[:, 2].astype(np.float32) * b1[:, 3].astype(np.float32)).astype(np.float64)
    a2 = (b2[:, 2].astype(np.float32) * b2[:, 3].astype(np.float32)).astype(np.float64)
    iou[(a1 < 1e-14)[:, None] | (a2 < 1e-14)[None, :]] = 0.0
    return iou, shifted.reshape(n, m)


def _po():
    from oracle import pyoracle
    return pyoracle


def _zero_area_quads():
    """quadrilaterals of zero area (points, segments, collinear corners) next to ordinary ones that touch them"""
    return np.array([(1, 1, 1, 1, 1, 1, 1, 1), (0, 0, 1, 1, 2, 2, 3, 3), (0, 0, 4, 0, 4, 0, 0, 0), (2, 0, 2, 3, 2, 3, 2, 0),
                     (1, 1, 1, 1, 1, 1, 1, 1), (0, 0, 3, 3, 0, 0, 3, 3),
                     (0, 0, 4, 0, 4, 3, 0, 3), (0, 0, 0, 3, 4, 3, 4, 0), (1, -1, 3, 1, 1, 3, -1, 1), (10, 10, 12, 10, 12, 12, 10, 12)],
                    np.float32)


def _concave_quads():
    """concave (arrowheads) and self-intersecting (bow ties) quadrilaterals, and convex ones they overlap"""
    return np.array([(0, 0, 4, 0, 1, 1, 0, 4), (0, 0, 4, 2, 0, 4, 1, 2), (4, 4, 0, 4, 3, 3, 4, 0),
                     (0, 0, 4, 4, 4, 0, 0, 4), (0, 0, 4, 0, 0, 4, 4, 4), (1, 0, 3, 4, 3, 0, 1, 4),
                     (0, 0, 4, 0, 4, 4, 0, 4), (1, 1, 5, 1, 5, 5, 1, 5), (2, -1, 5, 2, 2, 5, -1, 2), (0.5, 0.5, 3, 0.5, 3, 3, 0.5, 3)],
                    np.float32)


# ------------------------------------------------------------------------------------------------------------- minarearect
@pytest.mark.parametrize("name", ["minarearect_ref.npz", "geometry_edges.npz"])
def test_minarearect_reference_sets(cuda, golden, po, name):
    """sets the reference's own device code answered (duplicated, collinear, grid, equal, two-point, far and tied sets):
    hull index maps identical to it, -1 past the hull; boxes bit-identical to the oracle on every set"""
    g = golden(name)
    pts = g["mar_pts"]
    box, hmap = _minarearect(cuda, _t(pts, cuda))
    hn = g["mar_hull_n"]
    for i in range(len(pts)):
        assert np.array_equal(hmap[i, :hn[i]], g["mar_map"][i, :hn[i]]), i
        assert (hmap[i, hn[i]:] == -1).all(), i
    box_o, map_o, hn_o = po.minarearect(pts)
    assert np.array_equal(hn_o, hn) and np.array_equal(hmap, map_o)
    bad = np.nonzero(~np.all(box.view(np.uint32) == box_o.view(np.uint32), axis=1))[0]
    assert len(bad) == 0, (len(bad), bad[:10], box[bad[:3]], box_o[bad[:3]])


@pytest.mark.parametrize("n", [1, 127, 128, 129, 257])
def test_minarearect_launch_edges(cuda, po, n):
    """ragged last block; an input that is not 16-byte aligned (pts[1:] starts 72 B into the buffer: the scalar staging
    path); the fused `* scale + centre` affine - all bit-identical to the oracle"""
    rng = np.random.RandomState(n)
    pts = rng.normal(0, 3, (n + 1, 18)).astype(np.float32)
    pts[::5] = np.round(pts[::5])                                            # exact ties and collinear runs
    pts[3::7] = np.tile(pts[3::7, :2], (1, 9))                               # all nine points equal
    dev_pts = _t(pts, cuda)
    box_o, map_o, _ = po.minarearect(pts)
    for lo in (0, 1):
        view = dev_pts[lo:lo + n]
        assert (view.data_ptr() % 16 == 0) == (lo == 0)
        box, hmap = _minarearect(cuda, view)
        assert np.array_equal(box.view(np.uint32), box_o[lo:lo + n].view(np.uint32)), lo
        assert np.array_equal(hmap, map_o[lo:lo + n]), lo
    ctr = rng.uniform(-50, 1100, (n, 2)).astype(np.float32)
    for scale in (8.0, 128.0):
        fused, _ = _minarearect(cuda, dev_pts[1:], scale, _t(ctr, cuda))
        exp = box_o[1:] * np.float32(scale) + np.tile(ctr, (1, 4))           # two separately rounded fp32 operations
        assert np.array_equal(fused.view(np.uint32), exp.view(np.uint32)), scale


def test_minarearect_nonfinite(cuda, po):
    """NaN and +-inf points: the kernel's loops are bounded like the oracle's (the reference would not end); boxes and hull
    maps equal to the oracle's, NaN where it has NaN"""
    rng = np.random.RandomState(5)
    pts = rng.normal(0, 3, (300, 18)).astype(np.float32)
    r = rng.rand(300, 18)
    pts[(r < 0.04)] = np.nan
    pts[(r >= 0.04) & (r < 0.07)] = np.inf
    pts[(r >= 0.07) & (r < 0.10)] = -np.inf
    pts[:9] = np.nan
    pts[9:12, ::2] = np.inf
    box, hmap = _minarearect(cuda, _t(pts, cuda))
    box_o, map_o, _ = po.minarearect(pts)
    assert _same(box, box_o)
    assert np.array_equal(hmap, map_o)
    assert (~np.isfinite(pts)).any(1).sum() > 200


# ------------------------------------------------------------------------------------------------------------- decode path
def test_decode_path_equals_mirror_bitwise(cuda):
    """orp_head_postprocess with nothing filtered (score_thr -1), nothing suppressed (iou_thr 1) and room for every
    candidate: each decoded row comes out in candidate order.  Boxes and reppoints bitwise equal to the op-by-op mirror
    (minaerarect(scale, centre), then / scale_factor as separate torch operations), scores bitwise equal to torch.sigmoid.
    Level 0 has more locations than nms_pre (the top-k sort), the others fewer; two images with different scale factors."""
    from orientedreppoints_b200.core.get_bboxes import get_bboxes
    g = torch.Generator().manual_seed(3)
    levels, strides, nms_pre, C, B = [(12, 10), (6, 5), (3, 3)], [8, 16, 32], 50, 15, 2
    cls = [(torch.randn(B, h, w, C, generator=g) * 2).to(cuda) for h, w in levels]
    ref = [(torch.randn(B, h, w, 18, generator=g) * 3).to(cuda) for h, w in levels]
    ref[1][0, 2, 3] += 1000.0                                                 # a set far out, in stride units
    S = sum(min(h * w, nms_pre) for h, w in levels)
    cap = S * C + 7
    sf = [0.75, 1.3]
    cfg = dict(nms_pre=nms_pre, score_thr=-1.0, nms=dict(type='rnms', iou_thr=1.0), max_per_img=cap)
    n = len(levels)
    pa = (ctypes.c_void_p * n)(*[c.data_ptr() for c in cls])
    pr = (ctypes.c_void_p * n)(*[p.data_ptr() for p in ref])
    hs, ws = (ctypes.c_int * n)(*[h for h, _ in levels]), (ctypes.c_int * n)(*[w for _, w in levels])
    ss = (ctypes.c_int * n)(*strides)
    sft = torch.tensor(sf, dtype=torch.float32, device=cuda)
    L = _lib.lib()
    dets, labels, counts = _twice(
        cuda, [((B, cap, 27), torch.float32), ((B, cap), torch.int64), ((B,), torch.int32)],
        lambda d, l, c: L.orp_head_postprocess(n, pa, pr, hs, ws, ss, B, C, nms_pre, -1.0, 1.0, cap, _lib.ptr(sft), _lib.ptr(d),
                                               _lib.ptr(l), _lib.ptr(c), _stream()), "orp_head_postprocess")
    assert counts.tolist() == [S * C] * B
    mirror = get_bboxes(cls, ref, strides, [dict(scale_factor=s) for s in sf], cfg, rescale=True)
    for b in range(B):
        md, ml = (t.cpu().numpy() for t in mirror[b])
        assert md.shape == (S * C, 27)
        assert np.array_equal(labels[b, :S * C], np.tile(np.arange(C), S)) and np.array_equal(ml, labels[b, :S * C])
        assert (labels[b, S * C:] == -1).all() and (dets[b, S * C:] == 0).all()
        d = dets[b, :S * C]
        assert np.array_equal(d[:, :26].view(np.uint32), md[:, :26].view(np.uint32)), \
            float(np.abs(d[:, :26] - md[:, :26]).max())
        assert np.array_equal(d[:, 26].view(np.uint32), md[:, 26].view(np.uint32))
        # scores: torch.sigmoid of the logits at the candidate's location, in candidate order
        sig = []
        for (h, w), c in zip(levels, cls):
            s = torch.sigmoid(c[b].reshape(-1, C))
            if h * w > nms_pre:
                s = s[s.max(1)[0].sort(descending=True, stable=True)[1][:nms_pre]]
            sig.append(s)
        sig = torch.cat(sig).reshape(-1).cpu().numpy()
        assert np.array_equal(d[:, 26].view(np.uint32), sig.view(np.uint32))


# ------------------------------------------------------------------------------------------------------------- box_iou_rotated
def test_box_iou_rotated_edges(cuda, golden):
    """geometry_edges.npz (the reference's box_iou_rotated_cpu.cpp on identical, nested, edge- and corner-sharing, disjoint,
    zero / negative / threshold-area, far, thin and tiny boxes, angles 0, +-pi/2, +-pi, 2 pi, 1e3): within 1e-4 of the
    reference where the problem is well conditioned.  Where it is not (far, thin, tiny), both are compared with fp64: the
    kernel is no further from it than the reference, plus 1e-6, plus what the fp32 vertices allow.  Both evaluate the
    corners in fp32 after the centre shift, each rounded by up to half an ulp of the largest shifted coordinate L, which
    moves the IoU of boxes whose short side is s by about ulp(L) / s; the kernel's clip (a different algorithm from the
    reference's) lands up to 2 ulp(L) / s from fp64 - 3.7e-5 for two 1000 x 1 boxes at 45 degrees, where L = 354 and the
    reference happens to be within 1.8e-5.  Far from the origin (L ~ 2 after the shift) this leaves the 1e-6 alone."""
    g = golden("geometry_edges.npz")
    b1, b2, kind, ref = g["bir_b1"], g["bir_b2"], g["bir_kind"], g["bir_iou"]
    got = _box_iou(cuda, b1, b2)
    # an area of exactly float(1e-14) is below the reference's double threshold 1e-14: IoU 0, not ~1
    a1, a2 = (b1[:, 2] * b1[:, 3]).astype(np.float64), (b2[:, 2] * b2[:, 3]).astype(np.float64)   # float products
    i = int(np.nonzero(a1 == np.float64(np.float32(1e-14)))[0][0])
    assert kind[i] == 2 and ref[i, i] == 0 and got[i, i] == 0, got[i, i]
    zero = (a1 < 1e-14)[:, None] | (a2 < 1e-14)[None, :]
    assert (got[zero] == 0).all() and (ref[zero] == 0).all()
    fine = (kind != 1)[:, None] & (kind != 1)[None, :]
    assert np.abs(got[fine] - ref[fine]).max() < 1e-4
    # the centre shift collapses the 1e-7 box onto one fp32 point when the other box is far: the reference returns garbage
    # (-6e6 ... inf) for such disjoint pairs, the kernel 0 (its corner hulls are disjoint)
    f64, shifted = _box_iou_f64(b1, b2)
    va, vb = _rotbox_vertices_f64(b1), _rotbox_vertices_f64(b2)
    lo1, hi1, lo2, hi2 = (np.stack([v[:, 0::2].min(1), v[:, 1::2].min(1)], 1) if k == 0 else
                          np.stack([v[:, 0::2].max(1), v[:, 1::2].max(1)], 1) for v in (va, vb) for k in (0, 1))
    apart = ((lo1[:, None] > hi2[None, :] + 1e-3) | (lo2[None, :] > hi1[:, None] + 1e-3)).any(-1)
    tiny = (b1[:, 2] < 1e-6)[:, None] | (b2[:, 2] < 1e-6)[None, :]
    assert (got[apart] == 0).all() and (~np.isfinite(ref[apart & tiny])).any()
    assert np.isfinite(got).all()
    short = np.minimum(np.abs(b1[:, 2:4]).min(1)[:, None], np.abs(b2[:, 2:4]).min(1)[None, :]).astype(np.float64)
    # where one box is smaller than an ulp of the other's shifted corners, the fp32 centre shift collapses it: both the
    # reference and the kernel return meaningless values when the hulls overlap (4e4 for a 1e-7 box inside a 1000 x 1
    # one), which only an fp64 evaluation avoids.  Those pairs are the tiny box's alone
    collapsed = (np.spacing(shifted.astype(np.float32)).astype(np.float64) > short) & ~zero
    assert not (collapsed & ~tiny).any() and (collapsed & ~apart).sum() >= 4
    hard = ~fine & ~zero & ~collapsed
    e_got, e_ref = np.abs(got[hard] - f64[hard]), np.abs(ref[hard] - f64[hard])
    allow = 1e-6 + 2 * np.spacing(shifted[hard].astype(np.float32)).astype(np.float64) / short[hard]
    assert np.isfinite(f64).all()
    assert (e_got <= e_ref + allow).all(), (e_got.max(), e_ref.max(), np.nonzero(e_got > e_ref + allow))
    far = hard & (np.abs(b1[:, :2]).max(1) > 1e4)[:, None] & (np.abs(b2[:, :2]).max(1) > 1e4)[None, :]
    assert far.sum() >= 18 and (np.abs(got[far] - f64[far]) <= np.abs(ref[far] - f64[far]) + 1e-6).all()
    print("box_iou_rotated edges: worst |kernel - reference| %.2e (well conditioned), worst |kernel - fp64| %.2e, "
          "|reference - fp64| %.2e (far / thin / tiny)" % (np.abs(got[fine] - ref[fine]).max(), e_got.max(), e_ref.max()))
    assert (np.diag(ref)[kind == 0] > 0).sum() >= 8


def test_box_iou_rotated_ragged(cuda, golden):
    """N, M around the 32 x 32 tile against box_iou_rotated.npz (the reference's box_iou_rotated_cpu.cpp)"""
    g = golden("box_iou_rotated.npz")
    for n in SIZES:
        for m in SIZES:
            got = _box_iou(cuda, g["b1"][:n], g["b2"][:m])
            assert np.abs(got - g["iou"][:n, :m]).max() < 1e-4, (n, m)


# ------------------------------------------------------------------------------------------------------------- quad IoU, poly_overlaps
def test_poly_overlaps_reference_boxes(cuda, golden, po):
    """device_ops_ref.npz po_*: (cx, cy, w, h, theta) boxes of the reference's poly_overlaps test set, within 1e-5 of fp64
    on the corners (EXACT64 arithmetic, not the reference's fp32: DESIGN.md); geometry_edges.npz boxes likewise"""
    for name, bk, qk in (("device_ops_ref.npz", "po_boxes", "po_query"), ("geometry_edges.npz", "bir_b1", "bir_b2")):
        g = golden(name)
        b, q = g[bk], g[qk]
        got = _poly_overlaps(cuda, b, q)
        ref = po.iou_poly_f64_matrix(po.rotbox_to_quad_f32(b), po.rotbox_to_quad_f32(q))
        ref = np.where(np.isnan(ref), 1.0, ref)                               # union 0: the guard's (0 + 1) / (0 + 1)
        err = np.abs(got - ref).max()
        print("poly_overlaps %s: worst |kernel - fp64| %.2e" % (name, err))
        assert err < 1e-5, (name, err)


def test_quad_iou_zero_area_union_modes(cuda, po):
    """zero-area quadrilaterals (points, segments, collinear corners) in every union mode: the fp64 value of the oracle,
    exactly, wherever one side is degenerate; the guard mode's 1 where the union is 0"""
    q = _zero_area_quads()
    nq = len(q)
    f64 = po.iou_poly_f64_matrix(q, q)
    area = np.abs(_po_area(q))
    degen = (area == 0)[:, None] | (area == 0)[None, :]
    assert np.isnan(f64[degen]).any()
    for union in (_lib.ORP_UNION_NAN_KEEPS, _lib.ORP_UNION_GUARD, _lib.ORP_UNION_NAN_SUPPRESSES,
                  _lib.ORP_UNION_NAN_SUPPRESSES_ALL):
        got = _quad_iou(cuda, q, q, union=union)
        exp = f64.astype(np.float32)
        if union == _lib.ORP_UNION_GUARD:
            exp = np.where(np.isnan(exp), np.float32(1), exp)
        assert _same(got[degen], exp[degen]), union
        assert np.abs(got[~degen] - f64[~degen]).max() < 1e-5, union
    assert nq * nq == degen.size


def _po_area(q):
    q = q.reshape(-1, 4, 2).astype(np.float64)
    x, y = q[..., 0], q[..., 1]
    return 0.5 * (x * np.roll(y, -1, 1) - y * np.roll(x, -1, 1)).sum(1)


def test_quad_iou_concave_and_compat32(cuda, po):
    """concave and self-intersecting quadrilaterals take the fp64 fallback: (float) of the oracle's fp64 IoU, bitwise.
    COMPAT32 equals the oracle's fp32 rnms arithmetic bitwise on these and the zero-area sets"""
    q = _concave_quads()
    got = _quad_iou(cuda, q, q)
    exp = po.iou_poly_f64_matrix(q, q).astype(np.float32)
    nonconvex = np.zeros(len(q), bool)
    nonconvex[:6] = True
    sel = nonconvex[:, None] | nonconvex[None, :]
    assert _same(got[sel], exp[sel])
    assert np.abs(got[~sel] - exp[~sel]).max() < 1e-5
    for s in (q, _zero_area_quads(), _concave_quads()[::-1].copy()):
        got = _quad_iou(cuda, s, s, mode=_lib.ORP_NMS_COMPAT32)
        exp = po.iou_rnms_f32(np.repeat(s, len(s), 0), np.tile(s, (len(s), 1))).reshape(len(s), len(s))
        assert _same(got, exp)


def test_quad_iou_and_poly_overlaps_ragged(cuda, po):
    """N, K around the 32 x 32 tile: quad_iou_matrix (EXACT64 within 1e-5 of fp64, COMPAT32 bitwise the oracle),
    poly_overlaps on the device and through the host entry point (same values)"""
    from orientedreppoints_b200.dota import poly_nms_gpu as pg
    d = po.gen_clustered_boxes(20, 4, seed=7)[:, :8]
    rng = np.random.RandomState(1)
    b = np.stack([rng.uniform(0, 100, 65), rng.uniform(0, 100, 65), rng.uniform(5, 40, 65), rng.uniform(5, 40, 65),
                  rng.uniform(-3.2, 3.2, 65)], 1).astype(np.float32)
    for n in SIZES:
        for k in SIZES:
            qa, qb = d[:n], d[-k:]
            got = _quad_iou(cuda, qa, qb)
            ref = po.iou_poly_f64_matrix(qa, qb)
            assert np.abs(got - ref).max() < 1e-5, (n, k)
            got = _quad_iou(cuda, qa, qb, mode=_lib.ORP_NMS_COMPAT32)
            assert _same(got, po.iou_rnms_f32(np.repeat(qa, k, 0), np.tile(qb, (n, 1))).reshape(n, k)), (n, k)
            dev = _poly_overlaps(cuda, b[:n], b[-k:])
            host = pg.poly_overlaps(b[:n], b[-k:])
            assert np.array_equal(dev, host), (n, k)
            ref = po.iou_poly_f64_matrix(po.rotbox_to_quad_f32(b[:n]), po.rotbox_to_quad_f32(b[-k:]))
            assert np.abs(dev - ref).max() < 1e-5, (n, k)


# ------------------------------------------------------------------------------------------------------------- iou_poly_f64_pairs
def test_iou_poly_f64_pairs(cuda, po):
    """around the 128-thread block and on degenerate pairs (zero-area, concave, self-intersecting): the oracle bit for bit"""
    L = _lib.lib()
    d = po.gen_clustered_boxes(30, 8, seed=2)[:, :8].astype(np.float64)
    z, c = _zero_area_quads().astype(np.float64), _concave_quads().astype(np.float64)
    deg = np.concatenate([z, c])
    sets = [(d[:n], d[::-1][:n]) for n in (127, 128, 129)]
    sets.append((np.repeat(deg, len(deg), 0), np.tile(deg, (len(deg), 1))))
    for p, q in sets:
        n = len(p)
        x, y = _t(p, cuda), _t(q, cuda)
        got = _twice(cuda, [((n,), torch.float64)],
                     lambda o: L.orp_iou_poly_f64_pairs(_lib.ptr(x), _lib.ptr(y), n, _lib.ptr(o), _stream()),
                     "orp_iou_poly_f64_pairs")[0]
        exp = po.iou_poly_f64(p, q)
        assert _same(got, exp), n
        fin = ~np.isnan(exp)
        assert np.array_equal(got[fin].view(np.uint64), exp[fin].view(np.uint64)), n


# ------------------------------------------------------------------------------------------------------------- convex_iou
def test_convex_iou_reference_sets(cuda, golden, po):
    """device_ops_ref.npz cx_* (the reference's own devrIoU, 1500 x 40) and geometry_edges.npz (equal, two-point, collinear,
    grid, far and tied point sets against clockwise, counter-clockwise and zero-area quadrilaterals): equal to the reference
    bit for bit"""
    g = golden("device_ops_ref.npz")
    got = _convex_iou(cuda, g["cx_pts"], g["cx_quads"])
    assert np.array_equal(got.view(np.uint32), g["cx_iou"].view(np.uint32))
    e = golden("geometry_edges.npz")
    got = _convex_iou(cuda, e["mar_pts"], e["cx_quads"])
    assert _same(got, e["cx_iou"])
    fin = ~np.isnan(e["cx_iou"])
    assert np.array_equal(got[fin].view(np.uint32), e["cx_iou"][fin].view(np.uint32))
    assert _same(got, po.convex_iou(e["mar_pts"], e["cx_quads"]))


def test_convex_iou_past_the_grid_cap(cuda, po):
    """15 000 x 40 = 600 000 pairs, more than the grid-stride loop's 132 x 32 blocks of 128 threads (540 672): its second
    iteration runs.  Bit-identical to the oracle"""
    rng = np.random.RandomState(8)
    n, k = 15000, 40
    pts = (rng.rand(n, 9, 2) * 60 + rng.rand(n, 1, 2) * 100).astype(np.float32).reshape(n, 18)
    pts[:500, 6:] = np.tile(pts[:500, :2], (1, 6))
    quads = po.gen_rotated_boxes(k, seed=9, extent=160.0, wmin=10, wmax=80)[:, :8].astype(np.float32)
    assert n * k > 132 * 32 * 128
    got = _convex_iou(cuda, pts, quads)
    exp = po.convex_iou(pts, quads)
    assert np.array_equal(got.view(np.uint32), exp.view(np.uint32))
    assert (exp > 0.05).mean() > 0.05


# ------------------------------------------------------------------------------------------------------------- large row counts
def test_large_row_counts(cuda, po):
    """2 097 153 rows (65 536 row tiles of 32, plus one) against 3 queries: more row tiles than grid.y holds.  The rows
    tile a 1000-row set, so the result is the small result tiled"""
    n, k, base = 65536 * 32 + 1, 3, 1000
    idx = np.arange(n) % base
    rng = np.random.RandomState(4)
    b = np.stack([rng.uniform(0, 100, base), rng.uniform(0, 100, base), rng.uniform(5, 40, base), rng.uniform(5, 40, base),
                  rng.uniform(-3.2, 3.2, base)], 1).astype(np.float32)
    q = b[[3, 500, 999]].copy()
    q[:, 0] += 2.0
    quads = po.rotbox_to_quad_f32(b)
    qq = po.rotbox_to_quad_f32(q)
    for what, fn, rows, cols in (("quad_iou_matrix", _quad_iou, quads, qq), ("poly_overlaps", _poly_overlaps, b, q),
                                 ("box_iou_rotated", _box_iou, b, q)):
        small = fn(cuda, rows, cols)
        big = fn(cuda, rows[idx], cols)
        assert big.shape == (n, k)
        assert np.array_equal(big.view(np.uint32), small[idx].view(np.uint32)), what
        assert (small > 0.05).sum() > 10, what


# ------------------------------------------------------------------------------------------------------------- errors
def test_errors_and_empty_launches(cuda):
    """n < 0 and a NULL pointer with n > 0 are ORP_EINVAL; empty problems return ORP_OK and launch nothing"""
    L = _lib.lib()
    s = _stream()
    buf = torch.zeros(64, device=cuda)
    p, z = _lib.ptr(buf), _lib.ptr(None)
    hb = np.zeros(64, np.float32)
    h = hb.ctypes.data_as(ctypes.c_void_p)
    calls = {
        "orp_minarearect": lambda n, a: L.orp_minarearect(a, n, p, z, 1.0, z, s),
        "orp_box_iou_rotated": lambda n, a: L.orp_box_iou_rotated(a, n, p, 2, p, s),
        "orp_quad_iou_matrix": lambda n, a: L.orp_quad_iou_matrix(a, n, p, 2, 0, 0, p, s),
        "orp_poly_overlaps": lambda n, a: L.orp_poly_overlaps(a, n, p, 2, p, s),
        "orp_iou_poly_f64_pairs": lambda n, a: L.orp_iou_poly_f64_pairs(a, p, n, p, s),
        "orp_convex_iou": lambda n, a: L.orp_convex_iou(a, n, p, 2, p, s),
    }
    for name, call in calls.items():
        assert call(-1, p) == -1, name
        assert call(2, z) == -1, name
        before = _lib.launch_count()
        assert call(0, p) == 0 and call(0, z) == 0, name
        assert _lib.launch_count() == before, name
    assert L.orp_poly_overlaps_host(h, h, h, -1, 2, 0) == -1
    assert L.orp_poly_overlaps_host(h, None, h, 2, 2, 0) == -1
    before = _lib.launch_count()
    assert L.orp_poly_overlaps_host(h, h, h, 0, 2, 0) == 0 and L.orp_poly_overlaps_host(h, h, h, 2, 0, 0) == 0
    assert _lib.launch_count() == before
    # the second extent too
    assert L.orp_box_iou_rotated(p, 2, p, -1, p, s) == -1 and L.orp_convex_iou(p, 2, p, -1, p, s) == -1
    assert L.orp_quad_iou_matrix(p, 2, p, -1, 0, 0, p, s) == -1 and L.orp_poly_overlaps(p, 2, p, -1, p, s) == -1
    before = _lib.launch_count()
    assert L.orp_box_iou_rotated(p, 2, p, 0, p, s) == 0 and L.orp_quad_iou_matrix(p, 2, p, 0, 0, 0, p, s) == 0
    assert L.orp_convex_iou(p, 2, p, 0, p, s) == 0 and L.orp_poly_overlaps(p, 2, p, 0, p, s) == 0
    assert _lib.launch_count() == before
    torch.cuda.synchronize()
    assert bool((buf == 0).all())
