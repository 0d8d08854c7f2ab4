"""GPU: the rotated NMS (csrc/nms.cu) in every plan `run_nms` picks, against the CPU oracle.

`run_nms` chooses a plan from its arguments - EXACT64 sweep or COMPAT32 all pairs, y strips (R = 4) or none, a host retry
when the candidate list overflows or (no-sync callers) an overflow reported on the device, survivor flags or a keep list,
the union convention and the output order - and reports it through `orp_rnms_last_plan`.  Every case below asserts the
plan it reaches and compares the keep list with the oracle, indices AND order, bit-exact.  The inventory test runs the
NMS workloads of bench.py, reduces every call to a plan signature and fails when one has no case here.

Oracles: `po.nms_poly_f64(fast=True)` restates py_cpu_nms_poly_fast (ORP_UNION_NAN_KEEPS and ORP_UNION_NAN_SUPPRESSES
agree with it on finite, non-degenerate boxes), `po.nms_poly_f64(fast=False)` restates py_cpu_nms_poly (for finite input
and thr < 1 it equals the fp64 algorithm with poly_nms's (inter+1)/(union+1) guard, since a NaN IoU means union 0),
`po.nms_f32` the reference's fp32 rnms.  `_greedy` composes the greedy loop from `po.iou_poly_f64` where a convention has
no oracle of its own (NaN keeps: rnms)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

KEEPS, GUARD, SUPP, SUPP_ALL = 0, 1, 2, 3
ASC, DESC = 0, 1

# plan signature = (lazy, R, no_sync, flags_out, union_mode, order, retried) -> the parity case that covers it
PARITY = {
    (1, 1, 0, 0, KEEPS, DESC, 0): "test_scores_and_ties / test_resolve_chains (bench time_nms: rnms_indices, score order)",
    (1, 1, 0, 0, KEEPS, ASC, 0): "test_zero_area_public_entry_points (rnms)",
    (1, 1, 0, 0, GUARD, DESC, 0): "test_poly_gpu_nms_strips (n = 16383; the strip-less runs of every strip test) / "
                                  "test_zero_area_public_entry_points",
    (1, 4, 0, 0, GUARD, DESC, 0): "test_poly_gpu_nms_strips / test_strip_boundaries / test_zero_height_strips",
    (1, 4, 0, 0, KEEPS, DESC, 0): "test_poly_gpu_nms_strips (rnms_indices without segments: bench time_nms, n >= 16384)",
    (1, 1, 0, 0, SUPP, DESC, 0): "test_zero_area_public_entry_points (py_cpu_nms_poly_fast) / test_degenerate_pair_order_and_hulls",
    (1, 1, 0, 0, SUPP_ALL, DESC, 0): "test_zero_area_public_entry_points (py_cpu_nms_poly) / test_zero_area_task1_lines",
    (1, 1, 0, 0, KEEPS, DESC, 1): "test_candidate_list_retry[exact64]",
    (0, 1, 0, 0, KEEPS, DESC, 1): "test_candidate_list_retry[compat32]",
    (1, 1, 0, 0, KEEPS, ASC, 1): "test_no_sync_overflow (rnms_indices over the same rows)",
    (1, 1, 1, 1, KEEPS, ASC, 0): "test_fused_production_shapes (orp_head_postprocess, nms_pre 2000)",
    (1, 4, 1, 1, KEEPS, ASC, 0): "test_fused_segmented_strips (orp_head_postprocess, nms_pre -1)",
}

LEVELS_1024 = [(128, 128), (64, 64), (32, 32), (16, 16), (8, 8)]
STRIDES = (8, 16, 32, 64, 128)


def _sig(p):
    return (p["lazy"], p["R"], p["no_sync"], p["flags_out"], p["union_mode"], p["order"], int(p["attempts"] > 1))


def _plan():
    from orientedreppoints_b200 import _lib
    return _lib.rnms_last_plan()


def _rnms(cuda, d, thr, segments=None, mode="exact64", union=KEEPS, order=DESC):
    from orientedreppoints_b200 import _lib
    from orientedreppoints_b200.ops import rnms_indices
    seg = None if segments is None else torch.from_numpy(np.ascontiguousarray(segments, np.int32)).to(cuda)
    keep = rnms_indices(torch.from_numpy(np.ascontiguousarray(d, np.float32)).to(cuda), thr, segments=seg, mode=mode,
                        union_mode=union, order=order)
    torch.cuda.synchronize()
    return keep.cpu().numpy(), _plan(), _lib.last_nms_stats()


def _poly_gpu_nms(d, thr):
    from orientedreppoints_b200.dota.poly_nms_gpu import poly_gpu_nms
    keep = np.asarray(poly_gpu_nms(d, thr), np.int64)
    return keep, _plan()


def _strip_less(cuda, d, thr):
    """the same set through orp_rnms as one segment of unknown bound (seg_limit 0): no strips and 64-bit sweep keys, under
    poly_gpu_nms's guard and score-descending order"""
    keep, p, _ = _rnms(cuda, d, thr, segments=np.zeros(d.shape[0], np.int32), union=GUARD)
    _assert_plan(p, (1, 1, 0, 0, GUARD, DESC, 0), seg_limit=0, sweep_bits=64)
    return keep


def _score_order(d):
    """greedy order: higher score first, lower index first on ties (-0.0 and +0.0 are equal)"""
    return np.lexsort((np.arange(d.shape[0]), -d[:, 8].astype(np.float64)))


def _greedy(po, d, thr, conv):
    """greedy NMS over po.iou_poly_f64: conv 'keeps' suppresses on `iou > thr` (NaN keeps, rnms), 'all' on
    `!(iou <= thr)` (py_cpu_nms_poly).  Rows with a non-finite coordinate neither suppress nor are suppressed."""
    n = d.shape[0]
    q = d[:, :8].astype(np.float64)
    fin = np.isfinite(q).all(1)
    order = _score_order(d)
    alive = np.ones(n, bool)
    keep = []
    for a, i in enumerate(order):
        if not alive[i]:
            continue
        keep.append(i)
        if not fin[i]:
            continue
        rest = order[a + 1:]
        rest = rest[alive[rest] & fin[rest]]
        if rest.size == 0:
            continue
        with np.errstate(invalid="ignore"):
            v = po.iou_poly_f64(np.repeat(q[i:i + 1], rest.size, 0), q[rest])
            dead = (v > thr) if conv == "keeps" else ~(v <= thr)
        alive[rest[dead]] = False
    return np.asarray(keep, np.int64)


def _segmented_oracle(po, d, seg, thr, order=DESC):
    keep = []
    for s in np.unique(seg):
        ids = np.nonzero(seg == s)[0]
        keep.append(ids[po.nms_poly_f64(d[ids], thr, fast=True)])
    keep = np.sort(np.concatenate(keep))
    if order == DESC:
        keep = keep[np.argsort(-d[keep, 8].astype(np.float64), kind="stable")]
    return keep


def _assert_plan(p, sig, **fields):
    assert _sig(p) == sig, (p, sig)
    assert sig in PARITY
    for k, v in fields.items():
        assert p[k] == v, (k, p)


# ------------------------------------------------------------------------------------------------- box sets
def _zero_area_boxes(n, rng, extent):
    """quadrilaterals whose fp64 signed area is exactly 0: points, segments traversed p,q,q,p and p,p,q,q, collinear
    quads with four distinct points (dyadic coordinates, so the shoelace terms are exact)"""
    out = np.empty((n, 8), np.float32)
    for k in range(n):
        p = np.round(rng.uniform(64, extent, 2) * 4) / 4
        v = rng.randint(-16, 17, 2).astype(np.float64)
        kind = k % 4
        if kind == 0:
            pts = [p, p, p, p]
        elif kind == 1:
            pts = [p, p + v, p + v, p]
        elif kind == 2:
            pts = [p, p, p + v, p + v]
        else:
            pts = [p, p + v, p + 3 * v, p + 2 * v]
        out[k] = np.concatenate(pts).astype(np.float32)
    return out


def _task1_lines(n, rng):
    """Task1-style zero-area rows: four points on one horizontal line, coordinates rounded to 0.1 (`%.1f`), in the order
    x0 < x1 < x3 < x2.  The fan intersection of two such rings often leaves a rounding residue, so union = -inter != 0
    and the fp64 IoU is -1 (keeps) instead of NaN / guard 1 (suppresses): which zero-area pairs suppress is decided by
    the fp64 algorithm, not by their areas alone."""
    y = np.round(rng.uniform(1, 1000, n), 1)
    x = np.sort(np.round(rng.uniform(1, 900, (n, 4)), 1), 1)
    return np.stack([x[:, 0], y, x[:, 1], y, x[:, 3], y, x[:, 2], y], 1).astype(np.float32)


def _with_scores(quads, rng):
    sc = rng.permutation(quads.shape[0]).astype(np.float32) / np.float32(quads.shape[0]) + np.float32(0.001)
    return np.concatenate([quads, sc[:, None]], 1).astype(np.float32)


def _equal_height_boxes(n, h, seed):
    """axis-aligned boxes of height h (a power of two): the strip height is exactly 1.5 h and every ymin sits on a strip
    boundary, a third or two thirds of the way into a strip"""
    rng = np.random.RandomState(seed)
    s = 1.5 * h
    k = rng.randint(0, 100, n)
    ymin = (k * s + rng.choice([0.0, h / 2, h], n)).astype(np.float32)
    ymin[0] = 0.0
    xmin = np.round(rng.uniform(0, 60 * h, n)).astype(np.float32)
    w = np.float32(h) * rng.choice([0.5, 1.0, 2.0, 3.0], n).astype(np.float32)
    x1, y1 = xmin + w, ymin + np.float32(h)
    d = np.stack([xmin, ymin, x1, ymin, x1, y1, xmin, y1], 1).astype(np.float32)
    return _with_scores(d, rng)


# ------------------------------------------------------------------------------------------------- head outputs
def _head_outs(cuda, B, levels, seed, C=15, spread=1.5, logit_mu=-2.0):
    g = torch.Generator().manual_seed(seed)
    cls, ref = [], []
    for (h, w) in levels:
        cls.append((torch.randn(B, h, w, C, generator=g) * 1.5 + logit_mu).to(cuda))
        ref.append((torch.randn(B, h, w, 18, generator=g) * spread).to(cuda))
    return cls, ref


def _cfg(score_thr, nms_pre=2000, max_per_img=2000):
    return dict(nms_pre=nms_pre, min_bbox_size=0, score_thr=score_thr, nms=dict(type='rnms', iou_thr=0.4),
                max_per_img=max_per_img)


def _fused(cls, ref, cfg, metas):
    from orientedreppoints_b200.core.get_bboxes import get_bboxes_fused
    dets, labels, counts = get_bboxes_fused(cls, ref, STRIDES[:len(cls)], metas, cfg, rescale=True)
    torch.cuda.synchronize()
    return dets, labels, counts.tolist(), _plan()


def _check_fused_vs_mirror(cls, ref, cfg, metas, dets, labels, counts):
    """the op-by-op mirror (get_bboxes -> multiclass_rnms -> rnms_indices) performs the same fp32 operations: everything
    is compared bitwise, coordinates included"""
    from orientedreppoints_b200.core.get_bboxes import get_bboxes
    mirror = get_bboxes(cls, ref, STRIDES[:len(cls)], metas, cfg, rescale=True)
    for i, (md, ml) in enumerate(mirror):
        d, l = dets[i, :counts[i]], labels[i, :counts[i]]
        assert counts[i] == md.shape[0], (i, counts[i], md.shape)
        assert torch.equal(l, ml), i
        assert torch.equal(d, md), (i, float((d - md).abs().max()) if d.numel() else 0.0)
        assert bool((labels[i, counts[i]:] == -1).all())
    return mirror


def _check_fused_vs_oracle(cls, ref, cfg, metas, dets, labels, counts, images):
    """restated reference post-processing on the CPU oracle (po.minarearect + class-segmented fp64 NMS): labels, order and
    scores bit-exact.  Coordinates within 2e-2 px: the minaerarect oracle equals the kernel to <= 1e-4 stride units on
    near-tied rectangles (DESIGN section 2), times strides up to 128."""
    from oracle import torch_reference as tr
    for i in images:
        sf = metas[i]["scale_factor"]
        rd, rl = tr.get_bboxes_single([c[i].permute(2, 0, 1) for c in cls], [r[i].permute(2, 0, 1).cpu() for r in ref],
                                      strides=STRIDES[:len(cls)], nms_pre=cfg["nms_pre"], score_thr=cfg["score_thr"],
                                      iou_thr=cfg["nms"]["iou_thr"], max_per_img=cfg["max_per_img"], scale_factor=sf)
        d, l = dets[i, :counts[i]].cpu(), labels[i, :counts[i]].cpu()
        assert torch.equal(l, rl), i
        assert torch.equal(d[:, -1], rd[:, -1].float()), i
        if d.numel():
            assert float((d[:, :26].double() - rd[:, :26].double()).abs().max()) < 2e-2


# ================================================================================================= inventory
def test_inventory_of_bench_nms_workloads(cuda):
    """bench.py's NMS workloads: the poly_nms sweep 10k-200k (both variants) through rnms_indices and poly_gpu_nms, and
    the fused post-processing at B = 16 on 1024^2 level shapes with the bench's test_cfg at score_thr 0 and 0.05"""
    from orientedreppoints_b200.synth import const_density_extent, gen_rotated_boxes
    seen = {}
    for n in (10000, 20000, 50000, 100000, 200000):
        for dense in (False, True):
            d = gen_rotated_boxes(n, seed=100, extent=1024.0 if dense else const_density_extent(n))
            _, p, _ = _rnms(cuda, d, 0.1)
            seen.setdefault(_sig(p), "rnms_indices n=%d dense=%s" % (n, dense))
            _, p = _poly_gpu_nms(d, 0.1)
            seen.setdefault(_sig(p), "poly_gpu_nms n=%d dense=%s" % (n, dense))
    cls, ref = _head_outs(cuda, 16, LEVELS_1024, seed=3)
    metas = [dict(scale_factor=1.0)] * 16
    for thr in (0.0, 0.05):
        _, _, counts, p = _fused(cls, ref, _cfg(thr), metas)
        assert min(counts) >= 0
        seen.setdefault(_sig(p), "orp_head_postprocess B=16 score_thr=%g" % thr)
    print("signatures:", seen)
    missing = {s: w for s, w in seen.items() if s not in PARITY}
    assert not missing, missing
    assert len(seen) == 5


# ================================================================================================= strips
@pytest.mark.parametrize("n", [16383, 16384, 20000, 100000, 200000])
@pytest.mark.parametrize("dense", [False, True])
def test_poly_gpu_nms_strips(cuda, po, n, dense):
    """poly_gpu_nms - and orp_rnms without segments - cut sets of >= 16384 boxes into y strips; the keep list equals the
    oracle's and the strip-less run's"""
    from orientedreppoints_b200.synth import const_density_extent, gen_rotated_boxes
    d = gen_rotated_boxes(n, seed=11, extent=1024.0 if dense else const_density_extent(n))
    got, p = _poly_gpu_nms(d, 0.1)
    R = 4 if n >= 16384 else 1
    _assert_plan(p, (1, R, 0, 0, GUARD, DESC, 0), seg_limit=1, n=n)
    assert p["sweep_bits"] == (48 if R == 4 else 32) + 1
    flat = _strip_less(cuda, d, 0.1)
    assert np.array_equal(got, flat)
    kept, pk, _ = _rnms(cuda, d, 0.1)                # NaN keeps: the same decisions on these non-degenerate boxes
    _assert_plan(pk, (1, R, 0, 0, KEEPS, DESC, 0), seg_limit=1)
    assert np.array_equal(kept, got)
    if n <= 100000 and (dense or n <= 20000):       # the O(n * kept) oracle loop on the larger sparse sets takes minutes
        assert np.array_equal(got, po.nms_poly_f64(d, 0.1, fast=True))


@pytest.mark.parametrize("h", [4, 16, 64])
def test_strip_boundaries(cuda, po, h):
    d = _equal_height_boxes(20000, h, seed=h)
    got, p = _poly_gpu_nms(d, 0.1)
    _assert_plan(p, (1, 4, 0, 0, GUARD, DESC, 0))
    flat = _strip_less(cuda, d, 0.1)
    ref = po.nms_poly_f64(d, 0.1, fast=True)
    assert np.array_equal(flat, ref)
    assert np.array_equal(got, ref)


def test_tall_box_and_far_coordinates(cuda, po):
    """one 8000 px tall box among small ones (strip height = its height / 3), clusters at -5000 and at +16000.  The tall
    box starts half-way into a strip, so it is registered in four strips, and a shorter box with a better score overlaps
    only its top (IoU 0.11): the pair belongs to the tall box's fourth strip"""
    from orientedreppoints_b200.synth import gen_rotated_boxes
    d = gen_rotated_boxes(20000, seed=5, extent=2048.0)
    d[:10000, 0:8] -= np.float32(5000.0)
    d[10000:, 0:8] += np.float32(16000.0 - 2048.0)
    d[7, :8] = np.array([-4000, -5000, -3950, -5000, -3950, 3000, -4000, 3000], np.float32)
    y0 = d[:, 1:8:2].min()
    s = np.float32(8000.0) * (np.float32(1.0001) / np.float32(3.0))          # the kernel's strip height, fp32
    ya = np.float32(y0 + np.float32(10.5) * s)
    d[7, :8] = np.array([-4000, ya, -3950, ya, -3950, ya + 8000, -4000, ya + 8000], np.float32)
    yb = ya + np.float32(7000)
    d[8, :8] = np.array([-4000, yb, -3950, yb, -3950, yb + 2000, -4000, yb + 2000], np.float32)
    d[8, 8] = np.float32(0.9999)
    d[7, 8] = np.float32(0.9998)
    assert int(np.floor((ya + 8000 - y0) / s)) - int(np.floor((ya - y0) / s)) == 3
    assert int(np.floor((yb - y0) / s)) == int(np.floor((ya + 8000 - y0) / s))
    got, p = _poly_gpu_nms(d, 0.1)
    _assert_plan(p, (1, 4, 0, 0, GUARD, DESC, 0))
    flat = _strip_less(cuda, d, 0.1)
    ref = po.nms_poly_f64(d, 0.1, fast=True)
    assert 7 not in ref.tolist()
    assert np.array_equal(got, ref) and np.array_equal(flat, ref)


@pytest.mark.parametrize("kind", ["segments", "task1"])
def test_zero_height_strips(cuda, po, kind):
    """zero-height boxes only: strip height 1e-6, strip indices wrap past 16 bits.  'segments' are traversed p,q,q,p, so
    every fan term cancels exactly, union is 0 and under poly_nms's guard the best box suppresses all others; 'task1'
    lines leave a residue in some pairs, so a few of them survive"""
    rng = np.random.RandomState(9)
    n = 20000
    if kind == "segments":
        x0 = np.round(rng.uniform(0, 4000, n) * 4) / 4
        y = np.round(rng.uniform(0, 4000, n) * 4) / 4
        x1 = x0 + rng.randint(1, 64, n)
        q = np.stack([x0, y, x1, y, x1, y, x0, y], 1).astype(np.float32)
    else:
        q = _task1_lines(n, rng)
    d = _with_scores(q, rng)
    got, p = _poly_gpu_nms(d, 0.1)
    _assert_plan(p, (1, 4, 0, 0, GUARD, DESC, 0))
    ref = po.nms_poly_f64(d, 0.1)
    if kind == "segments":
        assert ref.tolist() == [int(np.argmax(d[:, 8]))]
    else:
        assert 1 < len(ref) < 100
    assert np.array_equal(got, ref)


# ================================================================================================= retry / overflow
@pytest.mark.parametrize("mode", ["exact64", "compat32"])
def test_candidate_list_retry(cuda, po, mode):
    """8192 near-identical boxes in one segment: the candidate pairs far exceed the first capacity (2^21), the call
    re-sweeps once with the exact size"""
    rng = np.random.RandomState(1)
    n = 8192
    x0, y0 = 500 + rng.uniform(-12, 12, n), 500 + rng.uniform(-12, 12, n)
    x1, y1 = x0 + 200 + rng.uniform(-12, 12, n), y0 + 200 + rng.uniform(-12, 12, n)
    q = np.stack([x0, y0, x1, y0, x1, y1, x0, y1], 1).astype(np.float32)
    d = _with_scores(q, rng)
    got, p, st = _rnms(cuda, d, 0.9, mode=mode)
    _assert_plan(p, (1 if mode == "exact64" else 0, 1, 0, 0, KEEPS, DESC, 1), attempts=2, cap_first=256 * n)
    assert p["cap_final"] > p["cap_first"] and st["edges"] > p["cap_first"] and st["overflow"] == 0
    ref = po.nms_poly_f64(d, 0.9, fast=True) if mode == "exact64" else po.nms_f32(d, np.float32(0.9))
    print(mode, "kept", len(ref), "edges", st["edges"])
    assert len(ref) > 10
    assert np.array_equal(got, ref)


def _overflow_outs(cuda):
    """B = 1, one 32x32 level at stride 8, 15 classes, the same reppoints at every location spanning +-100 stride units:
    every box of a class is a shifted copy of one ~1600 px box, every pair has IoU > 0.4 -> 15 * C(1024, 2) = 7.9 M
    candidates against a capacity of 256 * 15 * 1028 = 3.9 M.  The detector's four other levels are 1x1 with scores below
    the threshold."""
    g = torch.Generator().manual_seed(2)
    cls = [(torch.rand(1, 32, 32, 15, generator=g) * 2 - 1).to(cuda)] + [torch.full((1, 1, 1, 15), -50.0, device=cuda)] * 4
    pts = torch.tensor([[-100, -90], [-95, 100], [100, 95], [90, -100], [0, 0], [50, 20], [-30, 60], [10, -70], [-60, -20]],
                       dtype=torch.float32)
    ref = [pts.reshape(1, 1, 1, 18).expand(1, 32, 32, 18).contiguous().to(cuda)] + [torch.zeros(1, 1, 1, 18, device=cuda)] * 4
    return cls, ref


def test_no_sync_overflow(cuda, po):
    from orientedreppoints_b200 import _lib
    from orientedreppoints_b200.core.get_bboxes import get_bboxes
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    cls, ref = _overflow_outs(cuda)
    cfg = _cfg(0.05)
    metas = [dict(scale_factor=1.0)]
    _, _, counts, p = _fused(cls, ref, cfg, metas)
    _assert_plan(p, (1, 1, 1, 1, KEEPS, ASC, 0), attempts=1, cap_first=256 * 1028 * 15)
    assert counts == [-1]
    assert _lib.last_nms_stats()["overflow"] == 1
    # the detector turns the poisoned count into an error instead of returning incomplete results
    det = OrientedRepPointsDetector.__new__(OrientedRepPointsDetector)
    det.device, det.test_cfg = cuda, cfg
    det.forward_dense = lambda img: ([(c, None, r) for c, r in zip(cls, ref)], None)
    with pytest.raises(_lib.OrpError):
        det.simple_test(torch.zeros(1, 3, 256, 256, device=cuda))
    # the same rows through the host-synchronised entry point: retried, exact
    bb, sc = get_bboxes(cls, ref, STRIDES, metas, cfg, rescale=False, nms=False)[0]
    valid = sc[:, 1:] > cfg["score_thr"]
    nz = valid.nonzero()
    rows, labels = nz[:, 0], nz[:, 1]
    dets = torch.cat([bb[rows], sc[:, 1:][valid][:, None]], 1).cpu().numpy()
    seg = labels.cpu().numpy().astype(np.int32)
    got, p, st = _rnms(cuda, dets, 0.4, segments=seg, order=ASC)
    _assert_plan(p, (1, 1, 0, 0, KEEPS, ASC, 1), attempts=2)
    assert st["overflow"] == 0 and st["edges"] > 7_000_000
    assert np.array_equal(got, _segmented_oracle(po, dets, seg, 0.4, order=ASC))
    # and a normal call right afterwards is correct
    cls2, ref2 = _head_outs(cuda, 2, [(32, 32), (16, 16)], seed=4)
    metas2 = [dict(scale_factor=1.0)] * 2
    d2, l2, c2, p2 = _fused(cls2, ref2, cfg, metas2)
    assert min(c2) >= 0 and p2["attempts"] == 1
    _check_fused_vs_mirror(cls2, ref2, cfg, metas2, d2, l2, c2)


# ================================================================================================= resolve chains
@pytest.mark.parametrize("scores", ["descending", "ascending", "zigzag"])
def test_resolve_chains(cuda, po, scores):
    """4096 squares in a row, each overlapping only its two neighbours (IoU 0.25 > 0.2): every decision waits for the one
    before it, so the resolve takes about a round per box"""
    n = 4096
    x0 = np.arange(n, dtype=np.float32) * 6
    q = np.stack([x0, 0 * x0, x0 + 10, 0 * x0, x0 + 10, 0 * x0 + 10, x0, 0 * x0 + 10], 1).astype(np.float32)
    if scores == "descending":
        rank = np.arange(n)
    elif scores == "ascending":
        rank = np.arange(n)[::-1]
    else:                                   # from the middle outwards, alternating sides
        m = n // 2
        seq = [m] + [v for k in range(1, n) for v in (m + k, m - k) if 0 <= v < n][:n - 1]
        rank = np.empty(n, np.int64)
        rank[np.asarray(seq)] = np.arange(n)
    d = np.concatenate([q, (1.0 - rank / n).astype(np.float32)[:, None]], 1).astype(np.float32)
    got, p, st = _rnms(cuda, d, 0.2)
    _assert_plan(p, (1, 1, 0, 0, KEEPS, DESC, 0))
    print(scores, "rounds", st["rounds"])
    assert st["rounds"] >= n // 4
    assert np.array_equal(got, po.nms_poly_f64(d, 0.2, fast=True))


# ================================================================================================= scores and unions
def test_scores_and_ties(cuda, po):
    from orientedreppoints_b200.synth import gen_rotated_boxes
    base = gen_rotated_boxes(3000, seed=21, extent=600.0)
    rng = np.random.RandomState(3)
    cases = {}
    d = base.copy(); d[:, 8] = 0.5; cases["equal"] = d
    d = base.copy(); d[:, 8] = np.where(rng.rand(3000) < 0.5, np.float32(0.0), np.float32(-0.0)); cases["signed_zero"] = d
    d = base.copy()
    d[:, 8] = np.where(rng.rand(3000) < 0.3, rng.uniform(0, 1, 3000).astype(np.float32),
                       rng.randint(1, 1 << 23, 3000).astype(np.uint32).view(np.float32))
    d[:100, 8] = np.float32(0.0); d[100:200, 8] = np.float32(-0.0); d[200:300, 8] = np.uint32(5).view(np.float32)
    cases["subnormal"] = d
    for name, d in cases.items():
        got, p, _ = _rnms(cuda, d, 0.3)
        _assert_plan(p, (1, 1, 0, 0, KEEPS, DESC, 0))
        ref = po.nms_poly_f64(d, 0.3, fast=True)
        assert np.array_equal(ref, _greedy(po, d, 0.3, "keeps")), name      # the oracle's order breaks ties by index
        assert np.array_equal(got, ref), name


def test_non_finite_rows_keep(cuda, po):
    """NAN_KEEPS: a row with a non-finite coordinate is kept and suppresses nothing"""
    from orientedreppoints_b200.synth import gen_rotated_boxes
    d = gen_rotated_boxes(3000, seed=22, extent=600.0)
    rng = np.random.RandomState(4)
    bad = rng.choice(3000, 200, replace=False)
    d[bad, rng.randint(0, 8, 200)] = rng.choice(np.array([np.nan, np.inf, -np.inf], np.float32), 200)
    for order in (DESC, ASC):
        got, p, _ = _rnms(cuda, d, 0.3, order=order)
        _assert_plan(p, (1, 1, 0, 0, KEEPS, order, 0))
        ref = _greedy(po, d, 0.3, "keeps")
        assert set(bad.tolist()) <= set(ref.tolist())
        assert np.array_equal(got, ref if order == DESC else np.sort(ref))


def _zero_area_set(seed):
    """3000 random boxes and 400 zero-area ones (points, segments, collinear quads, some crossing each other) in one
    set; coordinates are positive with the minimum in [0, 1), so ResultMerge's move of a set to its own integer origin
    changes nothing"""
    from orientedreppoints_b200.synth import gen_rotated_boxes
    rng = np.random.RandomState(seed)
    a = gen_rotated_boxes(3000, seed=seed, extent=800.0)[:, :8] + np.float32(128.0)
    z = _zero_area_boxes(400, rng, 1000.0) + np.float32(8.0)
    q = np.concatenate([a, z, np.full((1, 8), 0.5, np.float32)])
    q = q[rng.permutation(q.shape[0])]
    return _with_scores(q, rng)


@pytest.mark.parametrize("seed", [31, 32])
def test_zero_area_public_entry_points(cuda, po, seed):
    """zero-area boxes in each union convention through its public entry point: rnms (NaN keeps), poly_gpu_nms (guard:
    union 0 -> IoU 1) and py_cpu_nms_poly (NaN suppresses, every pair): zero-area boxes suppress each other wherever they
    are; py_cpu_nms_poly_fast only where the axis-aligned hulls overlap"""
    from orientedreppoints_b200.dota import result_merge as rm
    from orientedreppoints_b200.ops import rnms
    d = _zero_area_set(seed)
    d64 = d.astype(np.float64)
    unfiltered = po.nms_poly_f64(d, 0.1)
    assert np.array_equal(unfiltered, _greedy(po, d, 0.1, "all"))
    fast = po.nms_poly_f64(d, 0.1, fast=True)
    assert len(fast) > len(unfiltered)                       # the set tells the conventions apart

    _, inds = rnms(torch.from_numpy(d).to(cuda), 0.1)
    _assert_plan(_plan(), (1, 1, 0, 0, KEEPS, ASC, 0))
    assert np.array_equal(inds.cpu().numpy(), np.sort(_greedy(po, d, 0.1, "keeps")))

    got, p = _poly_gpu_nms(d, 0.1)
    _assert_plan(p, (1, 1, 0, 0, GUARD, DESC, 0))
    assert np.array_equal(got, unfiltered)

    got = np.asarray(rm.py_cpu_nms_poly(d64, 0.1))
    _assert_plan(_plan(), (1, 1, 0, 0, SUPP_ALL, DESC, 0))
    assert np.array_equal(got, unfiltered)

    got = np.asarray(rm.py_cpu_nms_poly_fast(d64, 0.1))
    _assert_plan(_plan(), (1, 1, 0, 0, SUPP, DESC, 0))
    assert np.array_equal(got, fast)


def test_zero_area_task1_lines(cuda, po):
    """collinear %.1f lines whose pairs are decided by the fp64 algorithm, better-ranked box first: the two rows below
    have IoU -1 and both survive; 50 lines alone and 300 mixed into random boxes, through poly_gpu_nms,
    py_cpu_nms_poly and segmented ORP_UNION_NAN_SUPPRESSES_ALL"""
    from orientedreppoints_b200.dota import result_merge as rm
    from orientedreppoints_b200.synth import gen_rotated_boxes
    pair = np.array([[0.1, 417, 146.8, 417, 720.3, 417, 302.3, 417, 0.9],
                     [27.4, 419.2, 204.5, 419.2, 878.1, 419.2, 685.2, 419.2, 0.8]], np.float32)
    assert po.nms_poly_f64(pair, 0.1).tolist() == [0, 1]
    assert _poly_gpu_nms(pair, 0.1)[0].tolist() == [0, 1]
    moved = pair.copy()
    moved[:, 1:8:2] -= np.float32(417.0)                    # ResultMerge moves a set to its own integer origin first
    assert rm.py_cpu_nms_poly(pair.astype(np.float64), 0.1) == po.nms_poly_f64(moved, 0.1).tolist()
    rng = np.random.RandomState(41)
    alone = _with_scores(np.concatenate([_task1_lines(50, rng), np.full((1, 8), 0.5, np.float32)]), rng)
    rand = gen_rotated_boxes(3000, seed=42, extent=800.0)[:, :8] + np.float32(128.0)   # minimum 0.5: no origin move
    mixed = np.concatenate([rand, _task1_lines(300, rng), np.full((1, 8), 0.5, np.float32)])
    mixed = _with_scores(mixed[rng.permutation(mixed.shape[0])], rng)
    for d in (alone, mixed):
        ref = po.nms_poly_f64(d, 0.1)
        nz = int(np.sum(np.isin(ref, np.nonzero(d[:, 1] == d[:, 3])[0])))
        assert 1 < nz < 50                                  # neither "all kept" nor "only the best kept"
        got, p = _poly_gpu_nms(d, 0.1)
        _assert_plan(p, (1, 1, 0, 0, GUARD, DESC, 0))
        assert np.array_equal(got, ref)
        got = np.asarray(rm.py_cpu_nms_poly(d.astype(np.float64), 0.1))
        _assert_plan(_plan(), (1, 1, 0, 0, SUPP_ALL, DESC, 0))
        assert np.array_equal(got, ref)
    seg = rng.randint(0, 5, mixed.shape[0]).astype(np.int32)
    got, p, _ = _rnms(cuda, mixed, 0.1, segments=seg, union=SUPP_ALL)
    _assert_plan(p, (1, 1, 0, 0, SUPP_ALL, DESC, 0))
    keep = np.sort(np.concatenate([np.nonzero(seg == s)[0][po.nms_poly_f64(mixed[seg == s], 0.1)] for s in range(5)]))
    assert np.array_equal(got, keep[np.argsort(-mixed[keep, 8], kind="stable")])


@pytest.mark.parametrize("a_first", [True, False])
def test_degenerate_pair_order_and_hulls(cuda, po, a_first):
    """pairs whose decision depends on how the reference calls it.  (a, b): the fp64 IoU is -1 with a first and NaN with
    b first, so the better-ranked box must be the first polygon.  (v, c): a vertical segment (zero-width hull) crossing a
    diagonal one; py_cpu_nms_poly_fast compares a pair only when the hulls overlap with positive area, so it never
    compares these.  Every convention through rnms_indices, against its oracle"""
    a = [645.75, 451.5, 638.75, 452.5, 624.75, 454.5, 631.75, 453.5]
    b = [637, 452, 649, 468, 673, 500, 661, 484]
    v = [100, 50, 100, 150, 100, 150, 100, 50]
    c = [50, 50, 150, 150, 150, 150, 50, 50]
    hi, lo = (0.9, 0.8) if a_first else (0.8, 0.9)
    d = np.array([a + [hi], b + [lo], v + [hi], c + [lo]], np.float32)
    assert po.iou_poly_f64(np.array([a]), np.array([b]))[0] == -1.0
    assert np.isnan(po.iou_poly_f64(np.array([b]), np.array([a]))[0])
    fast, full = po.nms_poly_f64(d, 0.1, fast=True), po.nms_poly_f64(d, 0.1)
    for union, ref in ((KEEPS, _greedy(po, d, 0.1, "keeps")), (SUPP, fast), (SUPP_ALL, full), (GUARD, full)):
        got, p, _ = _rnms(cuda, d, 0.1, union=union)
        _assert_plan(p, (1, 1, 0, 0, union, DESC, 0))
        assert np.array_equal(got, ref), (union, got, ref)


def test_zero_area_per_segment(cuda, po):
    """segmented: in every segment the best zero-area box is kept and suppresses the segment's other zero-area boxes"""
    d = _zero_area_set(33)
    seg = np.random.RandomState(5).randint(0, 7, d.shape[0]).astype(np.int32)
    got, p, _ = _rnms(cuda, d, 0.1, segments=seg, union=SUPP_ALL)
    _assert_plan(p, (1, 1, 0, 0, SUPP_ALL, DESC, 0))
    keep = []
    for s in range(7):
        ids = np.nonzero(seg == s)[0]
        keep.append(ids[po.nms_poly_f64(d[ids], 0.1)])
    keep = np.sort(np.concatenate(keep))
    assert np.array_equal(got, keep[np.argsort(-d[keep, 8], kind="stable")])


# ================================================================================================= fused post-processing
def _exact_thr_logit(cuda, thr):
    """a float32 logit whose fp32 sigmoid is exactly `thr` (torch.sigmoid == the kernel's 1 / (1 + expf(-x))), or None"""
    if thr == 0.0:
        return -200.0                                       # expf(200) = inf -> sigmoid exactly 0
    x0 = np.float32(np.log(thr / (1 - thr)))
    xs = x0 + np.arange(-4096, 4097, dtype=np.float32) * np.spacing(x0)
    s = torch.sigmoid(torch.from_numpy(xs.astype(np.float32)).to(cuda)).cpu().numpy()
    hit = np.nonzero(s == np.float32(thr))[0]
    return float(xs[hit[0]]) if hit.size else None


def _adversarial_outs(cuda, B, levels, seed, score_thr):
    """quantised logits (max-scores tie across locations and levels), saturated logits (sigmoid exactly 1.0), logits whose
    sigmoid is exactly score_thr, collinear reppoints (zero-area boxes).  The collinear sets sit on every fourth row and
    column of the first level and are about one stride long, so no two zero-area boxes have overlapping axis-aligned hulls:
    rnms (NaN keeps) and the oracle's py_cpu_nms_poly_fast (NaN suppresses, only compared where the hulls overlap) then
    agree on them."""
    cls, ref = _head_outs(cuda, B, levels, seed, logit_mu=-2.5)
    g = torch.Generator().manual_seed(seed + 1)
    xt = _exact_thr_logit(cuda, score_thr)
    for c in cls:
        c.copy_((c * 2).round() / 2)
        u = torch.rand(c.shape, generator=g).to(cuda)
        c[u < 0.01] = 30.0
        if xt is not None:
            c[(u >= 0.01) & (u < 0.03)] = xt
    t = torch.linspace(-0.5, 0.5, 9, device=cuda)
    ref[0][:, ::4, ::4] = torch.stack([t * 0.5, t], 1).reshape(18)        # (dy, dx) along one direction
    return cls, ref


@pytest.mark.parametrize("score_thr", [0.0, 0.05])
def test_fused_production_shapes(cuda, po, score_thr):
    """bench configuration: B = 16 on 1024^2 level shapes, nms_pre 2000 (two levels through the top-k sort),
    max_per_img 2000 (more survive: the score-sorted select branch), a different scale_factor per image"""
    B = 16
    cls, ref = _adversarial_outs(cuda, B, LEVELS_1024, seed=7, score_thr=score_thr)
    metas = [dict(scale_factor=0.5 + 0.125 * i) for i in range(B)]
    cfg = _cfg(score_thr)
    dets, labels, counts, p = _fused(cls, ref, cfg, metas)
    _assert_plan(p, (1, 1, 1, 1, KEEPS, ASC, 0), seg_limit=B * 15, n=B * 5344 * 15)
    print("counts", counts)
    assert min(counts) >= 0 and max(counts) == 2000
    _check_fused_vs_mirror(cls, ref, cfg, metas, dets, labels, counts)
    _check_fused_vs_oracle(cls, ref, cfg, metas, dets, labels, counts, images=range(B))


def test_fused_exactly_max_per_img(cuda, po):
    """exactly max_per_img survivors keep candidate order (multiclass_rnms sorts by score only when MORE survive)"""
    levels = [(64, 64), (32, 32)]
    cls, ref = _head_outs(cuda, 2, levels, seed=8, logit_mu=-1.0)
    metas = [dict(scale_factor=1.0)] * 2
    _, _, counts, _ = _fused(cls, ref, _cfg(0.05, max_per_img=100000), metas)
    cap = counts[0]
    assert counts[1] != cap
    cfg = _cfg(0.05, max_per_img=cap)
    dets, labels, counts2, p = _fused(cls, ref, cfg, metas)
    assert counts2 == [cap, min(counts[1], cap)]
    _check_fused_vs_mirror(cls, ref, cfg, metas, dets, labels, counts2)
    _check_fused_vs_oracle(cls, ref, cfg, metas, dets, labels, counts2, images=range(2))


@pytest.mark.parametrize("score_thr", [0.0, 0.05])
def test_fused_segmented_strips(cuda, po, score_thr):
    """nms_pre = -1 at 1024^2: 21 824 candidates per (image, class) segment, so the fused NMS cuts them into strips"""
    B = 2
    cls, ref = _head_outs(cuda, B, LEVELS_1024, seed=12, logit_mu=-3.5)
    metas = [dict(scale_factor=1.0), dict(scale_factor=0.75)]
    cfg = _cfg(score_thr, nms_pre=-1, max_per_img=100000)
    dets, labels, counts, p = _fused(cls, ref, cfg, metas)
    _assert_plan(p, (1, 4, 1, 1, KEEPS, ASC, 0), seg_limit=B * 15, n=B * 21824 * 15)
    assert p["sweep_bits"] == 48 + 5
    _check_fused_vs_mirror(cls, ref, cfg, metas, dets, labels, counts)
    if score_thr > 0:                                   # every (image, class) against the oracle
        _check_fused_vs_oracle(cls, ref, cfg, metas, dets, labels, counts, images=range(B))


# ================================================================================================= small kernels
def test_dcn_offsets_multi_bitwise(cuda):
    """orp_dcn_offsets_multi: offset = ((1 - g) * pts + g * pts) - base[i % 18], each operation rounded to fp32, for 5
    problems of ragged sizes in one launch"""
    import ctypes
    from orientedreppoints_b200 import _lib
    rng = np.random.RandomState(6)
    g = np.float32(0.1)
    base = rng.uniform(-1, 1, 18).astype(np.float32)
    sizes = [18 * k for k in (1, 37, 0, 4099, 700)]
    pts = [torch.from_numpy(rng.normal(0, 3, max(s, 1)).astype(np.float32)).to(cuda) for s in sizes]
    off = [torch.full((max(s, 1),), float("nan"), device=cuda) for s in sizes]
    P = (ctypes.c_void_p * 5)(*[t.data_ptr() for t in pts])
    O = (ctypes.c_void_p * 5)(*[t.data_ptr() for t in off])
    N = (ctypes.c_longlong * 5)(*sizes)
    bp = (ctypes.c_float * 18)(*base.tolist())
    _lib.check(_lib.lib().orp_dcn_offsets_multi(5, P, O, N, ctypes.c_float(g), bp, _lib.current_stream_ptr()), "dcn_offsets")
    torch.cuda.synchronize()
    og = np.float32(1) - g
    for s, t, o in zip(sizes, pts, off):
        x = t.cpu().numpy()[:s]
        want = (og * x + g * x) - np.tile(base, s // 18)
        got = o.cpu().numpy()
        assert np.array_equal(got[:s].view(np.uint32), want.astype(np.float32).view(np.uint32))
        if s == 0:
            assert np.isnan(got[0])                         # nothing written


def test_pack_detections_layout(cuda):
    """orp_pack_detections: [B, cap + 1, 28] = 27 detection values | label per row, row `cap` carries the count"""
    from orientedreppoints_b200 import _lib
    B, cap = 3, 7
    g = torch.Generator().manual_seed(0)
    dets = torch.randn(B, cap, 27, generator=g).to(cuda)
    labels = torch.randint(-1, 15, (B, cap), generator=g).to(cuda)
    counts = torch.tensor([0, 7, 3], dtype=torch.int32, device=cuda)
    out = torch.full((B, cap + 1, 28), float("nan"), device=cuda)
    _lib.check(_lib.lib().orp_pack_detections(_lib.ptr(dets), _lib.ptr(labels), _lib.ptr(counts), B, cap, _lib.ptr(out),
                                              _lib.current_stream_ptr()), "pack")
    torch.cuda.synchronize()
    want = torch.zeros(B, cap + 1, 28, device=cuda)
    want[:, :cap, :27] = dets
    want[:, :cap, 27] = labels.float()
    want[:, cap, 0] = counts.float()
    assert torch.equal(out, want)
