"""GPU: multi-view test-time augmentation as one device pipeline (orp_head_postprocess_aug, get_bboxes_aug_fused, the
batched aug_test) against the op-by-op mirror of mmdet/models/detectors/orientedreppoints_detector.py:48-144
(get_bboxes(nms=False) per view -> flip / scale map-back -> torch.cat -> ONE multiclass_rnms) fed the SAME head outputs.
Every comparison is bit exact."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

STRIDES = (8, 16, 32, 64, 128)
LEVELS_1024 = [(128, 128), (64, 64), (32, 32), (16, 16), (8, 8)]
LEVELS_960 = [(120, 120), (60, 60), (30, 30), (15, 15), (8, 8)]
# rotated-NMS plan signatures (lazy, R, no_sync, flags_out, union_mode, order, retried) that tests/test_nms_plans_gpu.py
# compares with the CPU oracle through the fused head: test_fused_production_shapes, test_fused_segmented_strips
COVERED_PLANS = {(1, 1, 1, 1, 0, 0, 0), (1, 4, 1, 1, 0, 0, 0)}


def _cfg(score_thr, nms_pre=2000, max_per_img=2000):
    return dict(nms_pre=nms_pre, min_bbox_size=0, score_thr=score_thr, nms=dict(type='rnms', iou_thr=0.4),
                max_per_img=max_per_img)


def _view_outs(cuda, B, levels, seed, logit_mu=-2.0, spread=1.5):
    g = torch.Generator().manual_seed(seed)
    cls = [(torch.randn(B, h, w, 15, generator=g) * 1.5 + logit_mu).to(cuda) for h, w in levels]
    ref = [(torch.randn(B, h, w, 18, generator=g) * spread).to(cuda) for h, w in levels]
    return cls, ref


def _meta(width, flip, sf, B):
    return [dict(img_shape=(256, width, 3), scale_factor=sf, flip=flip) for _ in range(B)]


def _eager(cls, ref, metas, cfg, rescale):
    """the eager aug_test merge, restated: per image (dets [k, 9] box | score, labels [k])"""
    from orientedreppoints_b200.core.bbox_nms import multiclass_rnms
    from orientedreppoints_b200.core.get_bboxes import get_bboxes
    nl = len(cls[0])
    out = []
    for i in range(cls[0][0].shape[0]):
        boxes, scores = [], []
        for c, p, ms in zip(cls, ref, metas):
            m = ms[i]
            b, s = get_bboxes([t[i:i + 1] for t in c], [t[i:i + 1] for t in p], STRIDES[:nl], [m], cfg, False, nms=False)[0]
            if m["flip"]:
                b = b.clone()
                b[:, 0::2] = m["img_shape"][1] - b[:, 0::2] - 1
            boxes.append(b / m["scale_factor"])
            scores.append(s)
        d, l = multiclass_rnms(torch.cat(boxes), torch.cat(scores), cfg["score_thr"], cfg["nms"], cfg["max_per_img"])
        if not rescale:
            d = d.clone()
            d[:, :8] *= metas[0][i]["scale_factor"]
        out.append((d, l))
    return out


def _fused(cls, ref, metas, cfg, rescale):
    from orientedreppoints_b200.core.get_bboxes import get_bboxes_aug_fused
    dets, labels, counts = get_bboxes_aug_fused(cls, ref, STRIDES[:len(cls[0])], metas, cfg, rescale)
    return dets, labels, counts.tolist()


def _assert_equal(dets, labels, counts, eager):
    for i, (d, l) in enumerate(eager):
        n = counts[i]
        assert n == d.shape[0], (i, n, d.shape)
        assert torch.equal(labels[i, :n], l), i
        assert torch.equal(dets[i, :n, 18:], d), (i, float((dets[i, :n, 18:] - d).abs().max()) if n else 0.0)
        assert not dets[i, :, :18].any() and not dets[i, n:].any()          # no reppoints; zero padding
        assert bool((labels[i, n:] == -1).all())


def test_python_float_division_is_a_reciprocal_product(cuda):
    """the finding the kernel's map-back rests on: torch divides a CUDA tensor by a Python float as x * (1.0f / sf), which is
    not x / sf (the division by a device tensor simple_test's rescale performs) for a factor like 0.9375"""
    x = (torch.rand(1 << 16, generator=torch.Generator().manual_seed(0)) * 1024).to(cuda)
    for sf in (0.9375, 1.171875, 0.78125):
        by_float = x / sf
        by_tensor = x / torch.tensor(sf, dtype=torch.float32, device=cuda).expand_as(x)
        recip = x * (torch.ones((), dtype=torch.float32, device=cuda) / torch.tensor(sf, dtype=torch.float32, device=cuda))
        assert torch.equal(by_float, recip), sf
        assert not torch.equal(by_float, by_tensor), sf


@pytest.mark.parametrize("rescale", [True, False], ids=["rescale", "first_view_frame"])
@pytest.mark.parametrize("max_per_img", [100000, 50], ids=["candidate_order", "best_by_score"])
@pytest.mark.parametrize("case", ["plain", "empty_view", "empty_image"])
def test_c_abi_three_views(cuda, case, max_per_img, rescale):
    """V = 3 views with different level shapes (the third flipped), B = 2, nms_pre 400: the first level of every view takes
    the top-k sort, the others do not; scale factors that are not powers of two"""
    B = 2
    shapes = [[(32, 48), (16, 24), (8, 12)], [(24, 40), (12, 20), (6, 10)], [(32, 48), (16, 24), (8, 12)]]
    outs = [_view_outs(cuda, B, lv, seed=20 + v) for v, lv in enumerate(shapes)]
    cls, ref = [o[0] for o in outs], [o[1] for o in outs]
    metas = [_meta(384, False, 1.0, B), _meta(317, False, 0.9375, B), _meta(380, True, 1.171875, B)]
    if case == "empty_view":                             # view 1 of image 0 has nothing above the threshold
        for c in cls[1]:
            c[0] = -10.0
    if case == "empty_image":                            # image 1 has nothing at all
        for v in cls:
            for c in v:
                c[1] = -10.0
    cfg = _cfg(0.05, nms_pre=400, max_per_img=max_per_img)
    dets, labels, counts = _fused(cls, ref, metas, cfg, rescale)
    eager = _eager(cls, ref, metas, cfg, rescale)
    _assert_equal(dets, labels, counts, eager)
    assert counts[0] > 0 and (counts[1] == 0) == (case == "empty_image")
    if max_per_img == 50:
        assert counts[0] == 50
    else:
        assert 50 < counts[0] < max_per_img


def test_cross_view_suppression(cuda):
    """identity view + flipped view of the mirrored input: every box has its twin in the other view, the views share NMS
    segments, so fewer boxes survive than the two views keep apart"""
    B, H, W, st = 2, 32, 48, 8
    cls, ref = _view_outs(cuda, B, [(H, W)], seed=5, logit_mu=-3.0)
    mcls = [cls[0].flip(2).contiguous()]
    mref = ref[0].flip(2).clone()
    mref[..., 1::2] = -mref[..., 1::2]                   # (dy, dx): dx mirrors
    width = (W - 1) * st + 1                             # w - ((W-1-x)*st) - 1 == x*st: the twin lands on the original
    ident, flipped = _meta(width, False, 1.0, B), _meta(width, True, 1.0, B)
    cfg = _cfg(0.05, nms_pre=-1, max_per_img=100000)
    _, _, c0 = _fused([cls], [ref], [ident], cfg, True)
    _, _, c1 = _fused([mcls], [[mref]], [flipped], cfg, True)
    dets, labels, both = _fused([cls, mcls], [ref, [mref]], [ident, flipped], cfg, True)
    _assert_equal(dets, labels, both, _eager([cls, mcls], [ref, [mref]], [ident, flipped], cfg, True))
    for i in range(B):
        assert c0[i] > 50 and c1[i] > 50 and 0 < both[i] < 1.1 * max(c0[i], c1[i]), (c0, c1, both)


@pytest.mark.parametrize("nms_pre,max_per_img", [(400, 100000), (400, 80), (-1, 100000)])
def test_one_view_is_the_simple_pipeline(cuda, nms_pre, max_per_img):
    """V = 1, no flip, scale 1: boxes, scores, labels and counts of orp_head_postprocess on the same tensors"""
    from orientedreppoints_b200.core.get_bboxes import get_bboxes_fused
    B = 3
    cls, ref = _view_outs(cuda, B, [(32, 48), (16, 24), (8, 12)], seed=9)
    cfg = _cfg(0.05, nms_pre=nms_pre, max_per_img=max_per_img)
    sd, sl, sc = get_bboxes_fused(cls, ref, STRIDES[:3], [dict(scale_factor=1.0)] * B, cfg, rescale=False)
    dets, labels, counts = _fused([cls], [ref], [_meta(384, False, 1.0, B)], cfg, True)
    assert counts == sc.tolist() and min(counts) > 0
    assert torch.equal(labels, sl) and torch.equal(dets[:, :, 18:], sd[:, :, 18:])
    assert sd[:, :, :18].any() and not dets[:, :, :18].any()


def _freeze_dense(det, views):
    """GroupNorm sums use atomics (not bit-reproducible run to run): evaluate the dense graph once per view and let
    both sides of a comparison consume the same outputs"""
    cache = {id(v): det.forward_dense(v) for v in views}
    det.forward_dense = lambda v: cache[id(v)]
    return cache


def test_detector_batched_aug_test(cuda):
    """N = 3 images x (2 scales x flip) through the detector: one dense pass per view, the fused merge equals the eager
    merge image by image on slices of the same dense outputs, in every return form"""
    from orientedreppoints_b200.core.transforms import rbbox2result
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    from orientedreppoints_b200.weights import random_state_dict
    det = OrientedRepPointsDetector(random_state_dict(50, seed=0, reference_init=True), 50, cuda, "fp32",
                                    test_cfg=dict(score_thr=0.0, max_per_img=300))
    g = torch.Generator().manual_seed(6)
    a = torch.randn(3, 3, 128, 160, generator=g).to(cuda)
    b = torch.randn(3, 3, 96, 128, generator=g).to(cuda)
    views = [a, a.flip(-1), b, b.flip(-1)]
    metas = [[dict(img_shape=(128, 160, 3), scale_factor=1.0, flip=f) for _ in range(3)] for f in (False, True)] + \
            [[dict(img_shape=(90, 120, 3), scale_factor=0.75, flip=f) for _ in range(3)] for f in (False, True)]
    cache = _freeze_dense(det, views)
    dense = [cache[id(v)][0] for v in views]
    cls, ref = [[o[0] for o in outs] for outs in dense], [[o[2] for o in outs] for outs in dense]
    for rescale in (True, False):
        eager = _eager(cls, ref, metas, det.test_cfg, rescale)
        want = [rbbox2result(d, l, 16) for d, l in eager]
        dets, labels, counts = det.aug_test(views, metas, rescale, None, return_tensors="padded")
        cnt = counts.tolist()
        _assert_equal(dets, labels, cnt, eager)
        assert max(cnt) == 300                                       # more survive: the best-by-score select
        got = det.aug_test(views, metas, rescale)
        assert len(got) == 3
        for res, ref_res in zip(got, want):
            assert len(res) == 15 and all(np.array_equal(x, y) and x.shape[1] == 9 for x, y in zip(res, ref_res))
        # the eager route of the same call (fused_post off), looped over the images of the batch
        det.fused_post = False
        loop = det.aug_test(views, metas, rescale)
        det.fused_post = True
        assert all(np.array_equal(x, y) for res, ref_res in zip(loop, want) for x, y in zip(res, ref_res))
    # one image per view keeps the single-image return form: that image's list itself (rescale is False here)
    one = [v[1:2] for v in views]
    sliced = {id(o): ([tuple(t[1:2] for t in lvl) for lvl in cache[id(v)][0]], None) for o, v in zip(one, views)}
    det.forward_dense = lambda v: sliced[id(v)]
    single = det.aug_test(one, [[m[1]] for m in metas], False)
    assert len(single) == 15 and all(np.array_equal(x, y) for x, y in zip(single, got[1]))
    with pytest.raises(ValueError):
        det.aug_test(views[:2], metas[:3])


def _pipeline(scales, flip):
    return [dict(type='LoadImageFromFile'),
            dict(type='MultiScaleFlipAug', img_scale=scales, flip=flip,
                 transforms=[dict(type='RotateResize', keep_ratio=True), dict(type='RotateRandomFlip'),
                             dict(type='Normalize', mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375], to_rgb=True),
                             dict(type='Pad', size_divisor=32), dict(type='ImageToTensor', keys=['img']),
                             dict(type='Collect', keys=['img'])])]


def test_detect_image_one_aug_test_call_per_batch(cuda):
    """a 2 scales x flip pipeline over 6 tiles in batches of 4: two aug_test calls per composition, each over a whole batch
    of 4 views, and the tensor composition equals the text composition string for string (the detections of a batch are
    served from one run: GroupNorm sums use atomics)"""
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    from orientedreppoints_b200.dota.pipeline import DOTA_CLASSES, detect_image, detect_image_tensors
    from orientedreppoints_b200.weights import random_state_dict
    det = OrientedRepPointsDetector(random_state_dict(50, seed=0, reference_init=True), 50, cuda, "bf16",
                                    test_cfg=dict(score_thr=0.0, max_per_img=60))
    real, cache, calls = det.aug_test, {}, []

    def aug_test(imgs, img_metas, rescale=False, valid_hws=None):
        calls.append((len(imgs), imgs[0].shape[0], rescale))
        k = tuple((tuple(v.shape), int(v.long().sum())) for v in imgs)
        if k not in cache:
            cache[k] = real(imgs, img_metas, rescale, valid_hws)
        return cache[k]
    det.aug_test = aug_test
    img = np.random.RandomState(11).randint(0, 256, size=(420, 610, 3)).astype(np.uint8)
    pipe = _pipeline([(1333, 200), (1333, 160)], True)
    text = detect_image(det, img, "P0042", 1, subsize=256, gap=64, batch=4, test_pipeline=pipe)
    assert calls == [(4, 4, True), (4, 2, True)]
    m = detect_image_tensors(det, img, 0, 1, subsize=256, gap=64, batch=4, test_pipeline=pipe)
    assert calls == [(4, 4, True), (4, 2, True)] * 2 and len(cache) == 2
    assert m.to_lines(["P0042"], DOTA_CLASSES) == text
    assert 0 < len(m) <= 6 * 60


@pytest.mark.parametrize("score_thr", [0.0, 0.05])
def test_production_size_nms_plan_is_covered(cuda, score_thr):
    """V = 4 views of B = 4 tiles at the 1024^2 and 960^2 level shapes: four times the candidates per (image, class) segment
    of simple_test.  The rotated NMS must take a plan test_nms_plans_gpu.py compares with the CPU oracle, without
    overflowing its candidate list; image 0 is compared with the eager merge"""
    from orientedreppoints_b200 import _lib
    B = 4
    shapes = [LEVELS_1024, LEVELS_1024, LEVELS_960, LEVELS_960]
    outs = [_view_outs(cuda, B, lv, seed=40 + v) for v, lv in enumerate(shapes)]
    cls, ref = [o[0] for o in outs], [o[1] for o in outs]
    metas = [_meta(1024, False, 1.0, B), _meta(1024, True, 1.0, B), _meta(960, False, 0.9375, B), _meta(960, True, 0.9375, B)]
    cfg = _cfg(score_thr)
    dets, labels, counts = _fused(cls, ref, metas, cfg, True)
    torch.cuda.synchronize()
    p = _lib.rnms_last_plan()
    sig = (p["lazy"], p["R"], p["no_sync"], p["flags_out"], p["union_mode"], p["order"], int(p["attempts"] > 1))
    print("plan", p, "counts", counts)
    assert sig in COVERED_PLANS, p
    per_img = sum(min(h * w, 2000) for lv in shapes for h, w in lv) * 15
    assert p["seg_limit"] == B * 15 and p["n"] == B * per_img
    assert min(counts) >= 0 and max(counts) == 2000
    one = _eager([[c[:1] for c in v] for v in cls], [[r[:1] for r in v] for v in ref], [m[:1] for m in metas], cfg, True)
    _assert_equal(dets[:1], labels[:1], counts[:1], one)
