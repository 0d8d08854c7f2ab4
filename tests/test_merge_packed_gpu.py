"""GPU: ResultMerge over the packed detection buffer (orp_result_merge, merge_packed, detect_image_tensors,
evaluate_merged) against the reference's mergesingle output, its numpy restatement, and the text path it replaces."""
import importlib.util
import json
import os
import sys

import numpy as np
import pytest
import torch

from orientedreppoints_b200 import _lib, gather
from orientedreppoints_b200.dota import evaluation as ev
from orientedreppoints_b200.dota import result_merge as rm
from orientedreppoints_b200.dota.pipeline import DOTA_CLASSES

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
from merge_packed_ref import merge_packed_ref, packed_rows  # noqa: E402

FIELDS = ("cls", "img", "score", "quad", "src_row", "cls_off")


@pytest.fixture(scope="module")
def fx():
    g = dict(np.load(os.path.join(HERE, "golden", "result_merge_packed.npz")))
    g.update(json.load(open(os.path.join(HERE, "golden", "result_merge_packed.json"))))
    return g


@pytest.fixture(scope="module")
def perf_merge():
    spec = importlib.util.spec_from_file_location("perf_merge", os.path.join(os.path.dirname(HERE), "tools", "perf_merge.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def host(m):
    return {k: getattr(m, k).cpu().numpy() for k in FIELDS}


def assert_same(a, b):
    for k in FIELDS:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, k
        assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k       # bit for bit


def meta_of(fx):
    return fx["tile_slot"], fx["tile_xy"], fx["tile_rate"], fx["tile_img"]


def one_tile(rows, cap, dev):
    """packed [1, cap + 1, 28] holding `rows` = [(quad8, score, label), ...]"""
    buf = np.zeros((1, cap + 1, 28), np.float32)
    for r, (q, s, l) in enumerate(rows):
        buf[0, r, 18:26], buf[0, r, 26], buf[0, r, 27] = q, s, l
    buf[0, cap, 0] = len(rows)
    return torch.from_numpy(buf).to(dev)


def square(x, y, s):
    return [x, y, x + s, y, x + s, y + s, x, y + s]


def test_fixture_lines_and_tensors(cuda, fx, po):
    packed = torch.from_numpy(fx["packed"]).to(cuda)
    m = rm.merge_packed(packed, *meta_of(fx), 3)
    assert m.to_lines(fx["images"], fx["classes"]) == fx["merged"]
    ref = merge_packed_ref(fx["packed"], *meta_of(fx), 3, 15, fx["nms_thresh"], nms=po.nms_poly_f64)
    assert_same(host(m), ref)
    plan = _lib.rnms_last_plan()
    assert plan["seg_limit"] == 15 * 3 and plan["order"] == _lib.ORP_ORDER_SCORE_DESC and plan["attempts"] == 1
    assert plan["lazy"] == 1 and plan["union_mode"] == _lib.ORP_UNION_NAN_SUPPRESSES and plan["n"] == sum(map(len, fx["lines"]))
    # the text path on the same lines
    for c, lines in zip(fx["classes"], fx["lines"]):
        assert rm.merge_lines(lines) == fx["merged"][c], c
    # the plain variant compares the zero-area boxes with each other; on this set it keeps the same rows
    mp = rm.merge_packed(packed, *meta_of(fx), 3, plain=True)
    assert_same(host(mp), merge_packed_ref(fx["packed"], *meta_of(fx), 3, 15, fx["nms_thresh"], plain=True, nms=po.nms_poly_f64))


def test_gathered_layout_equals_dataset_order(cuda, fx):
    """a [2, T, cap + 1, 28] buffer as two ranks' all-gather leaves it (tile i at rank i % 2, slot i // 2, the last slot
    of rank 1 the sampler's padding) merges to the dataset-order result through gather.dataset_slots"""
    n = fx["packed"].shape[0]
    assert n % 2 == 0
    order = fx["packed"][fx["tile_slot"]][:n - 1]                   # dataset order, an odd number of tiles
    t = n // 2
    world = np.zeros((2, t) + order.shape[1:], np.float32)
    for i in range(n - 1):
        world[i % 2, i // 2] = order[i]
    world[1, t - 1] = order[0]                                       # the padding tile repeats the first, as the sampler does
    xy, rate, img = fx["tile_xy"][:n - 1], fx["tile_rate"][:n - 1], fx["tile_img"][:n - 1]
    a = rm.merge_packed(torch.from_numpy(order).to(cuda), np.arange(n - 1), xy, rate, img, 3)
    b = rm.merge_packed(torch.from_numpy(world).to(cuda), gather.dataset_slots(2, t, n - 1), xy, rate, img, 3)
    assert len(a) > 100
    assert_same(host(a), host(b))
    # a negative slot skips its tile
    skip = np.arange(n - 1)
    skip[3] = -1
    keep = np.delete(np.arange(n - 1), 3)
    c = rm.merge_packed(torch.from_numpy(order).to(cuda), skip, xy, rate, img, 3)
    d = rm.merge_packed(torch.from_numpy(order[keep]).to(cuda), np.arange(n - 2), xy[keep], rate[keep], img[keep], 3)
    assert_same(host(c), host(d))


def _frozen(det):
    """Serve every result form of the detector from ONE run per batch.  GroupNorm sums use atomics, so two runs of the
    network may differ in the last bit, and the text path and the tensor path must consume the same detections to be
    compared string for string.  simple_test is run once per batch in its "padded" form - the (dets, labels, counts)
    tensors of the fused head, or the per-tile (dets, labels) list of the unfused one - and the list form the text path
    asks for is cut from that as simple_test itself cuts it (rows below the count, then rbbox2result); aug_test results
    are cached per tile.  So these tests compare the two compositions after the detector, not two detector runs."""
    from orientedreppoints_b200.core.transforms import rbbox2result
    real, real_aug, cache = det.simple_test, det.aug_test, {}

    def key(t):
        return tuple(t.shape), int(t.long().sum())

    def simple_test(img, img_metas=None, rescale=False, return_tensors=False, valid_hw=None):
        k = ("simple", key(img), bool(rescale))
        if k not in cache:
            cache[k] = real(img, img_metas, rescale, "padded", valid_hw)
        out = cache[k]
        if isinstance(out, tuple):
            if return_tensors == "padded":
                return out
            dets, labels, counts = out
            cnt = counts.tolist()
            assert min(cnt) >= 0
            out = [(dets[i, :cnt[i]], labels[i, :cnt[i]]) for i in range(len(cnt))]
        return out if return_tensors else [rbbox2result(d, l, 16) for d, l in out]

    def aug_test(imgs, img_metas, rescale=False, valid_hws=None):
        k = ("aug",) + tuple(key(v) for v in imgs)
        if k not in cache:
            cache[k] = real_aug(imgs, img_metas, rescale, valid_hws)
        return cache[k]
    det.simple_test, det.aug_test = simple_test, aug_test
    return det


def _detector(cuda, fused=True):
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    from orientedreppoints_b200.weights import random_state_dict
    d = OrientedRepPointsDetector(random_state_dict(50, seed=0, reference_init=True), 50, cuda, "bf16",
                                  test_cfg=dict(score_thr=0.0, max_per_img=60))
    d.fused_post = fused
    return _frozen(d)


@pytest.fixture(scope="module")
def det(cuda):
    return _detector(cuda)


def _image(seed, h=420, w=610):
    return np.random.RandomState(seed).randint(0, 256, size=(h, w, 3)).astype(np.uint8)


def _pipeline(flip):
    return [dict(type='LoadImageFromFile'),
            dict(type='MultiScaleFlipAug', img_scale=(1333, 200), flip=flip,
                 transforms=[dict(type='RotateResize', keep_ratio=True), dict(type='RotateRandomFlip'),
                             dict(type='Normalize', mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375], to_rgb=True),
                             dict(type='Pad', size_divisor=32), dict(type='ImageToTensor', keys=['img']),
                             dict(type='Collect', keys=['img'])])]


@pytest.mark.parametrize("pipeline,fused", [(None, True), (_pipeline(False), True), (_pipeline(True), True), (None, False)],
                         ids=["tiles", "test_pipeline", "flip_views_aug_test", "unfused_head"])
def test_detect_image_tensors_equals_detect_image(cuda, det, pipeline, fused):
    """the tensor composition against the text composition over the same detections (see _frozen): the padded output of
    the fused head, a one-view test pipeline, two views per tile through aug_test (per-class arrays repacked), and the
    unfused head, whose simple_test hands back a per-tile list"""
    from orientedreppoints_b200.dota.pipeline import detect_image, detect_image_tensors
    d = det if fused else _detector(cuda, fused=False)
    img = _image(11)
    text = detect_image(d, img, "P0042", 1, subsize=256, gap=64, batch=4, test_pipeline=pipeline)
    m = detect_image_tensors(d, img, 0, 1, subsize=256, gap=64, batch=4, test_pipeline=pipeline)
    assert m.to_lines(["P0042"], DOTA_CLASSES) == text
    assert 0 < len(m) <= 6 * 60 and m.quad.dtype == torch.float64 and m.quad.is_cuda


def test_all_gather_output_goes_into_the_merge(cuda, fx):
    """pack -> all_gather_detections(packed=True) (one rank: no process group needed) -> merge_packed equals the merge of
    the dataset-order buffer; the default (all_buf, all_counts) pair has no count rows and is not an input of the merge"""
    order = torch.from_numpy(fx["packed"][fx["tile_slot"]]).to(cuda)
    cap = order.shape[1] - 1
    dets, labels, counts = order[:, :cap, :27].contiguous(), order[:, :cap, 27].long(), order[:, cap, 0].int()
    buf, cnt = gather.pack(dets, labels, counts)
    assert torch.equal(buf, order)
    whole = gather.all_gather_detections(buf, cnt, packed=True)
    assert whole.shape == (1,) + tuple(order.shape)
    handle = gather.all_gather_detections(buf, cnt, async_op=True, packed=True)
    assert torch.equal(handle.wait(), whole)
    meta = (fx["tile_xy"], fx["tile_rate"], fx["tile_img"])
    n = order.shape[0]
    a = rm.merge_packed(order, np.arange(n), *meta, 3)
    b = rm.merge_packed(whole, gather.dataset_slots(1, n, n), *meta, 3)
    assert len(a) > 100
    assert_same(host(a), host(b))
    # the split pair: its buffer ends in a detection row.  Where that row holds a detection the merge refuses it
    all_buf, all_counts = gather.all_gather_detections(buf, cnt)
    assert all_buf.shape[2] == cap and torch.equal(all_counts[0], counts)
    full = all_buf.clone()
    full[0, 0, :, 18:26] = torch.tensor(square(5.0, 5.0, 20.0), device=cuda)
    with pytest.raises(_lib.OrpError, match="count"):
        rm.merge_packed(full, gather.dataset_slots(1, n, n), *meta, 3)
    # and a count row with anything after the count is not the packed layout
    stray = order.clone()
    stray[4, cap, 9] = 1.0
    with pytest.raises(_lib.OrpError, match="count"):
        rm.merge_packed(stray, np.arange(n), *meta, 3)


def _gts_from(lines_by_class, names, every=3):
    """ground truth cut from the detections themselves: every third merged box, moved a little, some marked difficult"""
    gts = {n: [] for n in names}
    k = 0
    for c, lines in lines_by_class.items():
        for line in lines[::every]:
            sp = line.split(' ')
            gts[sp[0]].append({'name': c, 'difficult': int(k % 7 == 0), 'bbox': [float(v) + 0.75 for v in sp[2:]]})
            k += 1
    return gts


def assert_same_eval(a, b):
    assert a['npos'] == b['npos'] and repr((a['map'], a['ap'])) == repr((b['map'], b['ap']))   # repr: an ap is NaN when npos is 0
    for f in ('rec', 'prec', 'order'):
        for c in DOTA_CLASSES:
            assert a[f][c].dtype == b[f][c].dtype and a[f][c].tobytes() == b[f][c].tobytes(), (f, c)   # bits: rec is NaN when npos is 0


def test_multi_image_merge_and_evaluation_equal_the_text_path(cuda, det):
    from orientedreppoints_b200.dota.pipeline import detect_image, detect_image_tensors, detect_images_tensors
    images = [("P0042", _image(11)), ("P0007", _image(12, 300, 700)), ("P0100", _image(13, 520, 256))]
    names = [n for n, _ in images]
    text = {c: [] for c in DOTA_CLASSES}
    singles = []
    for k, (n, im) in enumerate(images):
        for c, lines in detect_image(det, im, n, 1, subsize=256, gap=64, batch=16).items():
            text[c] += lines
        singles.append(detect_image_tensors(det, im, k, 1, subsize=256, gap=64, batch=16, nimg=3))
    m = detect_images_tensors(det, images, 1, subsize=256, gap=64, batch=16)
    assert m.to_lines(names, DOTA_CLASSES) == text
    # the multi-image call == the per-image calls concatenated class by class
    for c in range(15):
        sl = slice(int(m.cls_off[c]), int(m.cls_off[c + 1]))
        for f in ("img", "score", "quad"):
            parts = [getattr(s, f)[int(s.cls_off[c]):int(s.cls_off[c + 1])] for s in singles]
            assert torch.equal(getattr(m, f)[sl], torch.cat(parts)), (c, f)
    gts = _gts_from(text, names)
    gts["P9999"] = [{'name': 'plane', 'difficult': 0, 'bbox': [float(v) for v in square(10, 10, 20)]}]   # an image without detections
    gts = {k: gts[k] for k in ("P0007", "P9999", "P0100", "P0042")}                                       # another order than the merge's ids
    a, b = ev.evaluate_merged(m, gts, names), ev.evaluate(text, gts)
    assert_same_eval(a, b)
    assert 0 < a['map'] < 1 and sum(a['npos'].values()) > 20
    a, b = ev.evaluate_merged(m, gts, names, ovthresh=0.7, use_07_metric=False), ev.evaluate(text, gts, ovthresh=0.7, use_07_metric=False)
    assert_same_eval(a, b)
    with pytest.raises(KeyError, match="P0042"):                     # an image with detections must be in the image set
        ev.evaluate_merged(m, {k: gts[k] for k in ("P0007", "P0100")}, names)
    # one without detections need not be, as the text path only looks up the names on its lines
    a = ev.evaluate_merged(detect_images_tensors(det, images, 1, subsize=256, gap=64, batch=16, image_ids=[0, 1, 2], nimg=4),
                           gts, names + ["P5555"])
    assert_same_eval(a, ev.evaluate(text, gts))
    # two rates of one image share its id, as their tile names share the image name
    two = detect_images_tensors(det, images[:1], (1, 0.5), subsize=256, gap=64, batch=16)
    from orientedreppoints_b200.dota.pipeline import task1_lines
    from orientedreppoints_b200.dota.split_tiles import split_image
    per_class = [[] for _ in DOTA_CLASSES]
    for r in (1, 0.5):
        tiles, tnames, _ = split_image(images[0][1], "P0042", r, 256, 64, device=cuda)
        for c, lines in enumerate(task1_lines(det.simple_test(tiles), tnames)):
            per_class[c] += lines
    assert two.to_lines(["P0042"], DOTA_CLASSES) == {c: rm.merge_lines(l) for c, l in zip(DOTA_CLASSES, per_class)}


def test_empty_single_and_full_tiles(cuda):
    empty = torch.zeros((3, 9, 28), dtype=torch.float32, device=cuda)
    meta = (np.arange(3), np.zeros((3, 2), np.int32), np.ones(3), np.zeros(3, np.int32))
    m = rm.merge_packed(empty, *meta, 2)
    assert len(m) == 0 and m.cls_off.tolist() == [0] * 16 and m.quad.shape == (0, 8) and m.score.dtype == torch.float64
    assert m.to_lines(["a", "b"], DOTA_CLASSES) == {c: [] for c in DOTA_CLASSES}
    gts = {"a": [{'name': 'plane', 'difficult': 0, 'bbox': square(0, 0, 10)}], "b": []}
    res = ev.evaluate_merged(m, gts, ["a", "b"])
    assert res['map'] == 0.0 and all(v == 0.0 for v in res['ap'].values()) and res['npos']['plane'] == 1
    assert_same_eval(res, ev.evaluate({}, gts))
    # no tiles at all, and a bound of zero rows
    none = rm.merge_packed(empty, np.zeros(0, np.int32), np.zeros((0, 2), np.int32), np.zeros(0), np.zeros(0, np.int32), 2)
    assert len(none) == 0 and len(rm.merge_packed(empty, *meta, 2, max_rows=0)) == 0
    # a single detection, restored with its tile's origin and rate
    one = one_tile([(square(10.5, 20.25, 8), 0.625, 3)], 4, cuda)
    m = rm.merge_packed(one, [0], [[100, 200]], [0.5], [1], 2)
    assert host(m)["quad"].tolist() == [[(v + o) / 0.5 for v, o in zip(square(10.5, 20.25, 8), [100, 200] * 4)]]
    assert (m.cls.tolist(), m.img.tolist(), m.score.tolist(), m.src_row.tolist()) == ([3], [1], [0.625], [0])
    assert m.cls_off.tolist() == [0] * 4 + [1] * 12
    # a tile filled to cap: 3 stacks of duplicates over 16 rows, one survivor (the best) per stack and class
    rows = [(square(40.0 * (k % 3), 0, 30), 0.1 + 0.05 * k, k % 2) for k in range(16)]
    m = rm.merge_packed(one_tile(rows, 16, cuda), [0], [[0, 0]], [1.0], [0], 1)
    assert m.cls.tolist() == [0] * 3 + [1] * 3
    assert m.src_row.tolist() == [14, 12, 10, 15, 13, 11]            # score descending inside each class
    # rows whose label is no class are left out of the numbering
    rows = [(square(0, 0, 10), 0.9, 15), (square(0, 0, 10), 0.8, -1), (square(0, 0, 10), 0.7, 1.5), (square(50, 0, 10), 0.6, 14)]
    m = rm.merge_packed(one_tile(rows, 4, cuda), [0], [[0, 0]], [1.0], [0], 1)
    assert (m.cls.tolist(), m.src_row.tolist()) == ([14], [0])


def test_refused_input_is_an_error_not_an_empty_tile(cuda, fx):
    packed = torch.from_numpy(fx["packed"]).to(cuda)
    cap = packed.shape[1] - 1
    bad = packed.clone()
    bad[int(fx["tile_slot"][2]), cap, 0] = -1.0                      # orp_head_postprocess marks an NMS overflow so
    with pytest.raises(_lib.OrpError, match="count"):
        rm.merge_packed(bad, *meta_of(fx), 3)
    skipped = fx["tile_slot"].copy()
    skipped[2] = -1                                                  # the marked slot does no harm when it is not selected
    assert len(rm.merge_packed(bad, skipped, *meta_of(fx)[1:], 3)) > 0
    bad[int(fx["tile_slot"][2]), cap, 0] = cap + 1
    with pytest.raises(_lib.OrpError, match="count"):
        rm.merge_packed(bad, *meta_of(fx), 3)
    for k, v in ((2, np.where(np.arange(len(fx["tile_rate"])) == 4, 0.0, fx["tile_rate"])),
                 (3, np.where(np.arange(len(fx["tile_img"])) == 4, 3, fx["tile_img"])),
                 (0, np.where(np.arange(len(fx["tile_slot"])) == 4, packed.shape[0], fx["tile_slot"]))):
        meta = list(meta_of(fx))
        meta[k] = v
        with pytest.raises(_lib.OrpError, match="out of range"):
            rm.merge_packed(packed, *meta, 3)
    with pytest.raises(_lib.OrpError, match="max_rows"):
        rm.merge_packed(packed, *meta_of(fx), 3, max_rows=17)
    # a bound above the row total pads the NMS with rows that never reach the result
    rows = int(fx["packed"][:, cap, 0].sum())
    assert_same(host(rm.merge_packed(packed, *meta_of(fx), 3, max_rows=rows + 1000)), host(rm.merge_packed(packed, *meta_of(fx), 3)))


def test_plain_variant_on_separated_zero_area_boxes(cuda):
    """py_cpu_nms_poly compares every pair, so zero-area boxes suppress each other wherever they are; the fast variant
    only compares boxes whose hulls overlap and keeps them all"""
    pt = lambda x, y: [x, y] * 4   # noqa: E731
    rows = [(pt(10, 10), 0.9, 0), (pt(500, 500), 0.8, 0), (square(100, 100, 50), 0.7, 0), (pt(900, 20), 0.6, 0),
            (square(110, 110, 50), 0.5, 0), (pt(700, 700), 0.95, 1)]
    packed = one_tile(rows, 8, cuda)
    meta = ([0], [[0, 0]], [1.0], [0])
    fast, plain = rm.merge_packed(packed, *meta, 1), rm.merge_packed(packed, *meta, 1, plain=True)
    dets = np.array([q + [s] for q, s, l in rows if l == 0], np.float64)
    assert fast.src_row.tolist() == rm.py_cpu_nms_poly_fast(dets, 0.1) + [5] == [0, 1, 2, 3, 5]
    assert plain.src_row.tolist() == rm.py_cpu_nms_poly(dets, 0.1) + [5] == [0, 2, 5]


def test_non_finite_coordinates_are_kept_and_do_not_hang(cuda):
    """a row with a NaN or infinite coordinate is kept and suppresses nothing (what orp_rnms does with such a box), and the
    segment's origin comes from its finite coordinates only, so the other rows merge as if it were not there"""
    nan, inf = float("nan"), float("inf")
    good = [(square(3000, 3000, 40), 0.9, 0), (square(3002, 3001, 40), 0.8, 0), (square(3300, 3000, 40), 0.7, 0)]
    odd = [([nan] * 8, 0.99, 0), (square(3000, 3000, 40)[:7] + [inf], 0.95, 0), ([-inf] + square(3000, 3000, 40)[1:], 0.1, 0)]
    meta = ([0], [[0, 0]], [1.0], [0])
    m = rm.merge_packed(one_tile(odd[:2] + good + odd[2:], 8, cuda), *meta, 1)
    assert m.src_row.tolist() == [0, 1, 2, 4, 5]
    q = host(m)["quad"]
    assert np.isnan(q[0]).all() and q[1, 7] == inf and q[4, 0] == -inf
    ref = rm.merge_packed(one_tile(good, 8, cuda), *meta, 1)
    assert torch.equal(m.quad[2:4], ref.quad) and ref.src_row.tolist() == [0, 2]
    res = ev.evaluate_merged(m, {"a": [{'name': 'plane', 'difficult': 0, 'bbox': square(3000, 3000, 40)}]}, ["a"])
    assert res['npos']['plane'] == 1 and len(res['rec']['plane']) == 5


def test_validation_scale_set_against_per_class_segmented_nms(cuda, perf_merge):
    """~2 x 10^5 rows over 40 images of 25 tiles: the one call against the text path's own arithmetic without the text -
    15 calls of result_merge._nms_segmented on the same restored rows, survivors listed by first appearance"""
    packed, xy, rate, img, _ = perf_merge.synth_packed(40, 500, 6, 256, seed=3)
    slots = np.arange(packed.shape[0])
    m = rm.merge_packed(torch.from_numpy(packed).to(cuda), slots, xy, rate, img, 40)
    plan = _lib.rnms_last_plan()
    quad, score, cls, im = packed_rows(packed, slots, xy, rate, img, 40, 15)
    assert plan["n"] == quad.shape[0] > 150000 and plan["seg_limit"] == 600 and plan["attempts"] == 1
    rows, off = [], [0]
    for c in range(15):
        of_class = np.flatnonzero(cls == c)
        names, ids = np.unique(im[of_class], return_inverse=True)
        assert np.array_equal(names, np.sort(names)) and np.all(np.diff(im[of_class]) >= 0)   # first appearance == id order here
        keep = rm._nms_segmented(np.concatenate([quad[of_class], score[of_class, None]], 1), 0.1, segments=ids.astype(np.int32))
        for k in range(len(names)):
            rows.extend(of_class[keep[ids[keep] == k]].tolist())
        off.append(len(rows))
    got = host(m)
    assert got["cls_off"].tolist() == off and np.array_equal(got["src_row"], np.asarray(rows, np.int32))
    assert np.array_equal(got["quad"], quad[rows]) and np.array_equal(got["score"], score[rows])
    assert np.array_equal(got["cls"], cls[rows]) and np.array_equal(got["img"], im[rows])
    assert 0.2 * len(rows) < len(cls) - len(rows)                   # the merge suppressed a good share
