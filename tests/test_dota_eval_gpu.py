"""GPU: orp_dota_eval_task1 through orientedreppoints_b200.dota.evaluation against the reference's own
dota_evaluation_task1.py output (tests/golden/dota_eval.json) and, at sizes no golden file holds, against the oracle
restatement of voc_eval's matching loop (oracle/dota_eval_oracle.py, IoU from the reference's compiled polyiou or its C
port)."""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dota_eval.json")
CLASSES = ('plane', 'baseball-diamond', 'bridge', 'ground-track-field', 'small-vehicle', 'large-vehicle', 'ship',
           'tennis-court', 'basketball-court', 'storage-tank', 'soccer-ball-field', 'roundabout', 'harbor',
           'swimming-pool', 'helicopter')


def _same(a, b):
    return np.array_equal(np.asarray(a, np.float64), np.asarray(b, np.float64), equal_nan=True)


def _quad(cx, cy, w, h, a):
    c, s = np.cos(a), np.sin(a)
    return [float(v) for px, py in ((-w / 2, -h / 2), (w / 2, -h / 2), (w / 2, h / 2), (-w / 2, h / 2))
            for v in (cx + c * px - s * py, cy + s * px + c * py)]


def _line(img, score, q):
    return "%s %r %s" % (img, float(score), " ".join(repr(float(v)) for v in q))


def random_set(seed, n_img, n_obj, classes=CLASSES, dup=3, n_fp=10, extent=4000.0, equal_scores=False):
    """(gts {image: parse_gt objects}, dets {class: Task1 lines}): rotated objects, jittered copies spanning IoU ~0.3-0.9,
    duplicates and random false positives; unique scores unless equal_scores (then rounded to 0.1)"""
    rng = np.random.RandomState(seed)
    gts, dets = {}, {c: [] for c in classes}
    for k in range(n_img):
        name = "I%04d" % k
        objs = []
        for _ in range(n_obj):
            c = classes[rng.randint(len(classes))]
            w, h, a = rng.uniform(10, 200), rng.uniform(8, 120), rng.uniform(-np.pi, np.pi)
            cx, cy = rng.uniform(0, extent), rng.uniform(0, extent)
            objs.append({'name': c, 'difficult': int(rng.rand() < 0.1), 'bbox': _quad(cx, cy, w, h, a)})
            for _ in range(rng.randint(0, dup + 1)):
                j = rng.uniform(0.0, 0.4)
                dets[c].append((name, _quad(cx + rng.normal(0, j * w / 3), cy + rng.normal(0, j * h / 3),
                                            w * (1 + rng.normal(0, j / 3)), h * (1 + rng.normal(0, j / 3)), a + rng.normal(0, j))))
        for _ in range(n_fp):
            dets[classes[rng.randint(len(classes))]].append(
                (name, _quad(rng.uniform(0, extent), rng.uniform(0, extent), rng.uniform(10, 200), rng.uniform(8, 120), 0.3)))
        gts[name] = objs
    out = {}
    for c in classes:
        n = len(dets[c])
        sc = np.round(rng.uniform(0, 1, n), 1) if equal_scores else rng.permutation(n) / max(n, 1) + 1e-3
        out[c] = [_line(img, s, q) for (img, q), s in zip(dets[c], sc)]
    return gts, out


def oracle(dets, gts, classes, m07, kind="quicksort"):
    from oracle import dota_eval_oracle as orc
    res = {}
    for c in classes:
        gt = {}
        for name, objs in gts.items():
            sel = [o for o in objs if o['name'] == c]
            gt[name] = (np.array([o['bbox'] for o in sel], np.float64).reshape(-1, 8),
                        np.array([o['difficult'] for o in sel], np.int64).astype(bool))
        f = [l.strip().split(' ') for l in dets.get(c, ())]
        ids = [x[0] for x in f]
        sc = np.array([float(x[1]) for x in f])
        q = np.array([[float(v) for v in x[2:]] for x in f]).reshape(-1, 8)
        if not f:
            npos = sum(int((~g[1]).sum()) for g in gt.values())
            res[c] = (np.zeros(0, np.int64), np.zeros(0), np.zeros(0), orc.voc_ap(np.zeros(0), np.zeros(0), m07), npos)
            continue
        order, rec, prec, ap = orc.eval_class(ids, sc, q, gt, 0.5, m07, kind)
        res[c] = (order, rec, prec, ap, sum(int((~g[1]).sum()) for g in gt.values()))
    return res


def check_against_oracle(dets, gts, classes=CLASSES, kind="quicksort", check_order=False):
    from orientedreppoints_b200.dota.evaluation import evaluate
    for m07 in (True, False):
        got = evaluate(dets, gts, classes, 0.5, m07)
        want = oracle(dets, gts, classes, m07, kind)
        for c in classes:
            order, rec, prec, ap, npos = want[c]
            assert got['npos'][c] == npos, c
            assert _same(got['rec'][c], rec) and _same(got['prec'][c], prec), (c, m07)
            if m07:
                assert _same(got['ap'][c], ap), (c, got['ap'][c], ap)
            else:
                assert (np.isnan(ap) and np.isnan(got['ap'][c])) or abs(got['ap'][c] - ap) <= 1e-12, (c, got['ap'][c], ap)
            if check_order:
                assert np.array_equal(got['order'][c], order), c
        total = 0
        for c in classes:                      # main()'s running sum (Python's sum() compensates since 3.12)
            total = total + got['ap'][c]
        assert _same(got['map'], total / len(classes))
    return got


def test_golden_reference_output(cuda):
    from orientedreppoints_b200.dota.evaluation import evaluate
    with open(GOLDEN) as f:
        g = json.load(f)
    gts = {n: g["parse_gt"][n] for n in g["imagenames"]}
    for key, m07 in (("07", True), ("area", False)):
        res = evaluate(g["detections"], gts, g["classnames"], g["ovthresh"], m07)
        for c in g["classnames"]:
            r = g["results"][key][c]
            assert _same(res['rec'][c], r["rec"]) and _same(res['prec'][c], r["prec"]), (key, c)
            if m07:
                assert _same(res['ap'][c], r["ap"]), (key, c)
            else:
                assert (np.isnan(r["ap"]) and np.isnan(res['ap'][c])) or abs(res['ap'][c] - r["ap"]) <= 1e-12, (key, c)


@pytest.mark.parametrize("seed,n_img,n_obj", [(0, 24, 30), (1, 40, 12)])
def test_random_sets_against_oracle(cuda, seed, n_img, n_obj):
    gts, dets = random_set(seed, n_img, n_obj)
    assert sum(len(v) for v in dets.values()) > 1000
    check_against_oracle(dets, gts, check_order=True)


def test_equal_scores_are_taken_in_input_order(cuda):
    gts, dets = random_set(7, 20, 25, equal_scores=True)
    check_against_oracle(dets, gts, kind="stable", check_order=True)


def test_launch_edges(cuda):
    rng = np.random.RandomState(3)
    # one (class, image) bucket with 300 ground-truth boxes (more than two shared-memory stages of 128); detections
    # on boxes in every stage, 700 of them in one class (more than two CTAs of 256)
    grid = [(x, y) for x in range(20) for y in range(15)]
    objs = [{'name': 'plane', 'difficult': int(k % 17 == 0), 'bbox': _quad(50 + 150 * x, 50 + 150 * y, 100, 60, 0.2)}
            for k, (x, y) in enumerate(grid)]
    lines = []
    for k, s in zip(rng.randint(0, len(grid), 700), rng.permutation(700) / 700.0):
        x, y = grid[k]
        lines.append(_line("BIG", s, _quad(50 + 150 * x + rng.normal(0, 8), 50 + 150 * y + rng.normal(0, 8), 100, 60, 0.2)))
    gts = {"BIG": objs, "ONE": [{'name': 'ship', 'difficult': 0, 'bbox': _quad(300, 300, 80, 40, 1.0)}],
           "EMPTY": [{'name': 'bridge', 'difficult': 0, 'bbox': _quad(10, 10, 5, 5, 0.0)}]}
    dets = {'plane': lines,
            'ship': [_line("ONE", 0.5, _quad(302, 301, 80, 40, 1.0))],                   # a single-detection bucket
            'harbor': [_line("BIG", 0.7, _quad(60, 60, 90, 50, 0.2))]}                  # no ground truth of the class
    # bridge: ground truth, no detections
    got = check_against_oracle(dets, gts, check_order=True)
    assert got['rec']['bridge'].size == 0 and got['ap']['bridge'] == 0.0 and got['npos']['bridge'] == 1
    assert got['npos']['harbor'] == 0 and len(got['rec']['harbor']) == 1


@pytest.mark.parametrize("nd", [1, 255, 256, 257, 511, 512, 513])
def test_detection_counts_around_the_block_size(cuda, nd):
    gts, dets = random_set(100 + nd, 10, 25, classes=CLASSES[:3], dup=4, n_fp=30)
    flat = [(c, l) for c in CLASSES[:3] for l in dets[c]]
    assert len(flat) >= nd
    keep = set(np.random.RandomState(nd).choice(len(flat), nd, replace=False).tolist())
    sub = {c: [l for k, (cc, l) in enumerate(flat) if cc == c and k in keep] for c in CLASSES[:3]}
    check_against_oracle(sub, gts, classes=CLASSES[:3], check_order=True)


def test_file_based_voc_eval_equals_evaluate(cuda, tmp_path):
    from orientedreppoints_b200.dota.evaluation import evaluate, voc_eval
    gts, dets = random_set(11, 8, 20)
    for name, objs in gts.items():
        text = "imagesource:GoogleEarth\ngsd:0.3\n" + "".join(
            " ".join(repr(v) for v in o['bbox']) + " " + o['name'] + " %d\n" % o['difficult'] for o in objs)
        (tmp_path / ("%s.txt" % name)).write_text(text)
    (tmp_path / "set.txt").write_text("\n".join(gts) + "\n")
    for c in CLASSES:
        (tmp_path / ("Task1_%s.txt" % c)).write_text("".join(l + "\n" for l in dets[c]))
    for m07 in (True, False):
        res = evaluate(dets, gts, CLASSES, 0.5, m07)
        for c in CLASSES:
            rec, prec, ap = voc_eval(str(tmp_path / "Task1_{:s}.txt"), str(tmp_path / "{:s}.txt"), str(tmp_path / "set.txt"),
                                     c, 0.5, m07)
            assert _same(rec, res['rec'][c]) and _same(prec, res['prec'][c]) and _same(ap, res['ap'][c]), c


def test_detect_image_then_evaluate_equals_oracle(cuda):
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    from orientedreppoints_b200.dota.pipeline import DOTA_CLASSES, detect_image
    from orientedreppoints_b200.weights import random_state_dict
    det = OrientedRepPointsDetector(random_state_dict(50, seed=0, reference_init=True), 50, cuda, "bf16",
                                    test_cfg=dict(score_thr=0.0, max_per_img=60))
    img = np.random.RandomState(11).randint(0, 256, size=(420, 610, 3)).astype(np.uint8)
    merged = detect_image(det, img, "P0042", 1, subsize=256, gap=64, batch=16)
    n = sum(len(v) for v in merged.values())
    assert n > 20
    # ground truth: jittered copies of about half the detections, some difficult
    rng = np.random.RandomState(5)
    objs = []
    for c, lines in merged.items():
        for l in lines:
            if rng.rand() < 0.5:
                q = np.array([float(v) for v in l.split(' ')[2:]]) + rng.normal(0, 2.0, 8)
                objs.append({'name': c, 'difficult': int(rng.rand() < 0.1), 'bbox': [float(v) for v in q]})
    check_against_oracle(merged, {"P0042": objs}, classes=DOTA_CLASSES, kind="stable")
