"""GPU: orp_dota_eval_aoe and orp_poly2rbox_v3 through orientedreppoints_b200.dota.aoe_evaluation / .poly2rbox against
the reference's own mAOE_evaluation.py and poly2rbox_single_v3 output (tests/golden/dota_aoe.json) and, at sizes no
golden file holds, against the numpy restatement (tests/aoe_ref.py)."""
import json
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
import aoe_ref  # noqa: E402
from test_dota_eval_gpu import CLASSES, _line, _quad, random_set  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "dota_aoe.json")
# 4 ulp of the atan2 result an angle comes from (|atan2| <= pi): norm_angle's shifts by pi/4 and pi keep its absolute error
ANGLE_TOL = 4 * np.spacing(np.pi)


@pytest.fixture(scope="module")
def gold():
    with open(GOLDEN) as f:
        g = json.load(f)
    with open(os.path.join(HERE, "golden", g["inputs"])) as f:
        g["case"] = json.load(f)
    return g


def _same_bits(a, b):
    """bit for bit, except that any NaN equals any NaN (the device's NaN and numpy's differ in sign and payload)"""
    a, b = np.atleast_1d(np.asarray(a, np.float64)), np.atleast_1d(np.asarray(b, np.float64))
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and a[~na].tobytes() == b[~nb].tobytes()


def check_sums(res, classes):
    """aoe == the host's left-to-right sum of the returned matched angle_dif over n, bit for bit; maoe likewise"""
    for c in classes:
        m = res['angle_dif'][c][~np.isnan(res['angle_dif'][c])]
        assert res['n'][c] == m.size, c
        assert _same_bits(res['aoe'][c], aoe_ref.running_mean(m.tolist())), c
    assert _same_bits(res['maoe'], aoe_ref.running_mean([res['aoe'][c] for c in classes]))


def check_against_restatement(dets, gts, classes=CLASSES, ovthresh=0.7):
    from orientedreppoints_b200.dota.aoe_evaluation import evaluate_aoe
    got = evaluate_aoe(dets, gts, classes, ovthresh)
    for c in classes:
        f = [l.strip().split(' ') for l in dets.get(c, ())]
        gt = {n: np.array([o['bbox'] for o in objs if o['name'] == c], np.float64).reshape(-1, 8) for n, objs in gts.items()}
        order, ad = aoe_ref.aoe_class([x[0] for x in f], np.array([float(x[1]) for x in f]),
                                      np.array([[float(v) for v in x[2:]] for x in f]).reshape(-1, 8), gt, ovthresh, "stable")
        assert np.array_equal(got['order'][c], order), c
        assert np.array_equal(np.isnan(got['angle_dif'][c]), np.isnan(ad)), c
        assert np.nanmax(np.abs(got['angle_dif'][c] - ad), initial=0.0) <= 1e-12, c
    check_sums(got, classes)
    return got


@pytest.mark.parametrize("thr", ["0.5", "0.7"])
def test_golden_reference_output(cuda, gold, thr):
    from orientedreppoints_b200.dota.aoe_evaluation import evaluate_aoe
    case = gold["case"]
    gts = {n: case["parse_gt"][n] for n in case["imagenames"]}
    res = evaluate_aoe(case["detections"], gts, gold["classnames"], float(thr))
    aoes = []
    for c in gold["classnames"]:
        want = np.array(gold["aoe_eval"][thr][c])
        sc = np.array([float(l.split(' ')[1]) for l in case["detections"][c]])
        assert np.array_equal(res['order'][c], np.argsort(-sc)), c                 # unique scores: the reference's order
        got = res['angle_dif'][c][~np.isnan(res['angle_dif'][c])]                  # matched ranks in rank order
        assert got.shape == want.shape and np.abs(got - want).max(initial=0.0) <= 1e-12, c
        aoes.append(aoe_ref.running_mean(want.tolist()))
        assert abs(res['aoe'][c] - aoes[-1]) <= 1e-12 * abs(aoes[-1]), c
    maoe = aoe_ref.running_mean(aoes)
    assert abs(res['maoe'] - maoe) <= 1e-12 * abs(maoe)
    check_sums(res, gold["classnames"])


def test_poly2rbox_v3_edge_set(cuda, gold):
    from orientedreppoints_b200.dota.poly2rbox import poly2rbox_single_v3, poly2rbox_v3
    e = gold["edge"]
    out = poly2rbox_v3(torch.tensor(e["quad"], dtype=torch.float64, device=cuda)).cpu().numpy()
    want = np.array(e["rbox"], np.float64)
    assert _same_bits(out[:, :4], want[:, :4])                                  # centres and sizes bit for bit
    for k, (kind, q) in enumerate(zip(e["kind"], e["quad"])):
        ref = aoe_ref.poly2rbox_v3(q)                                               # numpy's decisions, exact in the band
        a, r = out[k, 4], ref[4]
        assert (np.isnan(a) and np.isnan(r)) or abs(a - r) <= ANGLE_TOL, (kind, q, a, r)
        if not np.isnan(want[k, 4]) and abs(want[k, 4] - r) > ANGLE_TOL:
            assert kind in ("diamond", "rhombus", "mirror")                         # an exact tie the reference rounded
        elif not np.isnan(r):
            assert abs(a - want[k, 4]) <= ANGLE_TOL, (kind, q)
    assert poly2rbox_single_v3(e["quad"][0]) == tuple(float(v) for v in out[0])
    assert poly2rbox_v3(np.zeros((0, 8))).shape == (0, 5)


@pytest.mark.parametrize("seed,n_img,n_obj", [(0, 24, 30), (1, 40, 12)])
def test_random_sets_against_restatement(cuda, seed, n_img, n_obj):
    gts, dets = random_set(seed, n_img, n_obj)
    assert sum(len(v) for v in dets.values()) > 1000
    got = check_against_restatement(dets, gts)
    assert sum(got['n'].values()) > 100
    check_against_restatement(dets, gts, ovthresh=0.5)


def test_launch_edges(cuda):
    rng = np.random.RandomState(3)
    # one (class, image) bucket with 300 ground-truth boxes (more than two stages of 128), 700 detections of one class
    # (more than two CTAs of 256), all of them near a box
    grid = [(x, y) for x in range(20) for y in range(15)]
    objs = [{'name': 'plane', 'difficult': int(k % 17 == 0), 'bbox': _quad(50 + 150 * x, 50 + 150 * y, 100, 60, 0.2)}
            for k, (x, y) in enumerate(grid)]
    lines = []
    for k, s in zip(rng.randint(0, len(grid), 700), rng.permutation(700) / 700.0):
        x, y = grid[k]
        lines.append(_line("BIG", s, _quad(50 + 150 * x + rng.normal(0, 3), 50 + 150 * y + rng.normal(0, 3), 100, 60,
                                           0.2 + rng.normal(0, 0.05))))
    gts = {"BIG": objs, "ONE": [{'name': 'ship', 'difficult': 0, 'bbox': _quad(300, 300, 80, 40, 1.0)}],
           "EMPTY": [{'name': 'bridge', 'difficult': 0, 'bbox': _quad(10, 10, 5, 5, 0.0)}]}
    dets = {'plane': lines, 'ship': [_line("ONE", 0.5, _quad(301, 300, 80, 40, 1.02))],
            'harbor': [_line("BIG", 0.7, _quad(60, 60, 90, 50, 0.2))]}                # no ground truth of the class
    got = check_against_restatement(dets, gts)
    assert got['n']['plane'] > 500 and got['n']['ship'] == 1
    for c in ('bridge', 'harbor', 'tennis-court'):                                 # no detections / no ground truth
        assert got['n'][c] == 0 and np.isnan(got['aoe'][c]), c
    assert np.isnan(got['maoe'])


@pytest.mark.parametrize("nd", [1, 255, 256, 257, 511, 512, 513])
def test_detection_counts_around_the_block_size(cuda, nd):
    gts, dets = random_set(100 + nd, 10, 25, classes=CLASSES[:3], dup=4, n_fp=30)
    flat = [(c, l) for c in CLASSES[:3] for l in dets[c]]
    assert len(flat) >= nd
    keep = set(np.random.RandomState(nd).choice(len(flat), nd, replace=False).tolist())
    sub = {c: [l for k, (cc, l) in enumerate(flat) if cc == c and k in keep] for c in CLASSES[:3]}
    check_against_restatement(sub, gts, classes=CLASSES[:3], ovthresh=0.5)


def test_nothing_to_match(cuda):
    from orientedreppoints_b200.dota.aoe_evaluation import evaluate_aoe
    gts, dets = random_set(5, 3, 10, classes=CLASSES[:2])
    none = evaluate_aoe({}, gts, CLASSES[:2])                                       # nd = 0
    nogt = evaluate_aoe(dets, {n: [] for n in gts}, CLASSES[:2])                    # ng = 0
    for res in (none, nogt):
        assert all(res['n'][c] == 0 and np.isnan(res['aoe'][c]) for c in CLASSES[:2]) and np.isnan(res['maoe'])
    assert none['angle_dif']['plane'].size == 0
    assert nogt['angle_dif']['plane'].size == len(dets['plane']) > 0 and np.isnan(nogt['angle_dif']['plane']).all()


def test_two_calls_give_identical_bits(cuda):
    from orientedreppoints_b200.dota.aoe_evaluation import evaluate_aoe
    gts, dets = random_set(9, 30, 20)
    a, b = evaluate_aoe(dets, gts), evaluate_aoe(dets, gts)
    for f in ('angle_dif', 'order', 'aoe'):
        for c in CLASSES:
            assert np.asarray(a[f][c]).tobytes() == np.asarray(b[f][c]).tobytes(), (f, c)
    assert np.float64(a['maoe']).tobytes() == np.float64(b['maoe']).tobytes()


def test_merged_detections_equal_their_lines(cuda):
    from orientedreppoints_b200.dota import result_merge as rm
    from orientedreppoints_b200.dota.aoe_evaluation import evaluate_aoe, evaluate_aoe_merged
    from orientedreppoints_b200.dota.pipeline import DOTA_CLASSES
    fx = dict(np.load(os.path.join(HERE, "golden", "result_merge_packed.npz")))
    fx.update(json.load(open(os.path.join(HERE, "golden", "result_merge_packed.json"))))
    m = rm.merge_packed(torch.from_numpy(fx["packed"]).to(cuda), fx["tile_slot"], fx["tile_xy"], fx["tile_rate"],
                        fx["tile_img"], 3)
    names = list(fx["images"])
    text = m.to_lines(names, DOTA_CLASSES)
    rng = np.random.RandomState(1)
    gts = {n: [] for n in names}
    for c, lines in text.items():
        for line in lines[::2]:
            sp = line.split(' ')
            gts[sp[0]].append({'name': c, 'difficult': int(rng.rand() < 0.2),
                               'bbox': [float(v) + rng.normal(0, 0.5) for v in sp[2:]]})
    gts["P9999"] = []                                                                # an image without detections
    gts = dict(reversed(list(gts.items())))                                          # another order than the merge's ids
    for thr in (0.5, 0.7):
        a, b = evaluate_aoe_merged(m, gts, names, ovthresh=thr), evaluate_aoe(text, gts, ovthresh=thr)
        assert repr(a['maoe']) == repr(b['maoe']) and a['n'] == b['n'] and repr(a['aoe']) == repr(b['aoe'])
        for f in ('angle_dif', 'order'):
            for c in DOTA_CLASSES:
                assert a[f][c].dtype == b[f][c].dtype and a[f][c].tobytes() == b[f][c].tobytes(), (f, c)
    assert sum(a['n'].values()) > 10
    with pytest.raises(KeyError):
        evaluate_aoe_merged(m, {n: v for n, v in gts.items() if n != names[0]}, names)


def test_file_based_aoe_eval_equals_evaluate_aoe(cuda, tmp_path):
    from orientedreppoints_b200.dota.aoe_evaluation import aoe_eval, evaluate_aoe, main
    gts, dets = random_set(11, 8, 20)
    for name, objs in gts.items():
        text = "imagesource:GoogleEarth\ngsd:0.3\n" + "".join(
            " ".join(repr(v) for v in o['bbox']) + " " + o['name'] + " %d\n" % o['difficult'] for o in objs)
        (tmp_path / ("%s.txt" % name)).write_text(text)
    (tmp_path / "set.txt").write_text("\n".join(gts) + "\n")
    for c in CLASSES:
        (tmp_path / ("Task1_%s.txt" % c)).write_text("".join(l + "\n" for l in dets[c]))
    args = [str(tmp_path / "Task1_{:s}.txt"), str(tmp_path / "{:s}.txt"), str(tmp_path / "set.txt")]
    for thr in (0.5, 0.7):
        res = evaluate_aoe(dets, gts, CLASSES, thr)
        for c in CLASSES:
            lst = aoe_eval(*args, c, thr)
            m = res['angle_dif'][c][~np.isnan(res['angle_dif'][c])]
            assert isinstance(lst, list) and _same_bits(lst, m), c
    main(args)
