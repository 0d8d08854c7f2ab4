"""CPU: the host side of the DOTA Task1 evaluation (orientedreppoints_b200/dota/evaluation.py) and the oracle
restatement of voc_eval's matching loop (oracle/dota_eval_oracle.py) against tests/golden/dota_eval.json, the output of
the reference's own dota_evaluation_task1.py (tests/golden/gen_golden_dota_eval.py)."""
import json
import os

import numpy as np
import pytest

from orientedreppoints_b200.dota import evaluation as ev

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dota_eval.json")


@pytest.fixture(scope="module")
def gold():
    with open(GOLDEN) as f:
        return json.load(f)


def _write_labels(gold, d):
    for name, text in gold["labels"].items():
        (d / ("%s.txt" % name)).write_text(text)


def _same(a, b):
    return np.array_equal(np.asarray(a, np.float64), np.asarray(b, np.float64), equal_nan=True)


def test_parse_gt_matches_reference(gold, tmp_path):
    _write_labels(gold, tmp_path)
    for name in gold["imagenames"]:
        assert ev.parse_gt(str(tmp_path / ("%s.txt" % name))) == gold["parse_gt"][name], name


def test_voc_ap_matches_reference(gold):
    for key, m07 in (("07", True), ("area", False)):
        for c, r in gold["results"][key].items():
            assert _same(ev.voc_ap(np.array(r["rec"]), np.array(r["prec"]), m07), r["ap"]), (key, c)
    # the empty curve of a class without detections
    assert ev.voc_ap(np.zeros(0), np.zeros(0), True) == 0.0 and ev.voc_ap(np.zeros(0), np.zeros(0), False) == 0.0


def test_thresholds_are_numpys():
    assert ev.THRESHOLDS_07.shape == (11,) and ev.THRESHOLDS_07[3] == 0.30000000000000004


def _gt_arrays(gold, cname):
    gt = {}
    for name in gold["imagenames"]:
        objs = [o for o in gold["parse_gt"][name] if o["name"] == cname]
        gt[name] = (np.array([o["bbox"] for o in objs], np.float64).reshape(-1, 8),
                    np.array([o["difficult"] for o in objs]).astype(bool))
    return gt


def _det_arrays(lines):
    f = [l.split(' ') for l in lines]
    return [x[0] for x in f], np.array([float(x[1]) for x in f]), np.array([[float(v) for v in x[2:]] for x in f])


@pytest.mark.parametrize("key,m07", [("07", True), ("area", False)])
def test_oracle_restatement_matches_reference(gold, key, m07):
    from oracle import dota_eval_oracle as orc
    for c in gold["classnames"]:
        ids, sc, q = _det_arrays(gold["detections"][c])
        _, rec, prec, ap = orc.eval_class(ids, sc, q, _gt_arrays(gold, c), gold["ovthresh"], m07)
        r = gold["results"][key][c]
        assert _same(rec, r["rec"]) and _same(prec, r["prec"]) and _same(ap, r["ap"]), (key, c)


def test_golden_covers_the_edge_cases(gold):
    from oracle import dota_eval_oracle as orc
    # helicopter: ground truth only difficult (npos 0), rec = 0 / 0
    assert np.isnan(gold["results"]["07"]["helicopter"]["rec"]).all()
    # the zero-area ship gives a NaN candidate: its detection is a false positive
    ids, sc, q = _det_arrays(gold["detections"]["ship"])
    order, tp, fp = orc.match(ids, sc, q, _gt_arrays(gold, "ship"))
    zero = [k for k, d in enumerate(order) if q[d][0] == 500.25][0]
    assert fp[zero] == 1 and tp[zero] == 0
    # plane: the second detection on the first object is a false positive although a free object is above 0.5
    ids, sc, q = _det_arrays(gold["detections"]["plane"])
    order, tp, fp = orc.match(ids, sc, q, _gt_arrays(gold, "plane"))
    at = {float(sc[d]): k for k, d in enumerate(order)}
    assert (tp[at[0.99]], fp[at[0.99]], tp[at[0.98]], fp[at[0.98]]) == (1, 0, 0, 1)
    assert orc._iou_rows(np.array([[110, 100, 210, 100, 210, 200, 110, 200.]]), q[order[at[0.98]]])[0] > 0.5
    # two hits on difficult objects count as neither
    assert all(tp[at[s]] == 0 and fp[at[s]] == 0 for s in (0.97, 0.96, 0.5))


def test_image_outside_the_image_set_is_a_key_error(tmp_path):
    (tmp_path / "A.txt").write_text("imagesource:x\ngsd:1\n0 0 10 0 10 10 0 10 plane 0\n")
    (tmp_path / "set.txt").write_text("A\n")
    (tmp_path / "Task1_plane.txt").write_text("A 0.9 0 0 10 0 10 10 0 10\nB 0.8 0 0 10 0 10 10 0 10\n")
    with pytest.raises(KeyError):
        ev.voc_eval(str(tmp_path / "Task1_{:s}.txt"), str(tmp_path / "{:s}.txt"), str(tmp_path / "set.txt"), "plane")
    with pytest.raises(FileNotFoundError):
        ev.voc_eval(str(tmp_path / "Task1_{:s}.txt"), str(tmp_path / "{:s}.txt"), str(tmp_path / "set.txt"), "ship")
