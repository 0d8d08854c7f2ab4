"""CPU: the mAOE restatement (tests/aoe_ref.py) against tests/golden/dota_aoe.json, the output of the reference's own
mAOE_evaluation.py and poly2rbox_single_v3 (tests/golden/gen_golden_dota_aoe.py), and the argument checks of
orp_dota_eval_aoe / orp_poly2rbox_v3, which need no GPU."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import aoe_ref
from orientedreppoints_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "dota_aoe.json")
TIE_KINDS = ("diamond", "rhombus", "mirror")   # |angle1| == |angle2| exactly wherever the ratio branch compares them
Q = np.pi / 4
# 4 ulp of the atan2 result an angle comes from (|atan2| <= pi): norm_angle's shifts by pi/4 and pi keep its absolute error
ANGLE_TOL = 4 * np.spacing(np.pi)


@pytest.fixture(scope="module")
def gold():
    with open(GOLDEN) as f:
        g = json.load(f)
    with open(os.path.join(HERE, "golden", g["inputs"])) as f:
        g["case"] = json.load(f)
    return g


def class_inputs(case, c):
    """(image ids, scores, quads, {image: every box of class c}) of the golden case"""
    f = [l.split(' ') for l in case["detections"][c]]
    gt = {n: np.array([o["bbox"] for o in case["parse_gt"][n] if o["name"] == c], np.float64).reshape(-1, 8)
          for n in case["imagenames"]}
    return [x[0] for x in f], np.array([float(x[1]) for x in f]), np.array([[float(v) for v in x[2:]] for x in f]), gt


def _same(a, b):
    return np.array_equal(np.asarray(a, np.float64), np.asarray(b, np.float64), equal_nan=True)


@pytest.mark.parametrize("thr", ["0.5", "0.7"])
def test_restatement_reproduces_aoe_eval(gold, thr):
    for c in gold["classnames"]:
        _, ad = aoe_ref.aoe_class(*class_inputs(gold["case"], c), ovthresh=float(thr))
        want = np.array(gold["aoe_eval"][thr][c])
        got = ad[~np.isnan(ad)]
        assert got.shape == want.shape, (thr, c)
        assert np.abs(got - want).max(initial=0.0) <= 1e-12, (thr, c)
    assert any(len(v) for v in gold["aoe_eval"][thr].values())


def test_restatement_reproduces_poly2rbox_single_v3(gold):
    """centres and sizes bit for bit; angles within ANGLE_TOL of the reference's host, except exact ties that the
    reference's rounding sends to edge 1->4 (the restatement, like the kernel, decides those exactly)"""
    e = gold["edge"]
    flipped = 0
    for kind, q, want in zip(e["kind"], e["quad"], e["rbox"]):
        got = aoe_ref.poly2rbox_v3(q)
        assert _same(got[:4], want[:4]), (kind, q)
        if np.isnan(want[4]):
            assert np.isnan(got[4]), (kind, q)
        elif abs(got[4] - want[4]) > ANGLE_TOL:
            assert kind in TIE_KINDS and abs(got[4] + want[4]) <= 1e-12, (kind, q, got, want)   # the mirrored edge
            flipped += 1
    assert flipped <= 4


def test_ties_and_wraps_follow_exact_arithmetic(gold):
    """host-independent facts of the edge set: an exact tie takes edge 1->2; a direction on an axis or a diagonal gives
    a multiple of pi/4 exactly, the 3pi/4 direction wrapped to -pi/4"""
    e = gold["edge"]
    for kind, q in zip(e["kind"], e["quad"]):
        r = aoe_ref.poly2rbox_v3(q)
        if kind in TIE_KINDS:
            assert r[5] == 1, (kind, q)
        if kind in ("axis", "diag", "square", "diamond"):
            assert r[4] / Q in (-1.0, 0.0, 1.0, 2.0), (kind, q, r)
        if kind == "diag" and (q[2] - q[0]) == -(q[3] - q[1]) and q[2] < q[0] and r[5] == 1:
            assert r[4] == -Q                                        # the 3pi/4 edge
    kinds = set(e["kind"])
    assert {"axis", "diag", "square", "diamond", "rhombus", "ratio", "degenerate", "nan", "decimal", "mirror"} <= kinds


def test_ratio_rows_straddle_the_threshold(gold):
    """float32(1.15) and its neighbours: below it the smaller |angle| wins (0), at and above it the longer edge (pi/2)"""
    e = gold["edge"]
    rows = [(q, r) for k, q, r in zip(e["kind"], e["quad"], e["rbox"]) if k == "ratio"]
    assert [r[4] / Q for _, r in rows] == [0.0, 0.0, 2.0, 0.0, 2.0, 0.0]


def _aoe_call(**kw):
    a = dict(det_cls=256, det_img=256, det_score=256, det_quad=256, nd=4, gt_cls=256, gt_img=256, gt_quad=256, ng=3, ncls=15,
             nimg=2, ovthresh=0.7, cls_off=256, order=256, angle_dif=256, count=256, aoe=256)
    a.update(kw)
    vp = lambda v: ctypes.c_void_p(v)   # noqa: E731  (256: a non-NULL placeholder that a refused call never reads)
    return _lib.lib().orp_dota_eval_aoe(vp(a["det_cls"]), vp(a["det_img"]), vp(a["det_score"]), vp(a["det_quad"]), a["nd"],
                                        vp(a["gt_cls"]), vp(a["gt_img"]), vp(a["gt_quad"]), a["ng"], a["ncls"], a["nimg"],
                                        a["ovthresh"], vp(a["cls_off"]), vp(a["order"]), vp(a["angle_dif"]), vp(a["count"]),
                                        vp(a["aoe"]), None)


@pytest.mark.parametrize("bad", [dict(nd=-1), dict(ng=-1), dict(ncls=-1), dict(nimg=-1), dict(ncls=1 << 16, nimg=1 << 16),
                                 dict(det_cls=0), dict(det_img=0), dict(det_score=0), dict(det_quad=0), dict(order=0),
                                 dict(angle_dif=0), dict(gt_cls=0), dict(gt_img=0), dict(gt_quad=0), dict(cls_off=0),
                                 dict(count=0), dict(aoe=0)])
def test_eval_aoe_refuses_bad_arguments_before_any_cuda_call(bad):
    assert _aoe_call(**bad) == -1
    assert b"orp_dota_eval_aoe" in _lib.lib().orp_last_error()


@pytest.mark.parametrize("n,quad,out", [(-1, 256, 256), (3, 0, 256), (3, 256, 0)])
def test_poly2rbox_v3_refuses_bad_arguments(n, quad, out):
    assert _lib.lib().orp_poly2rbox_v3(ctypes.c_void_p(quad), n, ctypes.c_void_p(out), None) == -1
    assert b"orp_poly2rbox_v3" in _lib.lib().orp_last_error()


def test_poly2rbox_v3_of_nothing_needs_no_device():
    assert _lib.lib().orp_poly2rbox_v3(None, 0, None, None) == 0


def test_new_entries_are_declared_and_bound():
    src = open(os.path.join(os.path.dirname(HERE), "include", "orp_b200.h")).read()
    for name, nargs, dbl in (("orp_dota_eval_aoe", 18, 11), ("orp_poly2rbox_v3", 4, None)):
        assert ("int %s(" % name) in src and name in _lib.SIGNATURES
        res, args = _lib.SIGNATURES[name]
        assert res is ctypes.c_int and len(args) == nargs
        assert dbl is None or args[dbl] is ctypes.c_double
        getattr(_lib.lib(), name)


def test_generator_reproduces_the_committed_golden(tmp_path):
    """the reference's own code, run again, writes the committed file byte for byte"""
    ref_root = os.environ.get("ORP_REFERENCE_ROOT", "/root/reference")
    polyiou = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "polyiou.py")
    if not (os.path.isdir(os.path.join(ref_root, "DOTA_devkit")) and os.path.exists(polyiou)):
        pytest.skip("needs the reference's source tree and its SWIG polyiou built by oracle/build_ref.py")
    out = tmp_path / "dota_aoe.json"
    subprocess.run([sys.executable, os.path.join(HERE, "golden", "gen_golden_dota_aoe.py"), ref_root, str(out)], check=True,
                   capture_output=True)
    assert out.read_bytes() == open(GOLDEN, "rb").read()
