"""Golden vectors of the DOTA mAOE: the reference's own DOTA_devkit/mAOE_evaluation.py (aoe_eval) and
dota_poly2rbox.py (poly2rbox_single_v3) run unchanged, with IoU from its own SWIG polyiou (oracle/_ref, built by
oracle/build_ref.py).  The one change is in-process: numpy >= 1.24 removed the `np.float` alias both files use, and it
is put back as `float`.  Writes tests/golden/dota_aoe.json:

  aoe_eval   angle_dif_list of every class of gen_golden_dota_eval.build_case() (the detections and labels of
             dota_eval.json) at ovthresh 0.5 and 0.7
  edge       poly2rbox_single_v3 of a set of quads at the edges of its arithmetic, each with a kind: axis-aligned
             rectangles from every start vertex in both windings, edges at exactly +-45 / +-135 degrees, squares, and
             squares turned by 45 degrees and rhombi (|angle1| == |angle2|), edge ratios at float32(1.15) and its
             float32 neighbours, a zero-length edge and a point, NaN coordinates, 0.1 px decimals near 10 000 px,
             mirrored parallelograms

    python tests/golden/gen_golden_dota_aoe.py [REFERENCE_ROOT] [OUT]

The reference's host numpy computes the angles: they may differ from another host's in the last bit.
"""
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "dota_aoe.json")
sys.path.insert(0, HERE)

from gen_golden_dota_eval import CLASSES, _rot, build_case  # noqa: E402


def _reference_modules(ref_root):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    import polyiou  # noqa: F401  the reference's SWIG module
    np.float = float                 # the alias numpy >= 1.24 removed; nothing else is patched
    sys.path.insert(0, os.path.join(ref_root, "DOTA_devkit"))
    import dota_poly2rbox
    import mAOE_evaluation
    return mAOE_evaluation, dota_poly2rbox


def _starts(pts):
    """the quad from every start vertex, in both windings"""
    out = []
    for ring in (pts, pts[::-1]):
        for k in range(4):
            out.append([float(v) for p in ring[k:] + ring[:k] for v in p])
    return out


def edge_set():
    """[(kind, quad)]"""
    rows = []
    rows += [("axis", q) for q in _starts([(10, 20), (110, 20), (110, 60), (10, 60)])]
    rows += [("diag", q) for q in _starts([(500, 500), (530, 530), (520, 540), (490, 510)])]
    rows += [("square", q) for q in _starts([(0, 0), (10, 0), (10, 10), (0, 10)])]
    rows += [("diamond", q) for q in _starts([(200, 100), (210, 110), (200, 120), (190, 110)])]
    rows += [("rhombus", q) for q in _starts([(0, 0), (10, 3), (20, 0), (10, -3)])]
    f = np.float32(1.15)
    for r in (np.nextafter(f, np.float32(0)), f, np.nextafter(f, np.float32(2))):
        r = float(r)                 # short edge 1->2 horizontal, long edge vertical: the two branches disagree
        rows += [("ratio", [0.0, 0.0, 1.0, 0.0, 1.0, r, 0.0, r]), ("ratio", [0.0, 0.0, r, 0.0, r, 1.0, 0.0, 1.0])]
    rows += [("degenerate", [5.0, 5.0, 5.0, 5.0, 15.0, 5.0, 15.0, 8.0]), ("degenerate", [7.0, 3.0] * 4),
             ("degenerate", [0.0] * 8)]
    nan = float("nan")
    rows += [("nan", [nan] * 8), ("nan", [nan, 0.0, 10.0, 0.0, 10.0, 10.0, 0.0, 10.0]),
             ("nan", [0.0, 0.0, 10.0, 0.0, 10.0, nan, 0.0, 10.0]), ("nan", [0.0, 0.0, 10.0, 0.0, 10.0, 10.0, 0.0, nan])]
    rng = np.random.RandomState(5)
    for _ in range(24):
        w = rng.uniform(10, 300)
        h = w * rng.choice([rng.uniform(0.3, 0.95), rng.uniform(0.86, 0.88), 1.0])
        rows.append(("decimal", _rot(rng.uniform(9000, 10000), rng.uniform(9000, 10000), w, h, rng.uniform(-np.pi, np.pi))))
    for x0, y0, dx, dy in ((0.0, 0.0, 10.1, 3.3), (0.0, 0.0, 10.1, -3.3), (9000.0, 9000.0, 10.25, 3.5),
                           (-4.0, 0.0, 0.3, 7.9)):
        rows.append(("mirror", [x0, y0, x0 + dx, y0 + dy, x0 + 2 * dx, y0, x0 + dx, y0 - dy]))
    return rows


def main():
    ref_root = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("ORP_REFERENCE_ROOT", "/root/reference")
    out_path = sys.argv[2] if len(sys.argv) > 2 else OUT
    aoe, p2r = _reference_modules(ref_root)
    names, labels, dets = build_case()
    with open(os.path.join(HERE, "dota_eval.json")) as f:
        ev = json.load(f)
    assert ev["detections"] == dets and ev["labels"] == labels, "build_case() no longer gives dota_eval.json's case"
    out = {"classnames": list(CLASSES), "inputs": "dota_eval.json", "aoe_eval": {}, "edge": {"kind": [], "quad": [], "rbox": []}}
    with tempfile.TemporaryDirectory() as d:
        for n in names:
            with open(os.path.join(d, n + ".txt"), "w") as f:
                f.write(labels[n])
        for c in CLASSES:
            with open(os.path.join(d, "Task1_%s.txt" % c), "w") as f:
                f.write("\n".join(dets[c]) + "\n")
        with open(os.path.join(d, "imageset.txt"), "w") as f:
            f.write("\n".join(names) + "\n")
        for thr in (0.5, 0.7):
            out["aoe_eval"][repr(thr)] = {
                c: [float(v) for v in aoe.aoe_eval(os.path.join(d, "Task1_{:s}.txt"), os.path.join(d, "{:s}.txt"),
                                                   os.path.join(d, "imageset.txt"), c, ovthresh=thr)] for c in CLASSES}
    with np.errstate(all="ignore"):
        for kind, q in edge_set():
            out["edge"]["kind"].append(kind)
            out["edge"]["quad"].append(q)
            out["edge"]["rbox"].append(list(p2r.poly2rbox_single_v3(q)))
    with open(out_path, "w") as f:
        json.dump(out, f, indent=0)
    print("wrote", out_path, {k: len(v) for k, v in out["aoe_eval"]["0.7"].items()}, len(out["edge"]["kind"]), "edge rows")


if __name__ == "__main__":
    main()
