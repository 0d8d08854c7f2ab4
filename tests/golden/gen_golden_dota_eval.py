"""Golden vectors of the DOTA Task1 evaluation: the reference's own DOTA_devkit/dota_evaluation_task1.py
(parse_gt, voc_eval, voc_ap) run unchanged on synthetic label / detection files, with IoU from its own SWIG polyiou
(oracle/_ref, built by oracle/build_ref.py) and only matplotlib.pyplot stubbed.  Writes tests/golden/dota_eval.json.

    python tests/golden/gen_golden_dota_eval.py [REFERENCE_ROOT]

Scores are unique throughout: np.argsort's order of equal keys depends on numpy's sort implementation.
"""
import contextlib
import io
import json
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "dota_eval.json")
CLASSES = ("plane", "ship", "harbor", "small-vehicle", "helicopter")


def _rect(x0, y0, x1, y1):
    return [x0, y0, x1, y0, x1, y1, x0, y1]


def _rot(cx, cy, w, h, a):
    c, s = np.cos(a), np.sin(a)
    pts = [(-w / 2, -h / 2), (w / 2, -h / 2), (w / 2, h / 2), (-w / 2, h / 2)]
    return [round(float(v), 1) for px, py in pts for v in (cx + c * px - s * py, cy + s * px + c * py)]


def build_case():
    """(image names, {image: label text}, {class: Task1 lines})"""
    rng = np.random.RandomState(2024)
    used = set()

    def score():
        while True:
            s = round(float(rng.uniform(0.01, 0.999)), 6)
            if s not in used:
                used.add(s)
                return s

    labels, dets = {}, {c: [] for c in CLASSES}

    def det(cls, img, quad, s=None):
        if s is None:
            s = score()
        else:
            assert s not in used
            used.add(s)
        dets[cls].append("%s %r %s" % (img, s, " ".join(repr(float(v)) for v in quad)))

    # G0: hand-made cases
    g0 = ["imagesource:GoogleEarth", "gsd:0.146"]
    g0.append(" ".join(str(v) for v in _rect(100, 100, 200, 200)) + " plane 0")          # target of two detections
    g0.append(" ".join(str(v) for v in _rect(110, 100, 210, 200)) + " plane 0")          # free second-best object
    g0.append(" ".join(str(v) for v in _rect(400, 400, 480, 470)) + " plane 1")          # difficult, hit twice
    g0.append(" ".join(str(v) for v in _rect(400, 700, 480, 770)) + " plane 2")          # difficult (nonzero flag)
    g0.append(" ".join(str(v) for v in _rect(900, 900, 1000, 980)) + " plane")           # 9 fields: not difficult
    g0.append("500 500 500 500 500 500 500 500 ship 0")                                   # zero area: NaN candidate
    g0.append(" ".join(str(v) for v in _rect(300, 300, 350, 350)) + " ship")             # 1 px AABB gap cases
    g0.append(" ".join(str(v) for v in _rect(2000, 2000, 2100, 2050)) + " helicopter 1")  # npos = 0 class
    g0.append(" ".join(str(v) for v in _rect(2300, 2000, 2400, 2050)) + " helicopter 1")
    labels["G0"] = "\n".join(g0) + "\n"
    det("plane", "G0", _rect(100, 100, 200, 200), 0.99)
    det("plane", "G0", _rect(104, 100, 204, 200), 0.98)      # best match is the claimed box: false positive
    det("plane", "G0", _rect(401, 401, 480, 470), 0.97)      # difficult: neither
    det("plane", "G0", _rect(400, 402, 481, 470), 0.96)      # difficult again: neither
    det("plane", "G0", _rect(900, 902, 1000, 980), 0.95)
    det("plane", "G0", _rect(400, 700, 480, 770), 0.5)
    det("ship", "G0", [500.25, 500.25, 500.25, 500.25, 500.25, 500.25, 500.25, 500.25], 0.94)   # 0 / 0 IoU
    det("ship", "G0", _rect(350.5, 300, 400, 350), 0.93)     # gap below 1 px: kept by the +1 rule, IoU 0
    det("ship", "G0", _rect(351, 300, 400, 350), 0.92)       # gap of exactly 1 px: dropped
    det("ship", "G0", _rect(351.25, 300, 400, 350), 0.91)    # beyond
    det("ship", "G0", _rect(300, 300, 350, 351), 0.90)
    det("helicopter", "G0", _rect(2000, 2000, 2100, 2050), 0.89)
    det("helicopter", "G0", _rect(2150, 2000, 2250, 2050), 0.88)
    det("helicopter", "G0", _rect(2300, 2000, 2400, 2050), 0.87)
    # G1: no ground truth of any class
    labels["G1"] = "imagesource:GoogleEarth\ngsd:0.2\n"
    det("plane", "G1", _rect(10, 10, 60, 60))
    det("harbor", "G1", _rect(1000, 1000, 1300, 1200))
    # G2..G7: DOTA-like full images, rotated objects, jittered detections, duplicates and false positives
    for k in range(2, 8):
        name = "G%d" % k
        lines = ["imagesource:GoogleEarth", "gsd:%r" % round(float(rng.uniform(0.1, 0.6)), 3)]
        for _ in range(rng.randint(20, 40)):
            cls = CLASSES[rng.randint(0, 4)]
            w, h = rng.uniform(20, 300), rng.uniform(15, 150)
            cx, cy, a = rng.uniform(200, 5000), rng.uniform(200, 5000), rng.uniform(-np.pi, np.pi)
            q = _rot(cx, cy, w, h, a)
            diff = int(rng.rand() < 0.15)
            lines.append(" ".join(repr(v) for v in q) + " " + cls + ("" if rng.rand() < 0.2 else " %d" % diff))
            for _ in range(rng.randint(0, 4)):
                j = rng.uniform(0.0, 0.35)
                det(cls, name, _rot(cx + rng.normal(0, j * w / 3), cy + rng.normal(0, j * h / 3),
                                    w * (1 + rng.normal(0, j / 3)), h * (1 + rng.normal(0, j / 3)), a + rng.normal(0, j)))
        for _ in range(rng.randint(5, 15)):
            det(CLASSES[rng.randint(0, 4)], name, _rot(rng.uniform(0, 5500), rng.uniform(0, 5500), rng.uniform(20, 200),
                                                       rng.uniform(15, 120), rng.uniform(-np.pi, np.pi)))
        labels[name] = "\n".join(lines) + "\n"
    for c in CLASSES:
        order = rng.permutation(len(dets[c]))
        dets[c] = [dets[c][i] for i in order]
    return sorted(labels), labels, dets


def _reference_module(ref_root):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    import polyiou  # noqa: F401  the reference's SWIG module
    plt = types.ModuleType("matplotlib.pyplot")
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = plt
    sys.modules.setdefault("matplotlib", mpl)
    sys.modules["matplotlib.pyplot"] = plt
    sys.path.insert(0, os.path.join(ref_root, "DOTA_devkit"))
    import dota_evaluation_task1 as ev
    return ev


def _floats(a):
    return [float(v) for v in np.asarray(a, np.float64)]


def main():
    ref_root = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("ORP_REFERENCE_ROOT", "/root/reference")
    ev = _reference_module(ref_root)
    names, labels, dets = build_case()
    out = {"classnames": list(CLASSES), "imagenames": names, "labels": labels, "detections": dets, "ovthresh": 0.5,
           "parse_gt": {}, "results": {"07": {}, "area": {}}}
    with tempfile.TemporaryDirectory() as d:
        for n in names:
            with open(os.path.join(d, n + ".txt"), "w") as f:
                f.write(labels[n])
            out["parse_gt"][n] = ev.parse_gt(os.path.join(d, n + ".txt"))
        for c in CLASSES:
            with open(os.path.join(d, "Task1_%s.txt" % c), "w") as f:
                f.write("\n".join(dets[c]) + "\n")
        with open(os.path.join(d, "imageset.txt"), "w") as f:
            f.write("\n".join(names) + "\n")
        for key, m07 in (("07", True), ("area", False)):
            for c in CLASSES:
                with contextlib.redirect_stdout(io.StringIO()), np.errstate(all="ignore"):
                    rec, prec, ap = ev.voc_eval(os.path.join(d, "Task1_{:s}.txt"), os.path.join(d, "{:s}.txt"),
                                                os.path.join(d, "imageset.txt"), c, ovthresh=0.5, use_07_metric=m07)
                out["results"][key][c] = {"rec": _floats(rec), "prec": _floats(prec), "ap": float(ap)}
    with open(OUT, "w") as f:
        json.dump(out, f, indent=0)
    print("wrote", OUT, {c: len(v) for c, v in dets.items()})


if __name__ == "__main__":
    main()
