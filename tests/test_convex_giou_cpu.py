"""CPU: convex_giou's golden vectors (tests/golden/convex_giou_ref.npz, the reference's own devrIoU of
mmdet/ops/iou/src/convex_giou_kernel.cu run as host C++) against independent computations, the GIoULoss registry entry the
configs name, and the argument checks that fire before any launch.

- The GIoU against OpenCV: cv2.convexHull of the points, cv2.intersectConvexConvex with the quad, the hull of the union.
- The gradient against central differences of an fp64 GIoU of our own (monotone-chain hulls, Sutherland-Hodgman
  clipping), on pairs whose hull and union-hull vertex sets do not change within the step."""
import importlib.util
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "convex_giou_ref.npz")
GENERIC = ("realistic", "disjoint", "contains", "inside", "quad_ccw", "quad_cw")


@pytest.fixture(scope="module")
def g():
    d = np.load(GOLDEN)
    return {k: d[k] for k in d}


def _hull(p):
    """monotone chain, counter-clockwise, collinear points dropped -> (ring [k,2], input indices [k])"""
    order = sorted(range(len(p)), key=lambda i: (p[i][0], p[i][1]))

    def chain(idx):
        st = []
        for i in idx:
            while len(st) >= 2:
                a, b = p[st[-2]], p[st[-1]]
                if (b[0] - a[0]) * (p[i][1] - a[1]) - (b[1] - a[1]) * (p[i][0] - a[0]) <= 0:
                    st.pop()
                else:
                    break
            st.append(i)
        return st

    lo, hi = chain(order), chain(order[::-1])
    idx = lo[:-1] + hi[:-1]
    return p[idx], idx


def _area(r):
    x, y = r[:, 0], r[:, 1]
    return 0.5 * float(np.dot(x, np.roll(y, -1)) - np.dot(y, np.roll(x, -1)))


def _clip(subject, window):
    """Sutherland-Hodgman: convex subject inside convex counter-clockwise window"""
    out = list(subject)
    for k in range(len(window)):
        a, b = window[k], window[(k + 1) % len(window)]
        inp, out = out, []
        if not inp:
            break
        side = [(b[0] - a[0]) * (v[1] - a[1]) - (b[1] - a[1]) * (v[0] - a[0]) for v in inp]
        for i in range(len(inp)):
            j = (i + 1) % len(inp)
            if side[i] >= 0:
                out.append(inp[i])
            if (side[i] >= 0) != (side[j] >= 0):
                t = side[i] / (side[i] - side[j])
                out.append(inp[i] + t * (inp[j] - inp[i]))
    return np.array(out).reshape(-1, 2)


def giou64(pts, quad):
    """fp64 GIoU of the hull of 9 points and a quadrilateral; also the hull and union-hull vertex index sets"""
    p = pts.reshape(9, 2).astype(np.float64)
    q = quad.reshape(4, 2).astype(np.float64)
    if _area(q) < 0:
        q = q[::-1]
    h, hidx = _hull(p)
    inter = _clip(h, q)
    ia = abs(_area(inter)) if len(inter) >= 3 else 0.0
    u = abs(_area(h)) + abs(_area(q)) - ia
    _, cidx = _hull(np.concatenate([h, q]))
    c = abs(_area(np.concatenate([h, q])[cidx]))
    return ia / u - (c - u) / c, frozenset(hidx), frozenset(cidx)


def test_golden_covers_the_cases(g):
    kinds = set(g["kind"].tolist())
    assert kinds >= set(GENERIC) | {"shared_corners", "duplicated", "collinear", "collinear_int", "all_equal", "edges"}
    assert g["pts"].shape[1:] == (18,) and g["quads"].shape[1:] == (8,) and g["out"].shape[1:] == (19,)
    real = g["out"][g["kind"] == "realistic", 18]
    assert (real < 0).any() and (real > 0.5).any()                  # GIoU spread over both signs
    iou = np.array([_iou_cv2(p, q) for p, q in zip(g["pts"][g["kind"] == "realistic"][:400],
                                                  g["quads"][g["kind"] == "realistic"][:400])])
    assert (iou < 0.1).mean() > 0.05 and (iou > 0.5).mean() > 0.02   # IoU spread over 0..1
    assert np.abs(g["quads"]).max() > 3000


def _iou_cv2(pts, quad):
    cv2 = pytest.importorskip("cv2")
    c = quad.reshape(4, 2).astype(np.float64).mean(0)
    h = cv2.convexHull((pts.reshape(9, 2) - c).astype(np.float32)).reshape(-1, 2)
    q = (quad.reshape(4, 2) - c).astype(np.float32)
    ia, _ = cv2.intersectConvexConvex(h, q)
    return ia / (cv2.contourArea(h) + cv2.contourArea(q) - ia)


def test_golden_giou_agrees_with_opencv(g):
    cv2 = pytest.importorskip("cv2")
    sel = np.isin(g["kind"], GENERIC)
    worst = 0.0
    for pts, quad, out in zip(g["pts"][sel], g["quads"][sel], g["out"][sel]):
        c = quad.reshape(4, 2).astype(np.float64).mean(0)          # pair-local coordinates keep OpenCV's float32 exact enough
        p = (pts.reshape(9, 2) - c).astype(np.float32)
        q = (quad.reshape(4, 2) - c).astype(np.float32)
        h = cv2.convexHull(p).reshape(-1, 2)
        ia, _ = cv2.intersectConvexConvex(h, q)
        u = cv2.contourArea(h) + cv2.contourArea(q) - ia
        ch = cv2.convexHull(np.concatenate([h, q])).reshape(-1, 2)
        ca = cv2.contourArea(ch)
        worst = max(worst, abs(ia / u - (ca - u) / ca - float(out[18])))
    assert sel.sum() > 2500
    assert worst < 1e-5, worst


def test_golden_gradient_matches_central_differences(g):
    sel = np.nonzero(np.isin(g["kind"], GENERIC))[0][::5]
    h = 1e-3
    checked, errs = 0, []
    for i in sel:
        pts, quad, grad = g["pts"][i].astype(np.float64), g["quads"][i], g["out"][i, :18].astype(np.float64)
        v0, hs, cs = giou64(pts, quad)
        assert abs(v0 - g["out"][i, 18]) < 1e-5
        fd = np.zeros(18)
        stable = True
        for k in range(18):
            a, b = pts.copy(), pts.copy()
            a[k] += h
            b[k] -= h
            va, ha, ca = giou64(a, quad)
            vb, hb, cb = giou64(b, quad)
            stable = stable and ha == hs == hb and ca == cs == cb
            fd[k] = (va - vb) / (2 * h)
        if not stable:
            continue
        checked += 1
        errs.append(np.abs(fd - grad).max() / max(1e-6, np.abs(fd).max()))
        nonhull = [k for k in range(9) if k not in hs]
        assert (grad.reshape(9, 2)[nonhull] == 0).all()            # interior points get gradient 0
    assert checked > 300, checked
    assert max(errs) < 1e-2, (max(errs), np.median(errs))


def _config(name):
    spec = importlib.util.spec_from_file_location("cfg_" + name, os.path.join(ROOT, "configs", "dota", name + ".py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.mark.parametrize("name", ["orientedrepoints_r50_demo", "orientedrepoints_r101_demo",
                                  "orientedrepoints_swin_tiny_demo"])
def test_build_loss_from_the_configs(name):
    from orientedreppoints_b200.losses import GIoULoss
    from orientedreppoints_b200.models import LOSSES, build_loss
    head = _config(name).model["bbox_head"]
    assert LOSSES.get("GIoULoss") is GIoULoss
    for key, w in (("loss_rbox_init", 0.375), ("loss_rbox_refine", 1.0)):
        loss = build_loss(head[key])
        assert isinstance(loss, GIoULoss) and loss.loss_weight == w and loss.reduction == "mean"


def test_errors_before_the_launch():
    """shapes are checked first (a wrong row width would make the kernel read past the buffer), then the device"""
    from orientedreppoints_b200.losses import GIoULoss
    from orientedreppoints_b200.ops import convex_giou
    with pytest.raises(TypeError, match="CUDA"):
        convex_giou(torch.zeros(2, 18), torch.zeros(2, 8))
    with pytest.raises(TypeError, match="CUDA"):
        GIoULoss()(torch.zeros(2, 18), torch.zeros(2, 8))
    with pytest.raises(ValueError, match="aligned"):
        convex_giou(torch.zeros(3, 18), torch.zeros(2, 8))
    for shape in [(3, 16), (3, 19), (18,), (1, 3, 18)]:
        with pytest.raises(ValueError, match=r"\[N, 18\]"):
            convex_giou(torch.zeros(shape), torch.zeros(3, 8))
    for shape in [(3, 9), (8,), (3, 4, 2)]:
        with pytest.raises(ValueError, match=r"\[N, 8\]"):
            convex_giou(torch.zeros(3, 18), torch.zeros(shape))
