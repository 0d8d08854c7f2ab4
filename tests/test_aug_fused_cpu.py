"""CPU: the surface of the multi-view post-processing (orp_head_postprocess_aug) that needs no device - the symbol and its
binding, every refusal the host can make before the first CUDA call, the meta table of get_bboxes_aug_fused, and the
return forms of aug_test with the device call stubbed."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from orientedreppoints_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORP_EINVAL = -1
LEVELS_1024 = [(128, 128), (64, 64), (32, 32), (16, 16), (8, 8)]


def test_symbol_declared_exported_and_bound():
    src = open(os.path.join(ROOT, "include", "orp_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    m = re.search(r"\bint\s+orp_head_postprocess_aug\s*\(([^)]*)\)\s*;", src)
    assert m, "orp_head_postprocess_aug is not declared"
    params = [p.strip() for p in m.group(1).split(",")]
    res, args = _lib.SIGNATURES["orp_head_postprocess_aug"]
    assert res is ctypes.c_int and len(args) == len(params) == 19
    for p, a in zip(params, args):                       # pointers are void pointers in the binding, scalars keep their type
        want = ctypes.c_void_p if "*" in p else {"int": ctypes.c_int, "float": ctypes.c_float, "double": ctypes.c_double}[p.split()[0]]
        assert a is want, (p, a)
    assert hasattr(_lib.lib(), "orp_head_postprocess_aug")
    # the one-view entry keeps its signature
    assert len(_lib.SIGNATURES["orp_head_postprocess"][1]) == 17


def _call(nviews=2, levels=LEVELS_1024, B=2, num_cls=15, nms_pre=2000, max_per_img=100, meta=True, nlevels=None, outs=True):
    """orp_head_postprocess_aug on placeholder addresses: only calls the host refuses are made with them"""
    ph = 256
    nl = len(levels) if nlevels is None else nlevels
    n = max(1, nviews) * len(levels)
    ptrs = (ctypes.c_void_p * n)(*[ph] * n)
    hs = (ctypes.c_int * n)(*[h for h, _ in levels] * max(1, nviews))
    ws = (ctypes.c_int * n)(*[w for _, w in levels] * max(1, nviews))
    ss = (ctypes.c_int * n)(*[8 << i for i in range(len(levels))] * max(1, nviews))
    out = ph if outs else None
    rc = _lib.lib().orp_head_postprocess_aug(nviews, nl, ptrs, ptrs, hs, ws, ss, B, num_cls, nms_pre, 0.05, 0.4, max_per_img,
                                             ph if meta else None, None, out, out, out, None)
    return rc, _lib.lib().orp_last_error().decode()


@pytest.mark.parametrize("kw,word", [
    (dict(nviews=0), "bad arguments"),
    (dict(nviews=-3), "bad arguments"),
    (dict(nviews=17), "(view, level)"),                  # 17 views x 5 levels > the 80 entries of the level table
    (dict(nviews=14), "candidates per image"),           # 14 x 5344 x 15 >= 2^20 (13 views fit)
    (dict(nviews=2, nms_pre=-1, levels=[(512, 512)]), "candidates per image"),
    (dict(meta=False), "view_meta"),
    (dict(B=0), "bad arguments"),
    (dict(B=2048), "batch too large"),
    (dict(B=1024, num_cls=1024), "batch too large"),
    (dict(max_per_img=0), "bad arguments"),
    (dict(nlevels=0), "bad arguments"),
    (dict(nlevels=9), "bad arguments"),
    (dict(outs=False), "bad arguments"),
    (dict(levels=[(0, 16)]), "bad level"),
], ids=lambda v: "-".join("%s=%s" % kv for kv in v.items()).replace(" ", "") if isinstance(v, dict) else None)
def test_refusals_come_before_the_device(kw, word):
    """ORP_EINVAL with a message naming the entry; a call that reached the device would fault on the placeholder
    addresses or report the missing device instead"""
    rc, err = _call(**kw)
    assert rc == ORP_EINVAL, (rc, err)
    assert err.startswith("orp_head_postprocess_aug:") and word in err, err


def test_candidate_bound_is_the_select_key_width():
    """13 views of the full 1024^2 configuration stay under the 2^20 candidates per image the select keys hold, 14 do not"""
    per_view = sum(min(h * w, 2000) for h, w in LEVELS_1024) * 15
    assert 13 * per_view < (1 << 20) <= 14 * per_view and 13 * len(LEVELS_1024) <= 80


def test_meta_table():
    from orientedreppoints_b200.core.get_bboxes import aug_meta_table
    metas = [[dict(img_shape=(1024, 1024, 3), scale_factor=1.0, flip=False), dict(img_shape=(1024, 1000, 3), scale_factor=1.0, flip=False)],
             [dict(img_shape=(960, 960, 3), scale_factor=0.9375, flip=True, flip_direction='horizontal'),
              dict(img_shape=(960, 937, 3), scale_factor=np.array([1.171875] * 4, np.float32), flip=True)]]
    t = aug_meta_table(metas, rescale=True)
    assert t.dtype == np.float32 and t.shape == (2 * 2 * 3 + 2,)
    view = t[:12].reshape(2, 2, 3)
    assert view[0].tolist() == [[0.0, 0.0, 1.0], [0.0, 0.0, 1.0]]       # unflipped views need no width
    assert view[1].tolist() == [[1.0, 960.0, 0.9375], [1.0, 937.0, 1.171875]]
    assert t[12:].tolist() == [1.0, 1.0]
    # rescale=False: the result goes back into the first view's frame
    metas[0][1]['scale_factor'] = 0.78125
    assert aug_meta_table(metas, rescale=False)[12:].tolist() == [1.0, 0.78125]
    with pytest.raises(ValueError, match="horizontal"):
        aug_meta_table([[dict(img_shape=(8, 8, 3), scale_factor=1.0, flip=True, flip_direction='vertical')]], True)
    with pytest.raises(ValueError, match="one scale"):
        aug_meta_table([[dict(img_shape=(8, 8, 3), scale_factor=np.array([0.5, 0.75, 0.5, 0.75]), flip=False)]], True)
    with pytest.raises(ValueError, match="same"):
        aug_meta_table([metas[0], metas[1][:1]], True)


def _stub_detector(monkeypatch, n, counts, cap=6):
    """a detector without weights or device: the dense graph and the device pipeline are stand-ins"""
    from orientedreppoints_b200.core import get_bboxes as gb
    from orientedreppoints_b200.detector import OrientedRepPointsDetector as D
    det = object.__new__(D)
    det.device = torch.device("cpu")
    det.test_cfg = dict(nms_pre=2000, score_thr=0.05, nms=dict(type='rnms', iou_thr=0.4), max_per_img=cap)
    seen = dict(dense=[], fused=[])

    def dense(img, valid_hw):
        seen["dense"].append((id(img), valid_hw))
        return [(img, None, img)] * 5, None
    det._forward_dense_opt = dense
    dets = torch.arange(n * cap * 27, dtype=torch.float32).reshape(n, cap, 27)
    labels = (torch.arange(n * cap) % 15).reshape(n, cap)

    def fused(cls, ref, strides, img_metas, cfg, rescale):
        seen["fused"].append((len(cls), len(cls[0]), tuple(strides), rescale))
        return dets, labels, torch.tensor(counts, dtype=torch.int32)
    monkeypatch.setattr(gb, "get_bboxes_aug_fused", fused)
    return det, seen, dets, labels


def _views(n, nv=4):
    return [torch.zeros(n, 3, 8, 8) for _ in range(nv)], [[dict(img_shape=(8, 8, 3), scale_factor=1.0, flip=bool(v % 2))] * n for v in range(nv)]


def test_aug_test_return_forms(monkeypatch):
    # N > 1: a list of rbbox2result lists, rows box | score cut at the counts
    det, seen, dets, labels = _stub_detector(monkeypatch, 3, [2, 0, 6])
    views, metas = _views(3)
    valids = ["v%d" % k for k in range(4)]
    out = det._aug_test(views, metas, True, valids, False)
    assert seen["dense"] == [(id(v), k) for v, k in zip(views, valids)]       # one dense pass per view, the caller's tensors
    assert seen["fused"] == [(4, 5, (8, 16, 32, 64, 128), True)]
    assert len(out) == 3 and all(len(r) == 15 and all(a.shape[1] == 9 for a in r) for r in out)
    assert [sum(len(a) for a in r) for r in out] == [2, 0, 6]
    for c in range(15):
        want = dets[2, :6, 18:][labels[2, :6] == c].numpy()
        assert np.array_equal(out[2][c], want)
    # the padded form hands the device triple through, counts unread
    triple = det._aug_test(views, metas, False, None, "padded")
    assert triple[0] is dets and triple[1] is labels and triple[2].tolist() == [2, 0, 6]
    assert seen["fused"][-1][3] is False and seen["dense"][-1][1] is None
    # N == 1: the image's list itself
    det, seen, dets, labels = _stub_detector(monkeypatch, 1, [4])
    views, metas = _views(1, nv=2)
    one = det._aug_test(views, metas, True, None, False)
    assert len(one) == 15 and sum(len(a) for a in one) == 4 and isinstance(one[0], np.ndarray)


def test_aug_test_refusals(monkeypatch):
    det, _, _, _ = _stub_detector(monkeypatch, 2, [1, -1])
    views, metas = _views(2)
    with pytest.raises(_lib.OrpError, match="overflow"):           # the NMS overflow mark is never taken for a count
        det._aug_test(views, metas, True, None, False)
    with pytest.raises(ValueError, match="same"):
        det._aug_test(views[:3], metas, True, None, False)
    with pytest.raises(ValueError, match="same"):
        det._aug_test(views, metas[:3] + [metas[3][:1]], True, None, False)
    det.fused_post = False                                         # the op-by-op merge has no padded form
    with pytest.raises(ValueError, match="padded"):
        det._aug_test(views, metas, True, None, "padded")
