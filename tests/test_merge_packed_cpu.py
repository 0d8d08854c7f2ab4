"""CPU: the merge of packed detections (orp_result_merge / dota.result_merge.merge_packed) - its numpy restatement
against the reference's own mergesingle output, the slot arithmetic of the all-gather's layout, and the ABI's argument
checks, none of which needs a device."""
import ctypes
import json
import os
import sys

import numpy as np
import pytest
import torch

from orientedreppoints_b200 import _lib, gather
from orientedreppoints_b200.dota import result_merge as rm

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)
from merge_packed_ref import merge_packed_ref, packed_rows  # noqa: E402


@pytest.fixture(scope="module")
def fx():
    g = dict(np.load(os.path.join(HERE, "golden", "result_merge_packed.npz")))
    g.update(json.load(open(os.path.join(HERE, "golden", "result_merge_packed.json"))))
    return g


def as_merged(ref, nimg):
    return rm.MergedDetections(*(torch.from_numpy(ref[k]) for k in ("cls", "img", "score", "quad", "src_row", "cls_off")), nimg)


def test_fixture_holds_the_cases_it_is_for(fx):
    packed, cap = fx["packed"], fx["packed"].shape[1] - 1
    counts = packed[fx["tile_slot"], cap, 0]
    assert (counts == 0).sum() == 1 and counts.max() <= cap
    assert set(fx["tile_rate"].tolist()) == {1.0, 0.5} and len(fx["images"]) == 3
    quad, score, cls, img = packed_rows(packed, fx["tile_slot"], fx["tile_xy"], fx["tile_rate"], fx["tile_img"], 3, 15)
    assert sorted(set(cls.tolist())) == [0, 2, 4, 12]
    assert 1 not in set(img[cls == 2].tolist()) and set(img[cls == 0].tolist()) == {0, 1, 2}
    for m in range(3):                                             # rates 1 and 0.5 of the same image
        assert set(fx["tile_rate"][fx["tile_img"] == m].tolist()) == {1.0, 0.5}
    for c in (0, 2, 4, 12):                                        # equal scores across different images
        s, m = score[cls == c], img[cls == c]
        assert any(len(set(m[s == v].tolist())) > 1 for v in np.unique(s))
    x, y = quad[:, 0::2], quad[:, 1::2]
    area = 0.5 * np.abs((x * np.roll(y, -1, 1) - np.roll(x, -1, 1) * y).sum(1))
    assert (area == 0).sum() >= 3
    # the order of the images differs between classes: it is the first appearance among the class's rows
    firsts = {c: [l.split("__")[0] for l in fx["merged"][fx["classes"][c]]] for c in (0, 4, 12)}
    orders = {c: list(dict.fromkeys(v)) for c, v in firsts.items()}
    assert len({tuple(v) for v in orders.values()}) > 1


def test_restatement_and_to_lines_equal_the_reference_mergesingle_output(fx, po):
    ref = merge_packed_ref(fx["packed"], fx["tile_slot"], fx["tile_xy"], fx["tile_rate"], fx["tile_img"], 3, 15,
                           fx["nms_thresh"], nms=po.nms_poly_f64)
    lines = as_merged(ref, 3).to_lines(fx["images"], fx["classes"])
    assert lines == fx["merged"]
    assert sum(map(len, lines.values())) == len(ref["cls"]) == int(ref["cls_off"][-1]) > 100
    assert len(ref["cls"]) < sum(map(len, fx["lines"]))            # the merge had something to suppress


def test_write_task1_writes_every_class_file(fx, po, tmp_path):
    ref = merge_packed_ref(fx["packed"], fx["tile_slot"], fx["tile_xy"], fx["tile_rate"], fx["tile_img"], 3, 15,
                           fx["nms_thresh"], nms=po.nms_poly_f64)
    as_merged(ref, 3).write_task1(str(tmp_path), fx["images"], fx["classes"])
    for c in fx["classes"]:
        assert open(os.path.join(str(tmp_path), "Task1_%s.txt" % c)).read().splitlines() == fx["merged"][c]


@pytest.mark.parametrize("world,t,dataset_len", [(1, 5, 5), (2, 4, 7), (3, 3, 7), (3, 4, 12), (2, 3, 9)])
def test_dataset_slots_agrees_with_interleave(world, t, dataset_len):
    cap = 3
    buf = torch.zeros(world, t, cap + 1, 28)
    buf[:, :, :cap, 0] = torch.arange(world * t * cap, dtype=torch.float32).reshape(world, t, cap)
    counts = torch.arange(world * t).reshape(world, t) % (cap + 1)
    slots = gather.dataset_slots(world, t, dataset_len)
    assert slots.dtype == torch.int32 and slots.shape[0] == min(dataset_len, world * t)
    flat, flat_counts = buf.reshape(world * t, cap + 1, 28), counts.reshape(-1)
    tiles = gather.interleave(buf[:, :, :cap], counts, dataset_len)
    assert len(tiles) == slots.shape[0]
    for i, (rows, _) in enumerate(tiles):
        s = int(slots[i])
        assert torch.equal(rows, flat[s, :int(flat_counts[s]), :27])
    assert len(set(slots.tolist())) == slots.shape[0]


def _call(**kw):
    a = dict(packed=256, S=2, cap=4, tile_slot=256, tile_xy=256, tile_rate=256, tile_img=256, Tn=2, ncls=15, nimg=3, thresh=0.1,
             union_mode=_lib.ORP_UNION_NAN_SUPPRESSES, max_rows=8, count=256, cls_off=256, cls=256, img=256, score=256, quad=256,
             src_row=256, status=256)
    a.update(kw)
    vp = lambda v: ctypes.c_void_p(v)   # noqa: E731  (256: a non-NULL placeholder that a refused call never reads)
    return _lib.lib().orp_result_merge(vp(a["packed"]), a["S"], a["cap"], vp(a["tile_slot"]), vp(a["tile_xy"]), vp(a["tile_rate"]),
                                       vp(a["tile_img"]), a["Tn"], a["ncls"], a["nimg"], a["thresh"], a["union_mode"],
                                       a["max_rows"], vp(a["count"]), vp(a["cls_off"]), vp(a["cls"]), vp(a["img"]), vp(a["score"]),
                                       vp(a["quad"]), vp(a["src_row"]), vp(a["status"]), None)


@pytest.mark.parametrize("bad", [dict(packed=0), dict(tile_slot=0), dict(tile_xy=0), dict(tile_rate=0), dict(tile_img=0),
                                 dict(count=0), dict(cls_off=0), dict(status=0), dict(cls=0), dict(img=0), dict(score=0),
                                 dict(quad=0), dict(src_row=0), dict(cap=0), dict(S=-1), dict(Tn=-1), dict(max_rows=-1),
                                 dict(ncls=0), dict(nimg=0), dict(ncls=1 << 16, nimg=1 << 16), dict(S=1 << 20, cap=1 << 12), dict(Tn=1 << 20, cap=1 << 12),
                                 dict(union_mode=_lib.ORP_UNION_NAN_KEEPS), dict(union_mode=_lib.ORP_UNION_GUARD),
                                 dict(thresh=float("nan"))])
def test_result_merge_refuses_bad_arguments_before_any_cuda_call(bad):
    """every check a host can make returns ORP_EINVAL first: a call that went on to the device would report the missing
    GPU (ORP_ENOGPU / ORP_ECUDA) here, or read the placeholder pointers"""
    assert _call(**bad) == -1
    assert b"orp_result_merge" in _lib.lib().orp_last_error()


def test_result_merge_is_declared_and_bound():
    src = open(os.path.join(os.path.dirname(HERE), "include", "orp_b200.h")).read()
    assert "int orp_result_merge(" in src and "orp_result_merge" in _lib.SIGNATURES
    res, args = _lib.SIGNATURES["orp_result_merge"]
    assert res is ctypes.c_int and len(args) == 22 and args[10] is ctypes.c_double
    for name, v in (("ORP_MERGE_BAD_COUNT", 1), ("ORP_MERGE_BAD_TILE", 2), ("ORP_MERGE_ROWS_OVERFLOW", 4)):
        assert getattr(_lib, name) == v and ("#define %s %d" % (name, v)) in src


def test_merge_packed_refuses_a_host_buffer(fx):
    with pytest.raises(ValueError):
        rm.merge_packed(torch.from_numpy(fx["packed"]), fx["tile_slot"], fx["tile_xy"], fx["tile_rate"], fx["tile_img"], 3)


def test_all_gather_hands_over_the_packed_buffer_on_request():
    """packed=True keeps every tile's count row, which merge_packed reads; the default pair has it split off"""
    dets, labels = torch.randn(3, 4, 27), torch.randint(0, 15, (3, 4))
    buf, cnt = gather.pack(dets, labels, torch.tensor([4, 0, 2], dtype=torch.int32))
    whole = gather.all_gather_detections(buf, cnt, packed=True)
    assert whole.shape == (1, 3, 5, 28) and torch.equal(whole[0], buf) and whole[0, :, 4, 0].tolist() == [4.0, 0.0, 2.0]
    assert not whole[0, :, 4, 1:].any()                             # the rest of the count row is zero padding
    assert torch.equal(gather.all_gather_detections(buf, cnt, async_op=True, packed=True).wait(), whole)
    all_buf, all_counts = gather.all_gather_detections(buf, cnt)
    assert all_buf.shape == (1, 3, 4, 28) and all_counts.tolist() == [[4, 0, 2]]
