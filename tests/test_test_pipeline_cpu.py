"""CPU: the test pipeline's host side (orientedreppoints_b200/datasets/pipelines.py) - cv2's INTER_LINEAR coefficient
tables applied in integer numpy against cv2.resize, bit for bit; mmcv's rescale rule and the view metas on analytic cases;
the configs' test_pipeline against the reference configs (tests/golden/gen_golden_test_pipeline.py)."""
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

from orientedreppoints_b200.datasets import pipelines as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "test_pipelines.json")))

# (src h, w) -> (dst h, w): the configs' test scales of a 1024^2 tile, exact 2x, odd ratios up and down, 1-pixel sources
RESIZE_CASES = [((1024, 1024), (960, 960)), ((1024, 1024), (768, 768)), ((1024, 1024), (1280, 1280)),
                ((1024, 1024), (1000, 1000)), ((1024, 1024), (512, 512)), ((333, 517), (250, 388)), ((100, 77), (131, 203)),
                ((64, 64), (48, 48)), ((1, 50), (3, 70)), ((50, 1), (70, 3)), ((1, 1), (5, 7)), ((7, 9), (3, 2)),
                ((300, 420), (250, 350)), ((256, 256), (1024, 1024))]


def _cfg(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "configs", "dota", name + ".py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.mark.parametrize("flip", [False, True])
@pytest.mark.parametrize("src,dst", RESIZE_CASES, ids=lambda v: "x".join(map(str, v)))
def test_tables_reproduce_cv2_resize_bitwise(src, dst, flip):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.RandomState(src[0] * 131 + dst[1])
    img = rng.randint(0, 256, src + (3,)).astype(np.uint8)
    ref = cv2.resize(img, (dst[1], dst[0]), interpolation=cv2.INTER_LINEAR)
    if flip:
        ref = ref[:, ::-1]
    out = P.resize_u8_numpy(img, (dst[1], dst[0]), flip)
    assert out.shape == ref.shape and np.array_equal(out, ref)


def test_tables_layout():
    xt = P.resize_tables(1024, 960, True)
    yt = P.resize_tables(1024, 960, False)
    assert xt.dtype == np.int32 and xt.shape == (960, 4) and yt.shape == (960, 4)
    for t, n in ((xt, 1024), (yt, 1024)):
        assert t[:, :2].min() >= 0 and t[:, :2].max() <= n - 1
        assert np.all(np.abs(t[:, 2] + t[:, 3] - 2048) <= 1)
    # upscaling: the first row's weight keeps its negative offset (rows clamp only when read), the first column does not
    xt, yt = P.resize_tables(256, 1024, True), P.resize_tables(256, 1024, False)
    assert tuple(xt[0]) == (0, 1, 2048, 0)
    assert tuple(yt[0][:2]) == (0, 0) and tuple(yt[0][2:]) == (768, 1280)       # y = -0.375: row -1 (read as 0) x 0.375, row 0 x 0.625
    assert tuple(xt[-1]) == (255, 255, 2048, 0)


@pytest.mark.parametrize("scale,want", [((1333, 960), ((960, 960), 0.9375)), ((1333, 1280), ((1280, 1280), 1.25)),
                                        ((1333, 768), ((768, 768), 0.75)), ((1333, 1024), ((1024, 1024), 1.0))])
def test_rescale_size_tile(scale, want):
    assert P.rescale_size((1024, 1024), scale) == want


def test_rescale_size_rectangle():
    (w, h), sf = P.rescale_size((420, 300), (1333, 250))
    assert (h, w) == (250, 350) and sf == 250 / 300


def _views(pipeline, shape, n=1):
    """the per-view metas up to Pad (the device resize itself is not run here)"""
    cfg = [t for t in pipeline if t["type"] != "LoadImageFromFile"]
    assert len(cfg) == 1 and cfg[0]["type"] == "MultiScaleFlipAug"
    aug = cfg[0]
    inner = P.Compose([t for t in aug["transforms"] if t["type"] not in ("ImageToTensor", "Collect")])
    scales = aug["img_scale"] if isinstance(aug["img_scale"], list) else [aug["img_scale"]]
    out = []
    for s in scales:
        for f in ([False, True] if aug["flip"] else [False]):
            out.append(inner(dict(img=None, img_shape=shape, ori_shape=shape, scale=s, flip=f)))
    return out


def test_metas_of_the_config_scales():
    for name, side, sf in (("orientedrepoints_r50_demo", 1024, 1.0), ("orientedrepoints_r101_demo", 960, 0.9375),
                           ("orientedrepoints_swin_tiny_demo", 960, 0.9375)):
        (v,) = _views(_cfg(name).test_pipeline, (1024, 1024, 3))
        assert v["img_shape"] == (side, side, 3) and v["pad_shape"] == (side, side, 3), name
        assert v["scale_factor"] == sf and isinstance(v["scale_factor"], float)
        assert v["flip"] is False and v["flip_direction"] == "horizontal"
        assert v["img_norm_cfg"]["to_rgb"] is True and v["img_norm_cfg"]["mean"].dtype == np.float32


def test_metas_padded_multiscale_flip():
    pipe = [dict(type="MultiScaleFlipAug", img_scale=[(1333, 250), (1333, 768)], flip=True,
                 transforms=[dict(type="RotateResize", keep_ratio=True), dict(type="RotateRandomFlip"),
                             dict(type="Normalize", mean=[1, 2, 3], std=[4, 5, 6], to_rgb=False), dict(type="Pad", size_divisor=32)])]
    vs = _views(pipe, (300, 420, 3))
    assert [(v["img_shape"], v["pad_shape"], v["flip"]) for v in vs] == [
        ((250, 350, 3), (256, 352, 3), False), ((250, 350, 3), (256, 352, 3), True),
        ((768, 1075, 3), (768, 1088, 3), False), ((768, 1075, 3), (768, 1088, 3), True)]
    assert vs[0]["scale_factor"] == 250 / 300 and vs[2]["scale_factor"] == 768 / 300


def test_identity_view_runs_on_host_tensors():
    """R-50 at its config scale on a 1024^2 tile: the resize is the identity, no launch, the batch passes through"""
    tiles = torch.randint(0, 256, (2, 1024, 1024, 3), dtype=torch.uint8)
    data = P.run_test_pipeline(_cfg("orientedrepoints_r50_demo").test_pipeline, tiles, device=torch.device("cpu"))
    assert len(data["img"]) == 1 and data["img"][0].data_ptr() == tiles.data_ptr()
    assert data["valid_hw"][0].tolist() == [[1024, 1024]] * 2
    m = data["img_meta"][0]
    assert len(m) == 2 and m[0]["ori_shape"] == (1024, 1024, 3) and m[0]["scale_factor"] == 1.0 and m[0]["pad_shape"] == (1024, 1024, 3)
    assert set(m[0]) == {"filename", "ori_shape", "img_shape", "pad_shape", "scale_factor", "flip", "flip_direction", "img_norm_cfg"}


@pytest.mark.parametrize("cfg,what", [
    (dict(type="RotateResize", img_scale=(1333, 960), keep_ratio=False), "keep_ratio=False"),
    (dict(type="Resize", img_scale=(1333, 960), ratio_range=(0.5, 1.5)), "ratio_range"),
    (dict(type="RotateRandomFlip", direction=["vertical"]), "vertical"),
    (dict(type="RandomFlip", direction="vertical"), "vertical"),
])
def test_unsupported_transforms_raise(cfg, what):
    with pytest.raises(NotImplementedError, match=cfg["type"]):
        P.Compose([cfg])


def test_random_training_transforms_raise():
    with pytest.raises(NotImplementedError, match="RotateResize"):
        P.Compose([dict(type="RotateResize", img_scale=[(1333, 768), (1333, 1280)])])(dict(img_shape=(10, 10, 3)))
    with pytest.raises(NotImplementedError, match="RotateRandomFlip"):
        P.Compose([dict(type="RotateRandomFlip", flip_ratio=0.5)])(dict(img_shape=(10, 10, 3)))


@pytest.mark.parametrize("name", sorted(GOLD))
def test_configs_restate_the_reference_test_pipeline(name):
    m = _cfg(name)
    mine = json.loads(json.dumps(dict(img_norm_cfg=m.img_norm_cfg, test_pipeline=m.test_pipeline)))
    assert mine == GOLD[name]
    assert m.data["test"]["pipeline"] is m.test_pipeline
