"""GPU: the test pipeline on the device (datasets/pipelines.py, csrc/resize.cu) and what it feeds - the resize kernel
against cv2.resize bit for bit, the padded uint8 stems / Swin patch gather against the float path fed the host-normalised
zero-padded image, R-101 / Swin-T / R-50 at config scale against the fp64 graph, inference_detector with multi-scale + flip
against aug_test fed host-built views, detect_image(test_pipeline=...) against the file-based merge, and the conv launch
plans at the new input shapes against the parity cases of tests/test_conv_plans_gpu.py."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

MEAN = np.array([123.675, 116.28, 103.53], dtype=np.float32)
STDINV = (1.0 / np.array([58.395, 57.12, 57.375], dtype=np.float64)).astype(np.float32)
RESIZE_CASES = [((1024, 1024), (960, 960)), ((1024, 1024), (768, 768)), ((1024, 1024), (1280, 1280)),
                ((1024, 1024), (1000, 1000)), ((1024, 1024), (512, 512)), ((333, 517), (250, 388)), ((100, 77), (131, 203)),
                ((64, 64), (48, 48)), ((1, 50), (3, 70)), ((50, 1), (70, 3))]


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / (b.double().abs().max() + 1e-30))


def _host_view(img, scale, flip, div=32):
    """what the reference's pipeline makes of one HWC uint8 image on the host: cv2 resize, flip, zero pad; + the meta"""
    from orientedreppoints_b200.datasets.pipelines import rescale_size
    h, w = img.shape[:2]
    (nw, nh), sf = rescale_size((w, h), scale)
    r = cv2.resize(img, (nw, nh), interpolation=cv2.INTER_LINEAR)
    if flip:
        r = r[:, ::-1]
    ph, pw = -(-nh // div) * div, -(-nw // div) * div
    out = np.zeros((ph, pw, 3), np.uint8)
    out[:nh, :nw] = r
    return out, dict(img_shape=(nh, nw, 3), pad_shape=(ph, pw, 3), scale_factor=sf, flip=flip)


def _host_normalised(views_u8, shapes):
    """Normalize (to_rgb, (x - mean) * (1 / std) in fp32) then Pad with zeros, as float NCHW"""
    out = []
    for v, (h, w) in zip(views_u8, shapes):
        x = np.zeros(v.shape, np.float32)
        x[:h, :w] = (v[:h, :w, ::-1].astype(np.float32) - MEAN) * STDINV
        out.append(x)
    return torch.from_numpy(np.stack(out)).permute(0, 3, 1, 2).contiguous()


def _tiles(n, size=1024, seed=0):
    return np.random.RandomState(seed).randint(0, 256, (n, size, size, 3)).astype(np.uint8)


# ----------------------------------------------------------------------------------------------------------- kernel
@pytest.mark.parametrize("flip", [False, True])
@pytest.mark.parametrize("src,dst", RESIZE_CASES, ids=lambda v: "x".join(map(str, v)))
def test_resize_kernel_vs_cv2(cuda, src, dst, flip):
    from orientedreppoints_b200.datasets.pipelines import resize_u8
    img = np.random.RandomState(src[0] + dst[1]).randint(0, 256, (2,) + src + (3,)).astype(np.uint8)
    pad = (dst[0] + 5, dst[1] + 7)
    out = resize_u8(torch.from_numpy(img).to(cuda), dst, pad, flip).cpu().numpy()
    for i in range(2):
        ref = cv2.resize(img[i], (dst[1], dst[0]), interpolation=cv2.INTER_LINEAR)
        if flip:
            ref = ref[:, ::-1]
        assert np.array_equal(out[i, :dst[0], :dst[1]], ref)
    assert not out[:, dst[0]:].any() and not out[:, :, dst[1]:].any()


def test_resize_kernel_16_tile_batch(cuda):
    from orientedreppoints_b200.datasets.pipelines import resize_u8
    img = _tiles(16, seed=3)
    dev = torch.from_numpy(img).to(cuda)
    for flip in (False, True):
        out = resize_u8(dev, (960, 960), None, flip).cpu().numpy()
        for i in range(16):
            ref = cv2.resize(img[i], (960, 960), interpolation=cv2.INTER_LINEAR)
            assert np.array_equal(out[i], ref[:, ::-1] if flip else ref), (flip, i)


# ----------------------------------------------------------------------------------------------------- padded stems
@pytest.mark.parametrize("precision", ["bf16", "f16x3"])
def test_padded_stem_equals_float_path(cuda, precision):
    """odd valid widths / heights included: the pixel pair of the space-to-depth read is split at the extent"""
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    from orientedreppoints_b200.weights import random_state_dict
    det = OrientedRepPointsDetector(random_state_dict(50, seed=0, reference_init=False), 50, cuda, precision)
    u8 = np.random.RandomState(5).randint(0, 256, (3, 128, 160, 3)).astype(np.uint8)
    ext = [(117, 151), (128, 160), (64, 33)]
    valid = torch.tensor(ext, dtype=torch.int32).to(cuda)
    x = _host_normalised(u8, ext).to(cuda)
    a = det.eng.stem_u8(torch.from_numpy(u8).to(cuda), det.stem, det.img_norm_cfg, valid)
    b = det.eng.stem(x, det.stem)
    assert torch.equal(a, b)
    assert torch.equal(det.normalize(torch.from_numpy(u8).to(cuda), valid), x)       # the fp32 engine's masked Normalize


@pytest.mark.parametrize("precision", ["bf16", "f16x3"])
def test_padded_patch_embed_rows_equal_float_path(cuda, precision):
    from orientedreppoints_b200 import _lib
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    from orientedreppoints_b200.swin import random_swin_state_dict
    import ctypes
    det = OrientedRepPointsDetector(random_swin_state_dict(0), "swin_tiny", cuda, precision)
    sw = det.swin
    u8 = np.random.RandomState(6).randint(0, 256, (3, 96, 128, 3)).astype(np.uint8)
    ext = [(93, 127), (96, 128), (5, 2)]
    valid = torch.tensor(ext, dtype=torch.int32).to(cuda)
    x = _host_normalised(u8, ext).to(cuda)
    ra, rb = det.eng.alloc(3, 24, 32, 64), det.eng.alloc(3, 24, 32, 64)
    mean = (ctypes.c_float * 3)(*[float(v) for v in det.img_norm_cfg["mean"]])
    stdinv = (ctypes.c_float * 3)(*[1.0 / float(v) for v in det.img_norm_cfg["std"]])
    st = _lib.current_stream_ptr()
    _lib.check(sw._fn("patch_embed_rows_u8_padded")(_lib.ptr(torch.from_numpy(u8).to(cuda)), 3, 96, 128, mean, stdinv, 1,
                                                    _lib.ptr(valid), _lib.ptr(ra), st), "padded rows")
    _lib.check(sw._fn("patch_embed_rows")(_lib.ptr(x), 3, 96, 128, _lib.ptr(rb), st), "rows")
    assert torch.equal(ra, rb)
    fa = sw.forward(torch.from_numpy(u8).to(cuda), det.img_norm_cfg, valid)
    fb = sw.forward(x)
    for a, b in zip(fa, fb):
        assert torch.equal(det.eng.to_float(a), det.eng.to_float(b))


# ------------------------------------------------------------------------------------------------- config scale
def _fp64_dense(sd, depth, img):
    from oracle import torch_reference as tr
    from oracle import torch_swin as ts
    from orientedreppoints_b200.weights import STAGE_BLOCKS
    dev = img.device
    sdg = {k: v.to(dev).double() for k, v in sd.items()}
    with torch.no_grad():
        if depth == "swin_tiny":
            fpn = ts.swin_fpn(sdg, ts.swin_forward(sdg, img.double()))
            return [tr.head_single(sdg, f)[:3] for f in fpn], fpn
        return tr.forward_dense(sdg, img.double(), blocks=STAGE_BLOCKS[depth])


def _worst(det, outs, feats, ref_outs, ref_feats):
    worst = 0.0
    for lvl in range(5):
        worst = max(worst, _rel(det.eng.to_float(feats[lvl]).permute(0, 3, 1, 2), ref_feats[lvl]))
        for k in range(3):
            a, b = outs[lvl][k].permute(0, 3, 1, 2).double(), ref_outs[lvl][k]
            worst = max(worst, float((a - b).abs().max()) / max(1.0, float(b.abs().max())))
    return worst


def _sd(depth):
    if depth == "swin_tiny":
        from orientedreppoints_b200.swin import random_swin_state_dict
        return random_swin_state_dict(0)
    from orientedreppoints_b200.weights import random_state_dict
    # as tests/test_f16x3_gpu.py: randomised residual scales over R-101's 33 blocks would leave the fp16 range
    return random_state_dict(depth, seed=3, reference_init=False, residual_gain=1.0 if depth == 50 else 0.3)


def _pipeline(scale, flip=False):
    return [dict(type='LoadImageFromFile'),
            dict(type='MultiScaleFlipAug', img_scale=scale, flip=flip,
                 transforms=[dict(type='RotateResize', keep_ratio=True), dict(type='RotateRandomFlip'),
                             dict(type='Normalize', mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375], to_rgb=True),
                             dict(type='Pad', size_divisor=32), dict(type='ImageToTensor', keys=['img']),
                             dict(type='Collect', keys=['img'])])]


@pytest.mark.parametrize("depth,scale", [(101, (1333, 960)), ("swin_tiny", (1333, 960)), (50, (1333, 1000)), ("swin_tiny", (1333, 1000))],
                         ids=["r101-960", "swin-960", "r50-1000-padded", "swin-1000-padded"])
def test_config_scale_vs_fp64_graph(cuda, depth, scale):
    """1024^2 tile -> device pipeline -> f16x3 detector: dense outputs within 1e-4 of the fp64 graph run on the cv2-resized,
    host-normalised, zero-padded input; detections (rescale=True) equal the op-by-op post-processing mirror in tile
    coordinates.  (1333, 1000) resizes to 1000^2, padded to 1024^2."""
    from orientedreppoints_b200.core.get_bboxes import get_bboxes
    from orientedreppoints_b200.datasets.pipelines import run_test_pipeline
    from orientedreppoints_b200.detector import STRIDES, OrientedRepPointsDetector
    sd = _sd(depth)
    det = OrientedRepPointsDetector(sd, depth, cuda, "f16x3", test_cfg=dict(score_thr=0.0, max_per_img=300))
    det.eng.overflow_count()                                         # the counter is global: start from zero
    tile = _tiles(1, seed=11)
    data = run_test_pipeline(_pipeline(scale), torch.from_numpy(tile).to(cuda))
    (view,), (metas,), (valid,) = data["img"], data["img_meta"], data["valid_hw"]
    hv, meta = _host_view(tile[0], scale, False)
    assert np.array_equal(view[0].cpu().numpy(), hv)
    assert metas[0]["img_shape"] == meta["img_shape"] and metas[0]["pad_shape"] == meta["pad_shape"]
    assert metas[0]["scale_factor"] == meta["scale_factor"]
    outs, feats = det.forward_dense(view, valid)
    ref_outs, ref_feats = _fp64_dense(sd, depth, _host_normalised([hv], [meta["img_shape"][:2]]).to(cuda))
    worst = _worst(det, outs, feats, ref_outs, ref_feats)
    print("%s at %r: max rel err %.2e vs fp64" % (depth, scale, worst))
    assert worst < 1e-4
    assert det.eng.overflow_count() == 0
    det.forward_dense = lambda *a: (outs, feats)                     # freeze: GroupNorm sums use atomics
    dets = det.simple_test(view, metas, rescale=True, return_tensors=True, valid_hw=valid)
    mirror = get_bboxes([o[0] for o in outs], [o[2] for o in outs], STRIDES, metas, det.test_cfg, True)
    for (da, la), (db, lb) in zip(dets, mirror):
        assert da.shape == db.shape and torch.equal(la, lb)
        assert torch.allclose(da, db, rtol=1e-5, atol=1e-3)
    raw = det.simple_test(view, metas, rescale=False, return_tensors=True, valid_hw=valid)
    assert torch.allclose(dets[0][0][:, :26] * meta["scale_factor"], raw[0][0][:, :26], rtol=1e-5, atol=1e-3)


def test_graph_capture_with_extents(cuda):
    """the CUDA graph of the padded form replays with the extents copied into its static buffer"""
    from orientedreppoints_b200.datasets.pipelines import run_test_pipeline
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    det = OrientedRepPointsDetector(_sd(50), 50, cuda, "f16x3", test_cfg=dict(score_thr=0.0, max_per_img=100))
    data = run_test_pipeline(_pipeline((1333, 230)), torch.from_numpy(_tiles(2, 256, seed=4)).to(cuda))
    (view,), (metas,), (valid,) = data["img"], data["img_meta"], data["valid_hw"]
    assert tuple(view.shape) == (2, 256, 256, 3) and valid.tolist() == [[230, 230]] * 2
    eager, _ = det.forward_dense(view, valid)
    det.capture(view.shape, view.dtype, padded=True)
    assert det._graph_key(view, valid) == det._g_shape and det._graph_key(view, None) != det._g_shape
    graph, _ = det.forward_dense_graph(view, valid)
    for lvl in range(5):
        for k in range(3):
            assert _rel(graph[lvl][k], eager[lvl][k]) < 1e-5
    res = det.simple_test(view, metas, rescale=True, valid_hw=valid)
    assert len(res) == 2 and len(res[0]) == 15


# ---------------------------------------------------------------------------------------------- public interface
def _freeze_by_content(eng):
    """GroupNorm sums use atomics: evaluate every distinct (image, extents) once and hand both sides of a comparison the
    same dense outputs"""
    cache, real = {}, eng.forward_dense

    def key(img, valid):
        w = torch.arange(img.numel(), device=img.device, dtype=torch.int64) % 65521
        return (tuple(img.shape), int((img.reshape(-1).long() * w).sum()), None if valid is None else tuple(valid.reshape(-1).tolist()))

    def fwd(img, valid_hw=None):
        k = key(img, valid_hw)
        if k not in cache:
            cache[k] = real(img, valid_hw)
        return cache[k]
    eng.forward_dense = fwd
    return cache


def test_inference_detector_multiscale_flip_equals_aug_test(cuda):
    import importlib.util
    import os
    from orientedreppoints_b200.apis import init_detector, inference_detector
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("c", os.path.join(root, "configs", "dota", "orientedrepoints_r50_demo.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    scales = [(1333, 250), (1333, 196)]
    cfg = dict(model=m.model, test_cfg=dict(m.test_cfg, score_thr=0.0, max_per_img=200), img_norm_cfg=m.img_norm_cfg,
               data=dict(test=dict(pipeline=_pipeline(scales, flip=True))))
    model = init_detector(cfg, None, device=cuda)
    eng = model.engine()
    cache = _freeze_by_content(eng)
    img = np.random.RandomState(8).randint(0, 256, (300, 420, 3)).astype(np.uint8)
    res = inference_detector(model, img)
    assert len(cache) == 4                                           # two scales x (identity, flip)
    views, metas, valids = [], [], []
    for s in scales:
        for f in (False, True):
            v, meta = _host_view(img, s, f)
            views.append(torch.from_numpy(v)[None].to(cuda))
            metas.append([meta])
            valids.append(torch.tensor([meta["img_shape"][:2]], dtype=torch.int32).to(cuda))
    ref = eng.aug_test(views, metas, rescale=True, valid_hws=valids)
    assert len(cache) == 4                                           # host-built views are the device views, bit for bit
    assert len(res) == len(ref) == 15 and sum(len(r) for r in ref) > 0
    for a, b in zip(res, ref):
        assert np.array_equal(a, b)
    # a batch of two tiles sharing one shape: one result per tile
    both = inference_detector(model, np.stack([img, img]))
    assert len(both) == 2 and all(np.array_equal(a, b) for a, b in zip(both[1], res))


def test_detect_image_with_test_pipeline_equals_file_based_merge(cuda, tmp_path):
    from orientedreppoints_b200.datasets.pipelines import run_test_pipeline
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    from orientedreppoints_b200.dota import result_merge as rm
    from orientedreppoints_b200.dota.pipeline import DOTA_CLASSES, detect_image
    from orientedreppoints_b200.dota.split_tiles import split_image
    from orientedreppoints_b200.weights import random_state_dict
    det = OrientedRepPointsDetector(random_state_dict(50, seed=0, reference_init=True), 50, cuda, "bf16",
                                    test_cfg=dict(score_thr=0.0, max_per_img=60))
    img = np.random.RandomState(11).randint(0, 256, size=(420, 610, 3)).astype(np.uint8)
    pipe = _pipeline((1333, 200))
    tiles, names, _ = split_image(img, "P0042", 1, 256, 64, device=cuda)
    data = run_test_pipeline(pipe, tiles)
    assert tuple(data["img"][0].shape) == (6, 224, 224, 3) and data["img_meta"][0][0]["scale_factor"] == 200 / 256
    res = det.simple_test(data["img"][0], data["img_meta"][0], rescale=True, valid_hw=data["valid_hw"][0])
    calls = []

    def frozen(t, metas=None, rescale=False, valid_hw=None):
        calls.append((tuple(t.shape), rescale, valid_hw.tolist()))
        return res
    det.simple_test = frozen
    merged = detect_image(det, img, "P0042", 1, subsize=256, gap=64, batch=16, test_pipeline=pipe)
    assert calls == [((6, 224, 224, 3), True, [[200, 200]] * 6)]
    raw, out = tmp_path / "raw", tmp_path / "merged"
    rm.write_task1_raw(res, names, DOTA_CLASSES, str(raw))
    rm.mergebypoly(str(raw), str(out))
    total = 0
    for c in DOTA_CLASSES:
        lines = [l.rstrip("\n") for l in open(out / ("Task1_%s.txt" % c))]
        assert lines == merged[c], c
        total += len(lines)
    assert total > 0


# ------------------------------------------------------------------------------------------------ launch plans
# R-101 x4 and Swin-T x8 at 960 (their configs' test scale), R-50 views at 768 / 1280 (the training scale range's ends,
# typical multi-scale test views).  Every tensor-core launch plan is either pinned by a parity case of
# tests/test_conv_plans_gpu.py (PARITY) or, when it is not, its first production launch is replayed as a parity case with
# the production shapes (same Case harness: NaN-filled guarded outputs, launched twice, fp64 reference, plan asserted).
PIPE_WORKLOADS = [("r101", "f16x3", 4, (1333, 960)), ("swin_tiny", "f16x3", 8, (1333, 960)), ("r50", "f16x3", 1, (1333, 768)),
                  ("r50", "f16x3", 1, (1333, 1280))]


def _pipeline_plan_cases(cuda):
    """signature -> (case tuple of the first production launch with that plan, workloads that launch it)"""
    import test_conv_plans_gpu as cp
    from orientedreppoints_b200 import _lib
    from orientedreppoints_b200.bench_tile import build_detector
    from orientedreppoints_b200.datasets.pipelines import run_test_pipeline
    seen = {}
    for backbone, prec, batch, scale in PIPE_WORKLOADS:
        name = "%s %s x%d @%d" % (backbone, prec, batch, min(scale))
        _, det = build_detector(backbone, prec, cuda)
        eng = det.eng

        def note(case_of):
            def deco(fn):
                def wrapper(*a, **kw):
                    out = fn(*a, **kw)
                    sig = cp.signature(_lib.tc_last_plan())
                    if sig not in seen:
                        seen[sig] = ((sig, prec) + case_of(*a, **kw), set())
                    seen[sig][1].add(name)
                    return out
                return wrapper
            return deco

        def of_launch(xs, ys, tc, cout, kh, kw, cin, stride, pad, bias, relu, out_f32, deform, res=None, res32=None, offsets=None,
                      stats=None, masks=None):
            assert masks is None
            return ("deform" if deform else "conv", cin, cout, kh, stride, int(bias is not None), int(relu), int(bool(out_f32)),
                    1 if res is not None else (2 if res32 is not None else 0), int(stats is not None),
                    [tuple(x.shape[:3]) for x in xs])

        def of_splitk(x, y, tc, L, relu, ks, stats, f16x3):
            return ("conv", L.cin, L.cout, L.kh, L.stride, int(L.bias is not None), int(bool(relu)), 0, 0, int(stats is not None),
                    [tuple(x.shape[:3])])

        def of_stem(img, L, *a, **kw):
            n, h, w = (img.shape[0], img.shape[1], img.shape[2]) if img.dtype == torch.uint8 else (img.shape[0], img.shape[2], img.shape[3])
            return ("stem", 64, 64, 4, 1, 1, 1, 0, 0, 0, [(n, h, w)])
        eng._launch = note(of_launch)(eng._launch)
        eng._conv_splitk = note(of_splitk)(eng._conv_splitk)
        eng.stem = note(of_stem)(eng.stem)
        eng.stem_u8 = note(of_stem)(eng.stem_u8)
        tiles = torch.randint(0, 256, (batch, 1024, 1024, 3), generator=torch.Generator().manual_seed(1), dtype=torch.uint8)
        data = run_test_pipeline(_pipeline(scale), tiles.to(cuda))
        with torch.no_grad():
            det.forward_dense(data["img"][0], data["valid_hw"][0])
        torch.cuda.synchronize()
        del det, eng
        torch.cuda.empty_cache()
    return seen


def test_pipeline_shape_plans_vs_fp64(cuda):
    import test_conv_plans_gpu as cp
    from orientedreppoints_b200.engine_tc import EngineTC, EngineTCSplit
    seen = _pipeline_plan_cases(cuda)
    pinned = {c[0] for c in cp.PARITY}
    engines = {"f16x3": EngineTCSplit(cuda), "bf16": EngineTC(cuda)}
    checked = []
    for sig, (c, names) in sorted(seen.items(), key=lambda kv: str(kv[0])):
        print("%-7s %s  %s" % ("pinned" if sig in pinned else "checked", sig, ", ".join(sorted(names))))
        if sig in pinned:
            continue
        case = cp.Case(c, engines[c[1]], cuda, seed=sum(c[3:7]) + len(c[-1]))
        plan = cp._check_written_once(case)
        assert cp.signature(plan) == sig, "the replayed launch left its plan: %s" % dict(zip(cp.SIG_FIELDS, cp.signature(plan)))
        err = cp._check_values(case, plan)
        checked.append(sig)
        print("   %s %s: rel err %.2e (tol %.1e)" % (c[2], c[3:7], err, case.tol))
