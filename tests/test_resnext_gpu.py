"""GPU: the ResNeXt backbones (resnext.py) on every engine -
- every grouped conv2 launch of X-50/101/152 32x4d, 64x4d and 32x8d alone against F.conv2d(groups=) in fp64, at one 1024 tile,
  16 tiles and two 512 tiles, plus M-tile tails and odd stride-2 sizes, in f16x3, bf16 and fp32;
- whole X-50-32x4d, X-101-64x4d, X-50-32x8d and X-152-32x4d graphs in f16x3 within 1e-4 of the fp64 graph
  (tests/resnext_ref.py), and X-50-32x4d on the bf16 / fp32 engines;
- CUDA-graph capture, aug_test, a config-built model through init_detector with a checkpoint file;
- each entry point of include/orp_b200_group.h on a side stream behind a long kernel and from two host threads."""
import ctypes
import threading

import pytest
import torch
import torch.nn.functional as F

import resnext_ref as xr

pytestmark = pytest.mark.gpu

TOL = 1e-4             # north_star: "within 1e-4 fp32"
BF16_TOL = 1.5e-2      # the bf16 per-launch tolerance of tests/test_dcn_backbone_gpu.py (fp64 on bf16-rounded operands)
F32_TOL = 2e-5         # fp32 CUDA-core FMAs
SPIN = 50_000_000      # torch.cuda._sleep cycles ahead of the inputs (tests/test_streams_gpu.py)


def _nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / (b.double().abs().max() + 1e-30))


def _engine(prec, cuda):
    from orientedreppoints_b200.detector import EngineF32
    from orientedreppoints_b200.engine_tc import EngineTC, EngineTCSplit
    return {"f16x3": EngineTCSplit, "bf16": EngineTC, "fp32": EngineF32}[prec](cuda)


def _to_engine(e, x_nhwc):
    if e.name == "f16x3":
        return e.from_float(x_nhwc)
    return x_nhwc.to(e.device, e.act_dtype).contiguous()


def _from_engine(e, y):
    return e.to_float(y) if e.name == "f16x3" else y.float()


def _launch_cases():
    shapes = sorted({l for _, _, g, b in xr.MODELS for l in xr.group_launches(g, b)})
    out = []
    for n, tile in xr.BATCHES:
        for width, groups, h, s in shapes:
            for prec in ("f16x3", "bf16", "fp32"):
                if n == 16 and prec != "f16x3":
                    continue                       # the benchmark's batch runs f16x3
                out.append((prec, n, width, groups, h * tile // 1024, h * tile // 1024, s))
    # M-tile tails (pixel counts that leave the last 128-pixel tile partly empty) and odd stride-2 inputs
    for prec in ("f16x3", "bf16", "fp32"):
        for width, groups in ((128, 32), (256, 64), (512, 32), (2048, 32)):
            out += [(prec, 3, width, groups, 13, 11, 1), (prec, 1, width, groups, 33, 47, 2), (prec, 2, width, groups, 7, 5, 2)]
    return out


def _group_layer(width, groups, s, cuda, g):
    from orientedreppoints_b200.detector import ConvLayer
    gw = width // groups
    wt = torch.randn(width, gw, 3, 3, generator=g) * (2.0 / (9 * gw)) ** 0.5
    b = torch.randn(width, generator=g) * 0.1
    return wt, b, ConvLayer(wt, b, s, 1, cuda)


@pytest.mark.parametrize("prec,n,width,groups,h,w,s", _launch_cases(), ids=["%s-N%d-C%d-g%d-%dx%d-s%d" % c for c in _launch_cases()])
def test_group_launch_vs_fp64(cuda, prec, n, width, groups, h, w, s):
    """one grouped conv2 as the engine runs it (folded-BN weight and bias, ReLU, activation format out) against
    F.conv2d(groups=) in fp64 on the device"""
    e = _engine(prec, cuda)
    g = torch.Generator().manual_seed(width + groups + h + w + s + n)
    x = torch.relu(torch.randn(n, width, h, w, generator=g))
    wt, b, L = _group_layer(width, groups, s, cuda, g)
    xr_, wr = (x.bfloat16().double(), wt.bfloat16().double()) if prec == "bf16" else (x.double(), wt.double())
    with torch.no_grad():
        ref = torch.relu(F.conv2d(xr_.to(cuda), wr.to(cuda), b.double().to(cuda), s, 1, groups=groups))
    y = e.group_conv(_to_engine(e, x.permute(0, 2, 3, 1).contiguous().to(cuda)), L, groups, relu=True)
    assert tuple(y.shape[:3]) == tuple(ref.shape[:1]) + tuple(ref.shape[2:])
    err = _rel(_nchw(_from_engine(e, y)), ref)
    print("%s N%d C%d g%d %dx%d s%d: rel err %.2e" % (prec, n, width, groups, h, w, s, err))
    assert err < {"f16x3": TOL, "bf16": BF16_TOL, "fp32": F32_TOL}[prec], err
    if prec == "f16x3":
        assert e.overflow_count() == 0


def _case(cuda, depth, groups, base_width, n, h, w, seed, prec="f16x3", gain=1.0):
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    from orientedreppoints_b200.weights import random_state_dict
    sd = random_state_dict(depth, seed=0, reference_init=False, residual_gain=gain, groups=groups, base_width=base_width)
    det = OrientedRepPointsDetector(sd, depth, cuda, prec, test_cfg=dict(score_thr=0.02))
    assert det.groups == groups
    img = torch.randn(n, 3, h, w, generator=torch.Generator().manual_seed(seed)).to(cuda)
    outs, feats = det.forward_dense(img)
    torch.cuda.synchronize()
    if prec == "f16x3":
        assert det.eng.overflow_count() == 0
    sdg = {k: v.to(cuda).double() for k, v in sd.items()}
    with torch.no_grad():
        ref_outs, ref_feats = xr.forward_dense(sdg, img.double(), depth, groups)
    errs = {}
    for lvl in range(5):
        errs["feat%d" % lvl] = _rel(_nchw(_from_engine(det.eng, feats[lvl])), ref_feats[lvl])
        for k, name in enumerate(("cls", "init", "refine")):
            a, b = _nchw(outs[lvl][k]), ref_outs[lvl][k]
            assert a.shape == b.shape
            errs["%s%d" % (name, lvl)] = float((a.double() - b).abs().max()) / max(1.0, float(b.abs().max()))
    return det, img, outs, ref_outs, errs


# residual_gain 0.3 for the deep models, as the R-101 tests use (1.0 doubles the activation variance per block)
@pytest.mark.parametrize("depth,groups,base_width,n,size,gain", [(50, 32, 4, 1, 1024, 1.0), (50, 32, 4, 2, 512, 1.0),
                                                                 (101, 64, 4, 1, 1024, 0.3), (101, 64, 4, 2, 512, 0.3),
                                                                 (50, 32, 8, 1, 512, 1.0), (152, 32, 4, 1, 512, 0.3)])
def test_dense_graph_f16x3_vs_fp64(cuda, depth, groups, base_width, n, size, gain):
    """every FPN level and head output within 1e-4 of the fp64 graph; f16x3 overflow count 0"""
    _, _, _, _, errs = _case(cuda, depth, groups, base_width, n, size, size, 11, gain=gain)
    print("f16x3 X-%d-%dx%dd %dx%d^2 max rel err:" % (depth, groups, base_width, n, size), max(errs.values()), errs)
    for k, v in errs.items():
        assert v < TOL, (k, v)


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_dense_graph_other_engines(cuda, prec):
    """X-50-32x4d on the bf16 and fp32 engines: fp32 within 1e-4 of the fp64 graph; bf16 FPN levels within the 0.06 of
    tests/test_dense_gpu.py::test_dense_graph_bf16_vs_f32_engine"""
    _, _, _, _, errs = _case(cuda, 50, 32, 4, 2, 256, 320, 3, prec)
    print("%s X-50-32x4d max rel err:" % prec, max(errs.values()), errs)
    for k, v in errs.items():
        if prec == "fp32":
            assert v < TOL, (k, v)
        elif k.startswith("feat"):
            assert v < 0.06, (k, v)


def test_graph_replay_matches_eager(cuda):
    """CUDA-graph capture of the X-50-32x4d dense graph; a grouped conv2 captured alone replays to the eager pass's bits"""
    det, img, _, _, _ = _case(cuda, 50, 32, 4, 2, 512, 512, 7)
    eager, _ = det.forward_dense(img)
    eager = [[t.clone() for t in lvl] for lvl in eager]
    det.capture(img.shape)
    outs, _ = det.forward_dense_graph(img)
    torch.cuda.synchronize()
    for lvl in range(5):
        for k in range(3):
            assert _rel(outs[lvl][k], eager[lvl][k]) < 1e-5, (lvl, k)
    blk = det.blocks[2][0]
    x = det.eng.from_float(torch.relu(torch.randn(2, 64, 64, 512, generator=torch.Generator().manual_seed(2))).to(cuda))
    want = det._conv2(x, blk).clone()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = det._conv2(x, blk)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(y, want)


def test_aug_test_and_init_detector_with_checkpoint(cuda, tmp_path):
    """the README's override: a config-built X-101-64x4d detector loaded from a checkpoint file through init_detector runs
    simple_test and aug_test, and its engine takes the groups from the checkpoint's shapes"""
    import os
    from orientedreppoints_b200.apis import Config, init_detector
    from orientedreppoints_b200.weights import random_state_dict
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = Config.fromfile(os.path.join(root, "configs", "dota", "orientedrepoints_r50_demo.py"))
    cfg['model']['backbone'] = dict(cfg['model']['backbone'], type='ResNeXt', depth=101, groups=64, base_width=4)
    cfg['model']['pretrained'] = None
    cfg['test_cfg'] = dict(cfg['test_cfg'], score_thr=0.02)
    sd = random_state_dict(101, seed=4, reference_init=False, residual_gain=0.3, groups=64, base_width=4)
    ck = str(tmp_path / "x101_64x4d.pth")
    torch.save(dict(state_dict=sd), ck)
    model = init_detector(cfg, ck, device=str(cuda))
    assert model.engine().groups == 64 and model.backbone.layer1[0].conv2.groups == 64
    img = torch.randn(1, 3, 256, 256, generator=torch.Generator().manual_seed(3)).to(cuda)
    res = model(img, [dict(scale_factor=1.0)], return_loss=False, rescale=True)
    assert len(res) == 1 and len(res[0]) == 15 and sum(len(a) for a in res[0]) > 0
    metas = [[dict(img_shape=(256, 256, 3), scale_factor=1.0, flip=False)], [dict(img_shape=(256, 256, 3), scale_factor=1.0, flip=True)]]
    aug = model.aug_test([img, img.flip(-1)], metas, rescale=True)
    assert len(aug) == 15 and sum(len(a) for a in aug) > 0
    assert model.engine().eng.overflow_count() == 0


def _entry_calls(cuda):
    """per entry point of orp_b200_group.h: (name, make(): (inputs, run(inputs) -> output))"""
    from orientedreppoints_b200 import _lib
    from orientedreppoints_b200.engine_tc import EngineTC, EngineTCSplit
    g = torch.Generator().manual_seed(9)
    wt, b, L = _group_layer(256, 32, 2, cuda, g)
    x = torch.relu(torch.randn(2, 56, 56, 256, generator=g)).to(cuda)
    out = []
    for prec, E in (("bf16", EngineTC), ("f16x3", EngineTCSplit)):
        e = E(cuda)
        xe = _to_engine(e, x)

        def run(xin, e=e):
            return e.group_conv(xin, L, 32, relu=True)
        out.append(("orp_group_conv2d_" + prec, xe, run))

    def run32(xin):
        y = torch.empty((2, 28, 28, 256), device=cuda)
        _lib.check(_lib.lib().orp_group_conv2d_f32(_lib.ptr(xin), 2, 56, 56, 256, 32, _lib.ptr(L.w), 2, _lib.ptr(L.bias), 1,
                                                   _lib.ptr(y), _lib.current_stream_ptr()), "orp_group_conv2d_f32")
        return y
    out.append(("orp_group_conv2d_f32", x, run32))
    return out


def test_entry_points_on_a_side_stream_and_two_threads(cuda):
    """each entry point on a PyTorch side stream behind a long kernel, with its input written after the spin into a NaN
    buffer, gives the default stream's bits; two host threads calling it at once both do too"""
    from orientedreppoints_b200 import _lib
    calls = _entry_calls(cuda)
    assert sorted(c[0] for c in calls) + ["orp_tc_plan_group_conv"] == sorted(_lib.GROUP_SIGNATURES)
    for name, xin, run in calls:
        want = run(xin).clone()
        torch.cuda.synchronize()
        side = torch.cuda.Stream(device=cuda)
        buf = torch.full_like(xin, float("nan"))
        with torch.cuda.stream(side):
            torch.cuda._sleep(SPIN)
            buf.copy_(xin)
            got = run(buf)
        side.synchronize()
        assert torch.equal(got, want), name
        res, errs = [None, None], []

        def worker(i):
            try:
                st = torch.cuda.Stream(device=cuda)
                with torch.cuda.device(cuda), torch.cuda.stream(st):
                    for _ in range(3):
                        res[i] = run(xin)
                    st.synchronize()
            except Exception as exc:                       # reported below
                errs.append(exc)
        th = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        assert not errs, errs
        assert torch.equal(res[0], want) and torch.equal(res[1], want), name


def test_timing_counts_useful_flops(cuda):
    """orp_tc_timing_collect counts 2 * Ho*Wo*N * width * 9 * gw for a grouped launch"""
    from orientedreppoints_b200 import _lib
    e = _engine("f16x3", cuda)
    _, _, L = _group_layer(512, 32, 1, cuda, torch.Generator().manual_seed(1))
    x = e.from_float(torch.relu(torch.randn(2, 40, 40, 512)).to(cuda))
    _lib.set_timing(True)
    try:
        _lib.tc_timing_collect()
        e.group_conv(x, L, 32, relu=True)
        ms, n, fl = _lib.tc_timing_collect()
    finally:
        _lib.set_timing(False)
    assert n == 1 and ms > 0 and fl == 2.0 * 2 * 40 * 40 * 512 * 9 * 16
    p = _lib.tc_last_plan()
    assert p["BN"] == 64 and p["n_tiles_n"] == 8 and p["split"] == 1
    assert ctypes.sizeof(_lib.TcPlan) > 0
