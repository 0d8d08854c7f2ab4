"""GPU: HRNet + HRFPN on every engine -
- orp_hr_fuse / orp_hrfpn_reduce / orp_hrfpn_pool alone against fp64 at every launch shape of the HRNetV2p-W18 and W32 graphs
  at one 1024 tile, 16 tiles, two 512 tiles and one 960 tile (a 240 map: 15 at pool 16), fuse with 1, 2 and 3 upsampled
  sources, both poolings, in f16x3, bf16 and fp32;
- whole W18 / W32 graphs in f16x3 within 1e-4 of the fp64 graph (tests/hrnet_ref.py) with no f16x3 overflow, the fp32 engine
  within 1e-4, the bf16 levels within 0.06;
- CUDA-graph replay, a config-built HRNetV2p-W18 + HRFPN through init_detector with a checkpoint (simple_test, aug_test, uint8
  inference_detector);
- each entry point of include/orp_b200_hrnet.h on a side stream behind a long kernel and from two host threads."""
import os
import threading

import pytest
import torch
import torch.nn.functional as F

import hrnet_ref as hr

pytestmark = pytest.mark.gpu

TOL = 1e-4             # north_star: "within 1e-4 fp32"
BF16_TOL = 1.5e-2      # one bf16 rounding of inputs and output
F32_TOL = 2e-5
SPIN = 50_000_000      # torch.cuda._sleep cycles ahead of the inputs (tests/test_streams_gpu.py)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


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


def _seen(e, x_nhwc):
    """the fp64 values the engine holds for x"""
    return _from_engine(e, _to_engine(e, x_nhwc)).double()


def _precs(n):
    return ("f16x3",) if n == 16 else ("f16x3", "bf16", "fp32")   # the benchmark's batch runs f16x3


def _fuse_cases():
    shapes = sorted(set(hr.fuse_launches("hrnetv2p_w18")) | set(hr.fuse_launches("hrnetv2p_w32")))
    return [(prec, n, c, side * tile // 1024, nsrc) for n, tile in hr.BATCHES for c, side, nsrc in shapes for prec in _precs(n)]


@pytest.mark.parametrize("prec,n,c,h,nsrc", _fuse_cases(), ids=["%s-N%d-C%d-%d-src%d" % k for k in _fuse_cases()])
def test_fuse_launch_vs_fp64(cuda, prec, n, c, h, nsrc):
    """relu(base + sum_k nearest_up(src_k, 2^k)) against fp64 on the values the engine holds"""
    e = _engine(prec, cuda)
    g = torch.Generator(device=cuda).manual_seed(n + c + h + nsrc)
    base = torch.randn(n, h, h, c, device=cuda, generator=g)
    srcs = [torch.randn(n, h >> k, h >> k, c, device=cuda, generator=g) for k in range(1, nsrc + 1)]
    bs, ss = _to_engine(e, base), [_to_engine(e, s) for s in srcs]
    y = _from_engine(e, e.hr_fuse(bs, ss))
    ref = _seen(e, base)
    for k, s in enumerate(srcs, 1):
        ref = ref + _seen(e, s).repeat_interleave(2 ** k, 1).repeat_interleave(2 ** k, 2)
    ref = torch.relu(ref)
    err = _rel(y, ref)
    assert err < {"f16x3": TOL, "bf16": BF16_TOL, "fp32": F32_TOL}[prec], err
    if prec == "f16x3":
        assert e.overflow_count() == 0


def _map_cases():
    return [(prec, n, side, pool) for n, side in hr.pool_cases() for prec in _precs(n) for pool in ("AVG", "MAX")]


@pytest.mark.parametrize("prec,n,h,pool", _map_cases(), ids=["%s-N%d-%d-%s" % k for k in _map_cases()])
def test_reduce_and_pool_launches_vs_fp64(cuda, prec, n, h, pool):
    """orp_hrfpn_reduce (four fp32 parts, bilinear x2 / x4 / x8) and orp_hrfpn_pool (kernel = stride 2..16, floor) against
    F.interpolate / avg_pool2d / max_pool2d in fp64"""
    e = _engine(prec, cuda)
    g = torch.Generator(device=cuda).manual_seed(n + h)
    parts = [torch.randn(n, h >> i, h >> i, 256, device=cuda, generator=g) for i in range(4)]
    red = e.hrfpn_reduce(parts)
    want = sum(_nchw(p).double() if i == 0 else F.interpolate(_nchw(p).double(), scale_factor=2 ** i, mode='bilinear')
               for i, p in enumerate(parts))
    assert _rel(_nchw(_from_engine(e, red)), want) < {"f16x3": TOL, "bf16": BF16_TOL, "fp32": F32_TOL}[prec]
    levels = e.hrfpn_pool(red, pool == "MAX")
    x = _nchw(_from_engine(e, red)).double()
    fn = F.max_pool2d if pool == "MAX" else F.avg_pool2d
    for l, y in enumerate(levels, 1):
        ref = fn(x, 2 ** l, 2 ** l)
        got = _nchw(_from_engine(e, y))
        assert got.shape == ref.shape, (l, got.shape, ref.shape)
        tol = 0 if pool == "MAX" and prec != "bf16" else {"f16x3": TOL, "bf16": BF16_TOL, "fp32": F32_TOL}[prec]
        assert _rel(got, ref) <= tol, (l, _rel(got, ref))
    if prec == "f16x3":
        assert e.overflow_count() == 0


def test_launch_refusals(cuda):
    from orientedreppoints_b200 import _lib
    e = _engine("bf16", cuda)
    x = e.alloc(1, 8, 8, 24)
    with pytest.raises(_lib.OrpError, match="multiples of 2"):
        e.hr_fuse(e.alloc(1, 6, 6, 24), [e.alloc(1, 3, 3, 24)] * 2)
    with pytest.raises(_lib.OrpError, match="1..3 sources"):
        e.hr_fuse(x, [])
    with pytest.raises(_lib.OrpError, match="multiple of 8"):
        e.hrfpn_pool(e.alloc(1, 8, 8, 12), False)
    with pytest.raises(_lib.OrpError, match="multiples of 2"):
        e.hrfpn_reduce([torch.zeros(1, 6, 6, 8, device=cuda), torch.zeros(1, 3, 3, 8, device=cuda),
                        torch.zeros(1, 1, 1, 8, device=cuda)])


def _case(cuda, arch, n, h, w, seed, prec="f16x3", pooling="AVG", u8=False):
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    from orientedreppoints_b200.weights import random_hrnet_state_dict
    sd = random_hrnet_state_dict(arch, seed=0, reference_init=False, residual_gain=0.3)
    det = OrientedRepPointsDetector(sd, arch, cuda, prec, test_cfg=dict(score_thr=0.02), pooling_type=pooling)
    img = torch.randn(n, 3, h, w, generator=torch.Generator().manual_seed(seed)).to(cuda)
    outs, feats = det.forward_dense(img)
    torch.cuda.synchronize()
    if prec == "f16x3":
        assert det.eng.overflow_count() == 0
    sdg = {k: v.to(cuda).double() for k, v in sd.items()}
    with torch.no_grad():
        ref_outs, ref_feats = hr.forward_dense(sdg, img.double(), arch, pooling)
    errs = {}
    for lvl in range(5):
        errs["feat%d" % lvl] = _rel(_nchw(_from_engine(det.eng, feats[lvl])), ref_feats[lvl])
        for k, name in enumerate(("cls", "init", "refine")):
            a, b = _nchw(outs[lvl][k]), ref_outs[lvl][k]
            assert a.shape == b.shape
            errs["%s%d" % (name, lvl)] = float((a.double() - b).abs().max()) / max(1.0, float(b.abs().max()))
    return det, img, errs


@pytest.mark.parametrize("arch,n,size,pooling", [("hrnetv2p_w18", 1, 1024, "AVG"), ("hrnetv2p_w18", 2, 512, "MAX"),
                                                  ("hrnetv2p_w32", 1, 1024, "MAX"), ("hrnetv2p_w32", 2, 512, "AVG")])
def test_dense_graph_f16x3_vs_fp64(cuda, arch, n, size, pooling):
    """every HRFPN level and head output within 1e-4 of the fp64 graph; f16x3 overflow count 0"""
    _, _, errs = _case(cuda, arch, n, size, size, 11, pooling=pooling)
    print("f16x3 %s %dx%d^2 %s max rel err:" % (arch, n, size, pooling), max(errs.values()), errs)
    for k, v in errs.items():
        assert v < TOL, (k, v)


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_dense_graph_other_engines(cuda, prec):
    """W18 on the bf16 and fp32 engines: fp32 within 1e-4 of the fp64 graph; bf16 HRFPN levels within 0.06"""
    _, _, errs = _case(cuda, "hrnetv2p_w18", 2, 256, 320, 3, prec)
    print("%s W18 max rel err:" % prec, max(errs.values()), errs)
    for k, v in errs.items():
        if prec == "fp32":
            assert v < TOL, (k, v)
        elif k.startswith("feat"):
            assert v < 0.06, (k, v)


def test_graph_replay_matches_eager(cuda):
    """CUDA-graph capture of the W18 dense graph replays to the eager pass's results; one HRModule's fusion captured alone
    replays to its bits"""
    det, img, _ = _case(cuda, "hrnetv2p_w18", 2, 512, 512, 7)
    eager, _ = det.forward_dense(img)
    eager = [[t.clone() for t in lvl] for lvl in eager]
    det.capture(img.shape)
    outs, _ = det.forward_dense_graph(img)
    torch.cuda.synchronize()
    for lvl in range(5):
        for k in range(3):
            assert _rel(outs[lvl][k], eager[lvl][k]) < 1e-5, (lvl, k)     # the head's GroupNorm sums with atomics
    xs = det.hrnet.backbone(det._stem(img, None))
    fuse = det.hrnet.stages[2][0][1]
    want = [t.clone() for t in det.hrnet._fuse(xs, fuse)]
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ys = det.hrnet._fuse(xs, fuse)
    g.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(ys, want))


def test_init_detector_with_checkpoint(cuda, tmp_path):
    """the README's override: R-50 config with backbone / neck HRNetV2p-W18 + HRFPN(stride=2) from a checkpoint with the
    reference's keys: simple_test, aug_test and uint8 inference_detector"""
    import numpy as np
    from orientedreppoints_b200.apis import Config, inference_detector, init_detector
    from orientedreppoints_b200.hrnet import ARCHS
    from orientedreppoints_b200.weights import random_hrnet_state_dict
    cfg = Config.fromfile(os.path.join(ROOT, "configs", "dota", "orientedrepoints_r50_demo.py"))
    a = ARCHS["hrnetv2p_w18"]
    cfg['model']['backbone'] = dict(type='HRNet', extra=a.extra())
    cfg['model']['neck'] = dict(type='HRFPN', in_channels=list(a.out_widths), out_channels=256, stride=2)
    cfg['model']['pretrained'] = None
    cfg['test_cfg'] = dict(cfg['test_cfg'], score_thr=0.02)
    sd = random_hrnet_state_dict(a, seed=4, reference_init=False, residual_gain=0.3)
    ck = str(tmp_path / "hrnetv2p_w18.pth")
    torch.save(dict(state_dict=sd), ck)
    model = init_detector(cfg, ck, device=str(cuda))
    assert model.engine().hr_arch.stages == a.stages and model.engine().pooling_type == 'AVG'
    img = torch.randn(1, 3, 256, 256, generator=torch.Generator().manual_seed(3)).to(cuda)
    res = model(img, [dict(scale_factor=1.0)], return_loss=False, rescale=True)
    assert len(res) == 1 and len(res[0]) == 15 and sum(len(r) for r in res[0]) > 0
    metas = [[dict(img_shape=(256, 256, 3), scale_factor=1.0, flip=False)], [dict(img_shape=(256, 256, 3), scale_factor=1.0, flip=True)]]
    aug = model.aug_test([img, img.flip(-1)], metas, rescale=True)
    assert len(aug) == 15 and sum(len(r) for r in aug) > 0
    u8 = np.random.RandomState(0).randint(0, 256, (300, 410, 3)).astype(np.uint8)
    res = inference_detector(model, u8)
    assert len(res) == 15 and all(r.ndim == 2 for r in res)
    assert model.engine().eng.overflow_count() == 0


def _entry_calls(cuda):
    """per entry point of orp_b200_hrnet.h: (name, input, run(input) -> output)"""
    out = []
    g = torch.Generator().manual_seed(9)
    for prec in ("bf16", "f16x3", "fp32"):
        e = _engine(prec, cuda)
        srcs = [_to_engine(e, torch.randn(2, 64 >> k, 64 >> k, 40, generator=g).to(cuda)) for k in (1, 2)]
        base = _to_engine(e, torch.randn(2, 64, 64, 40, generator=g).to(cuda))
        sfx = "f32" if prec == "fp32" else prec
        out.append(("orp_hr_fuse_" + sfx, base, lambda x, e=e, s=srcs: e.hr_fuse(x, s)))
        parts = [torch.randn(2, 64 >> i, 64 >> i, 256, generator=g).to(cuda) for i in range(4)]
        out.append(("orp_hrfpn_reduce_" + sfx, parts[0], lambda x, e=e, p=parts: e.hrfpn_reduce([x] + p[1:])))
        red = _to_engine(e, torch.randn(2, 48, 48, 256, generator=g).to(cuda))
        out.append(("orp_hrfpn_pool_" + sfx, red, lambda x, e=e: torch.cat([t.flatten() for t in e.hrfpn_pool(x, True)] +
                                                                          [t.flatten() for t in e.hrfpn_pool(x, False)])))
    return out


def test_entry_points_on_a_side_stream_and_two_threads(cuda):
    """each entry point on a PyTorch side stream behind a long kernel, with its input written after the spin into a NaN
    buffer, gives the default stream's bits; two host threads calling it at once both do too"""
    from orientedreppoints_b200 import _lib
    calls = _entry_calls(cuda)
    assert sorted(c[0] for c in calls) == sorted(_lib.HRNET_SIGNATURES)
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
