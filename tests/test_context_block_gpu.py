"""Global context blocks on the H100 (include/orp_b200_context.h): every pool, transform and fuse launch of the golden backbones'
layouts at 16 x 1024^2 and 4 x 960^2 against the fp64 contract in all three formats, a peaked softmax, a uniform mask against
'avg', every (pooling x fusion) as a whole block, the golden backbones (R-50 r16 / r4 'avg' add + mul, X-50-32x4d, R-50-DCNv2,
R-50 + GA) as whole graphs against fp64, bitwise reproducibility, CUDA-graph capture, aug_test at two scales, init_detector
from a checkpoint with the reference's keys, the entry points on a side stream and two host threads each running a detector,
and the launch checker of tests/test_backbone_launches_gpu.py over R-50-GCB c3-c5."""
import ctypes
import threading
import time

import pytest
import torch

from orientedreppoints_b200 import _lib
from orientedreppoints_b200 import context_block as cb
from orientedreppoints_b200.detector import EngineF32, OrientedRepPointsDetector
from orientedreppoints_b200.weights import gcb_layout, gcb_spec, random_state_dict
import context_block_ref as cr
from test_context_block_cpu import BACKBONES, FUSIONS, GCB_PARITY, POOLS, backbone_case

pytestmark = pytest.mark.gpu
FORMATS = ["f16x3", "bf16", "fp32"]
C3_C5 = (False, True, True, True)
R16 = dict(ratio=1. / 16.)
R4_AVG = dict(ratio=1. / 4., pooling_type='avg', fusion_types=('channel_add', 'channel_mul'))


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    d = torch.device("cuda", 0)
    torch.cuda.set_device(d)
    return d


def _engine(fmt, dev):
    if fmt == "fp32":
        return EngineF32(dev)
    from orientedreppoints_b200.engine_tc import EngineTC, EngineTCSplit
    return EngineTCSplit(dev) if fmt == "f16x3" else EngineTC(dev)


def _held(e, t):
    """t (fp32 NHWC on the device) in the engine's format, and the exact values it holds (fp64)"""
    if e.name == "fp32":
        y = t.contiguous()
        return y, y.double()
    y = e.from_float(t)
    return y, e.to_float(y).double()


def _f(e, y):
    return (y if e.name == "fp32" else e.to_float(y)).double()


def _block(cfg, c, seed, dev, mask_scale=None):
    """(engine block, fp64 params, spec) of layer (c)'s block 0 with every term acting; mask_scale rescales conv_mask"""
    li = (256, 512, 1024, 2048).index(c)
    stages = [False] * 4
    stages[li] = True
    sd = random_state_dict(50, seed=seed, reference_init=False, gcb=cfg, stage_with_gcb=stages, gcb_gain=1.0)
    p = "backbone.layer%d.0" % (li + 1)
    if mask_scale is not None and cfg.get('pooling_type', 'att') == 'att':
        sd[p + ".context_block.conv_mask.weight"] = sd[p + ".context_block.conv_mask.weight"] * mask_scale
    spec = gcb_spec(cfg, c)
    return cb.ContextBlock(sd, p, spec, dev), {k: v.double().to(dev) for k, v in cr.block_params(sd, p).items()}, spec


def _contract(spec, p64, x64, idt64):
    """fp64: (mul, add, relu(x * mul + add + identity)) on NHWC inputs"""
    mul, add = cr.terms(spec, p64, x64.permute(0, 3, 1, 2))
    y = x64 * (mul[:, None, None, :] if mul is not None else 1.0) + (add[:, None, None, :] if add is not None else 0.0) + idt64
    return mul, add, torch.relu(y)


def _launches(e, blk, xd, idd):
    """the three launches of a block call, with the rows kept: (mul, add, y)"""
    n, h, w, c = cb.dims(e, xd)
    plan = _lib.context_plan_for(e.name, n, h, w, c)
    ws = torch.full((plan["workspace_bytes"] // 4,), float("nan"), device=xd.device)
    lib, st = _lib.lib(), _lib.current_stream_ptr()
    fn = "orp_context_pool_" + cb._SUFFIX[e.name]
    _lib.check(getattr(lib, fn)(_lib.ptr(xd), n, h, w, c, _lib.ptr(blk.mask_w), _lib.ptr(ws), ws.numel() * 4, st), fn)
    rows = {f: torch.full((n, c), float("nan"), device=xd.device) for f in blk.mlps}
    add, mul = blk.mlps.get('channel_add'), blk.mlps.get('channel_mul')
    _lib.check(lib.orp_context_transform(_lib.ptr(ws), n, plan["chunks"], c, blk.planes, ctypes.byref(add[0]) if add else None,
                                         ctypes.byref(mul[0]) if mul else None, _lib.ptr(rows.get('channel_add')),
                                         _lib.ptr(rows.get('channel_mul')), st), "orp_context_transform")
    y = cb.alloc(e, n, h, w, c)
    fn = "orp_context_fuse_" + cb._SUFFIX[e.name]
    _lib.check(getattr(lib, fn)(_lib.ptr(xd), _lib.ptr(idd), n, h, w, c, _lib.ptr(rows.get('channel_mul')),
                                _lib.ptr(rows.get('channel_add')), _lib.ptr(y), st), fn)
    return rows.get('channel_mul'), rows.get('channel_add'), y


def _rel(a, b):
    return float((a.double() - b).abs().max() / b.abs().max())


def _check_launches(e, blk, p64, spec, x, idt, y_tol=None):
    if e.name == "f16x3":
        e.overflow_count()                                              # the counter is one per process: start from zero
    xd, x64 = _held(e, x)
    idd, i64 = _held(e, idt)
    mul, add, y = _launches(e, blk, xd, idd)
    rmul, radd, ry = _contract(spec, p64, x64, i64)
    for got, ref in ((mul, rmul), (add, radd)):
        assert (got is None) == (ref is None)
        if ref is not None:
            assert _rel(got, ref) < 1e-4, _rel(got, ref)             # fp32 arithmetic on the held inputs in every format
    tol = y_tol or (1e-2 if e.name == "bf16" else 1e-4)
    assert _rel(_f(e, y), ry) < tol, _rel(_f(e, y), ry)
    if e.name == "f16x3":
        assert e.overflow_count() == 0
    return mul, add, y


# the layouts of the golden backbones: (cfg) x the stage maps of 16 x 1024^2 and 4 x 960^2
LAUNCHES = [(n, tile // (4 << li), 256 << li) for n, tile in ((16, 1024), (4, 960)) for li in (1, 2, 3)]


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("cfg", [R16, R4_AVG], ids=["att_add_r16", "avg_add_mul_r4"])
@pytest.mark.parametrize("n, h, c", LAUNCHES)
def test_launches_vs_fp64(dev, fmt, cfg, n, h, c):
    e = _engine(fmt, dev)
    blk, p64, spec = _block(cfg, c, seed=h + c, dev=dev)
    g = torch.Generator(device=dev).manual_seed(n * h + c)
    x = torch.randn(n, h, h, c, device=dev, generator=g)
    idt = torch.randn(n, h, h, c, device=dev, generator=g)
    _check_launches(e, blk, p64, spec, x, idt)


@pytest.mark.parametrize("fmt", ["f16x3", "fp32"])
def test_peaked_softmax(dev, fmt):
    """one pixel's logit ~80 above the rest: the context is that pixel's x"""
    e = _engine(fmt, dev)
    blk, p64, spec = _block(R16, 1024, seed=3, dev=dev)
    g = torch.Generator(device=dev).manual_seed(5)
    x = torch.randn(2, 33, 31, 1024, device=dev, generator=g)
    w = blk.mask_w
    x[:, 17, 9] += 80.0 * w / float((w * w).sum())
    logit = (x @ w)
    assert float((logit[:, 17, 9] - logit.flatten(1).sort(1).values[:, -2]).min()) > 70
    _check_launches(e, blk, p64, spec, x, torch.randn(2, 33, 31, 1024, device=dev, generator=g))


@pytest.mark.parametrize("fmt", FORMATS)
def test_uniform_mask_is_avg(dev, fmt):
    """a zero conv_mask weight (the bias alone, which cancels) gives every pixel the same weight: the 'avg' pooling"""
    e = _engine(fmt, dev)
    att, p64, spec = _block(dict(R4_AVG, pooling_type='att'), 512, seed=7, dev=dev, mask_scale=0.0)
    li = 1
    sd = random_state_dict(50, seed=7, reference_init=False, gcb=dict(R4_AVG, pooling_type='att'), stage_with_gcb=(False, True, False, False),
                           gcb_gain=1.0)
    for k in [k for k in sd if "conv_mask" in k]:
        del sd[k]
    avg = cb.ContextBlock(sd, "backbone.layer%d.0" % (li + 1), gcb_spec(R4_AVG, 512), dev)
    assert float(p64['conv_mask.bias'].abs().max()) > 0                     # the bias is drawn and does not matter
    g = torch.Generator(device=dev).manual_seed(8)
    x, idt = torch.randn(3, 21, 19, 512, device=dev, generator=g), torch.randn(3, 21, 19, 512, device=dev, generator=g)
    ma, aa, ya = _check_launches(e, att, p64, spec, x, idt)
    p_avg = {k: v for k, v in p64.items() if "conv_mask" not in k}
    mv, av, yv = _check_launches(e, avg, p_avg, gcb_spec(R4_AVG, 512), x, idt)
    assert torch.allclose(ma, mv, rtol=0, atol=1e-6) and torch.allclose(aa, av, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("pool", POOLS)
@pytest.mark.parametrize("fus", FUSIONS, ids=["add", "mul", "add_mul"])
def test_block_every_combination(dev, fmt, pool, fus):
    """ContextBlock as the detector calls it, against context_block_ref.block + identity, ReLU; odd map, N = 3"""
    e = _engine(fmt, dev)
    cfg = dict(ratio=1. / 4., pooling_type=pool, fusion_types=fus)
    blk, p64, spec = _block(cfg, 256, seed=11, dev=dev)
    g = torch.Generator(device=dev).manual_seed(3)
    xd, x64 = _held(e, torch.randn(3, 11, 14, 256, device=dev, generator=g))
    idd, i64 = _held(e, torch.randn(3, 11, 14, 256, device=dev, generator=g))
    y = _f(e, blk(e, xd, idd))
    ref = torch.relu(cr.block(spec, p64, x64.permute(0, 3, 1, 2)).permute(0, 2, 3, 1) + i64)
    assert float((y - torch.relu(x64 + i64)).abs().max()) > 0.05       # the block acts
    assert _rel(y, ref) < (1e-2 if fmt == "bf16" else 1e-4), _rel(y, ref)


def _graph_case(tag, fmt, dev, size=128, n=2):
    from test_gen_attention_gpu import _tame
    sd, lay, depth, groups, dl, gal = backbone_case(tag)
    if gal is not None:
        _tame(sd)
    det = OrientedRepPointsDetector(sd, depth, dev, fmt, dcn=dl, gen_attention=gal, gcb=lay)
    img = torch.randn(n, 3, size, size, generator=torch.Generator().manual_seed(4))
    return det, sd, img, (lay, depth, groups, dl, gal)


@pytest.mark.parametrize("tag", sorted(BACKBONES))
@pytest.mark.parametrize("fmt", ["f16x3", "fp32"])
def test_whole_graph_vs_fp64(dev, tag, fmt):
    det, sd, img, (lay, depth, groups, dl, gal) = _graph_case(tag, fmt, dev)
    if fmt == "f16x3":
        det.eng.overflow_count()
    outs, feats = det.forward_dense(img.to(dev))
    rdev = dev if gal is None else torch.device("cpu")                 # tests/gen_attention_ref.py evaluates on the host
    sd64 = {k: v.double().to(rdev) for k, v in sd.items()}
    ref_outs, ref_feats = cr.forward_dense(sd64, img.double().to(rdev), lay, depth, groups, dl, gal)
    ref_outs = [[r.to(dev) for r in o] for o in ref_outs]
    ref_feats = [f.to(dev) for f in ref_feats]
    for f, r in zip(feats, ref_feats):
        got = _f(det.eng, f).permute(0, 3, 1, 2)
        assert _rel(got, r) < 1e-4, _rel(got, r)
    for (c, i, rf), (rc, ri, rr) in zip(outs, ref_outs):          # head outputs as tests/test_dcn_backbone_gpu.py measures them
        for a, b in ((c, rc), (i, ri), (rf, rr)):
            a = a.double().permute(0, 3, 1, 2)
            assert float((a - b).abs().max()) / max(1.0, float(b.abs().max())) < 1e-4
    if fmt == "f16x3":
        assert det.eng.overflow_count() == 0
    assert len(det.simple_test(img.to(dev), rescale=False)) == 2


def _gcb_outputs(monkeypatch):
    """every context block output of the calls that follow, cloned, in call order"""
    got, real = [], cb.ContextBlock.__call__

    def recording(blk, eng, x, identity):
        y = real(blk, eng, x, identity)
        got.append(y.clone())
        return y
    monkeypatch.setattr(cb.ContextBlock, "__call__", recording)
    return got


def _same(fmt, a, b):
    """bitwise for the tensor-core engines; the fp32 engine's GroupNorm statistics (neck and head) accumulate with atomics, so
    its FPN levels agree to rounding only"""
    return torch.equal(a, b) if fmt != "fp32" else torch.allclose(a, b, rtol=1e-5, atol=1e-5 * float(a.abs().max()))


@pytest.mark.parametrize("fmt", FORMATS)
def test_two_runs_bitwise_equal(dev, monkeypatch, fmt):
    det, sd, img, _ = _graph_case("r50_avg_r4", fmt, dev, size=256)
    img = img.to(dev)
    rec = _gcb_outputs(monkeypatch)
    a = [t.clone() for t in det.forward_dense(img)[1]]
    first = list(rec)
    rec.clear()
    b = det.forward_dense(img)[1]
    assert len(first) == len(rec) == 13
    for x, y in zip(first, rec):                                       # the context blocks: bitwise in every format
        assert torch.equal(x, y)
    for x, y in zip(a, b):
        assert _same(fmt, x, y)


def test_capture_and_two_shapes(dev):
    det, sd, img, _ = _graph_case("r50_r16", "f16x3", dev, size=256)
    img = img.to(dev)
    eager, _ = det.forward_dense(img)
    eager = [x[0].clone() for x in eager]
    det.capture(tuple(img.shape))
    outs, _ = det.forward_dense_graph(img)
    for a, b in zip(eager, [o[0] for o in outs]):
        assert torch.equal(a, b)
    small = torch.nn.functional.interpolate(img, scale_factor=0.5)
    metas = [[dict(img_shape=(256, 256, 3), scale_factor=1.0, flip=False)] * 2,
             [dict(img_shape=(128, 128, 3), scale_factor=0.5, flip=False)] * 2]
    assert len(det.aug_test([img, small], metas)) == 2
    outs2, _ = det.forward_dense_graph(img)                            # the graph still replays after the eager scales
    for a, b in zip(eager, [o[0] for o in outs2]):
        assert torch.equal(a, b)


@pytest.mark.parametrize("prec", FORMATS)
@pytest.mark.parametrize("variant", ["resnet", "resnext", "dcn", "ga"])
def test_init_detector_with_checkpoint(dev, tmp_path, prec, variant):
    """a config with gcb=dict(ratio=1/16), stage_with_gcb=(False, True, True, True) through init_detector (a checkpoint saved
    with the reference's keys) and inference_detector, on ResNet, ResNeXt, with DCN and with GA"""
    import os
    from orientedreppoints_b200.apis import Config, inference_detector, init_detector
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = Config.fromfile(os.path.join(root, "configs", "dota", "orientedrepoints_r50_demo.py"))
    bb = dict(cfg['model']['backbone'], gcb=dict(R16), stage_with_gcb=C3_C5)
    draw = dict(gcb=dict(R16), stage_with_gcb=C3_C5, gcb_gain=1.0)
    if variant == "resnext":
        bb.update(type='ResNeXt', groups=32, base_width=4)
        draw.update(groups=32, base_width=4)
    if variant == "dcn":
        bb.update(dcn=dict(type='DCN', deformable_groups=1, fallback_on_stride=False), stage_with_dcn=C3_C5)
        draw.update(dcn=dict(type='DCN'), stage_with_dcn=C3_C5)
    if variant == "ga":
        from test_gen_attention_gpu import _tame
        ga = dict(spatial_range=-1, num_heads=8, kv_stride=2, attention_type='1111')
        bb.update(gen_attention=ga, stage_with_gen_attention=[[], [], [0, 1, 2, 3, 4, 5], [0, 1, 2]])
        draw.update(gen_attention=ga, stage_with_gen_attention=[[], [], [0, 1, 2, 3, 4, 5], [0, 1, 2]], gen_attention_gamma=0.7)
    cfg['model']['backbone'] = bb
    cfg['model']['pretrained'] = None
    sd = random_state_dict(50, seed=8, reference_init=False, residual_gain=0.5, **draw)
    if variant == "ga":
        _tame(sd)
    ck = tmp_path / "ck.pth"
    torch.save(dict(state_dict=sd), str(ck))
    m = init_detector(cfg, str(ck), device="cuda:0", precision=prec)
    key = "backbone.layer4.2.context_block.channel_add_conv.3.bias"
    assert torch.equal(m.state_dict()[key].cpu(), sd[key])
    img = (torch.rand(200, 260, 3, generator=torch.Generator().manual_seed(1)) * 255).to(torch.uint8).numpy()
    res = inference_detector(m, img)
    assert len(res) == 15


def _busy(dev):
    a = torch.randn(4096, 4096, device=dev)
    for _ in range(8):
        a = a @ a
        a = a / a.norm()
    return a


@pytest.mark.parametrize("fmt", FORMATS)
def test_side_stream_and_threads(dev, fmt):
    """every entry point (pool, transform, fuse) on a side stream behind queued work; then two host threads, each running
    its own R-50-GCB detector on its own stream"""
    e = _engine(fmt, dev)
    blk, p64, spec = _block(dict(R4_AVG, pooling_type='att'), 512, seed=12, dev=dev)
    g = torch.Generator(device=dev).manual_seed(9)
    xd, _ = _held(e, torch.randn(2, 24, 24, 512, device=dev, generator=g))
    idd, _ = _held(e, torch.randn(2, 24, 24, 512, device=dev, generator=g))
    want = [t.clone() for t in _launches(e, blk, xd, idd)]
    torch.cuda.synchronize()
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _busy(dev)
        got = _launches(e, blk, xd, idd)
    torch.cuda.current_stream().wait_stream(side)
    for a, b in zip(want, got):
        assert torch.equal(a, b)
    dets = [_graph_case("r50_r16", fmt, dev, size=128)[0] for _ in range(2)]
    img = torch.randn(2, 3, 128, 128, generator=torch.Generator().manual_seed(2)).to(dev)
    ref = [t.clone() for t in dets[0].forward_dense(img)[1]]
    torch.cuda.synchronize()
    res, errs = [None, None], []

    def work(i):
        try:
            with torch.cuda.device(dev):
                s = torch.cuda.Stream(device=dev)
                with torch.cuda.stream(s):
                    r = [t.clone() for t in dets[i].forward_dense(img)[1]]
                s.synchronize()
                res[i] = r
        except Exception as ex:                                          # noqa: BLE001
            errs.append(ex)

    th = [threading.Thread(target=work, args=(i,)) for i in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs
    for r in res:
        for a, b in zip(ref, r):
            assert _same(fmt, a, b)


def test_refusals_on_device(dev):
    lib = _lib.lib()
    x = torch.zeros(1, 4, 4, 2, 256, dtype=torch.float16, device=dev)
    ws = torch.zeros(16, device=dev)
    assert lib.orp_context_pool_f16x3(_lib.ptr(x), 1, 4, 4, 256, None, _lib.ptr(ws), 64, None) == -1      # workspace too small
    assert lib.orp_context_fuse_f16x3(_lib.ptr(x), _lib.ptr(x), 1, 4, 4, 256, None, None, _lib.ptr(ws), None) == -1   # no term
    assert lib.orp_context_transform(_lib.ptr(ws), 1, 1, 256, 16, None, None, None, None, None) == -1         # no mlp


# ------------------------------------------------------------------------------------------------ the launch checker
def _checker_cls():
    import test_backbone_launches_gpu as tbl

    class GcbChecker(tbl.BackboneChecker):
        """BackboneChecker plus every context block call, checked against the fp64 contract on the operands the engine holds
        and re-run for bitwise equality"""

        def __init__(self, det, name, monkeypatch, sd):
            super().__init__(det, name, monkeypatch)
            self.gcb_checked, self.sd = 0, sd
            real = cb.ContextBlock.__call__
            chk = self

            def checked(blk, eng, x, identity):
                y = real(blk, eng, x, identity)
                chk._gcb(blk, eng, x, identity, y, real)
                return y
            monkeypatch.setattr(cb.ContextBlock, "__call__", checked)

        def _gcb(self, blk, eng, x, identity, y, real):
            torch.cuda.synchronize()
            n, h, w, c = cb.dims(eng, x)
            p = next(pre for pre, b in ((("backbone.layer%d.%d" % (li + 1, j)), bb["gcb"]) for li, st in enumerate(self.det.blocks)
                                        for j, bb in enumerate(st)) if b is blk)
            p64 = {k: v.double().to(x.device) for k, v in cr.block_params(self.sd, p).items()}
            what = "%s %s.context_block %dx%d C %d" % (self.name, p, h, w, c)
            for j in range(n):                                   # per image, as the pool runs
                x64, i64 = _f(eng, x[j:j + 1]), _f(eng, identity[j:j + 1])
                _, _, ry = _contract(blk.spec, p64, x64, i64)
                err = _rel(_f(eng, y[j:j + 1]), ry)
                tol = 1e-4 if self.split else 1e-2
                assert err < tol, "%s: image %d: rel err %.3e >= %.1e" % (what, j, err, tol)
                if err > self.worst.get("gcb", (-1.0,))[0]:
                    self.worst["gcb"] = (err, tol, "%s image %d" % (what, j))
            self.replaying = True
            try:
                again = real(blk, eng, x, identity)
            finally:
                self.replaying = False
            torch.cuda.synchronize()
            assert torch.equal(again, y), "%s: a second run differs" % what
            self.gcb_checked += 1

    return GcbChecker


@pytest.mark.parametrize("c", GCB_PARITY)
def test_gcb_parity_case_vs_fp64(dev, c):
    """the plan of conv3 + bn3 without residual and ReLU that only R-50-GCB reaches, launched against fp64 as
    tests/test_conv_plans_gpu.py launches PARITY"""
    from conv_plan_cases import planned, signature
    from orientedreppoints_b200.engine_tc import EngineTC
    from test_conv_plans_gpu import Case, _check_values, _check_written_once
    case = Case(c, EngineTC(dev), dev, seed=sum(c[3:7]) + len(c[-1]))
    plan = _check_written_once(case)
    assert signature(plan) == c[0] and plan == planned(c)
    _check_values(case, plan)


GCB_WORKLOADS = [("f16x3", 16, False), ("bf16", 16, False), ("f16x3", 4, True)]


@pytest.mark.parametrize("prec,batch,test_scale", GCB_WORKLOADS,
                         ids=["%s-x%d%s" % (p, n, "-960" if t else "") for p, n, t in GCB_WORKLOADS])
def test_every_launch_vs_fp64_r50_gcb(dev, monkeypatch, prec, batch, test_scale):
    import test_backbone_launches_gpu as tbl
    import test_production_launches_gpu as tpl
    t0 = time.time()
    name = "r50_gcb_r16 %s x%d%s" % (prec, batch, " at 960^2" if test_scale else "")
    sd = random_state_dict(50, seed=0, reference_init=False, residual_gain=0.5, gcb=dict(R16), stage_with_gcb=C3_C5, gcb_gain=1.0)
    lay = gcb_layout(50, dict(R16), C3_C5)
    img, valid = tpl._inputs("r101", batch, test_scale, dev)
    det = OrientedRepPointsDetector(sd, 50, dev, prec, test_cfg=dict(score_thr=0.0), gcb=lay)
    chk = _checker_cls()(det, name, monkeypatch, sd)
    if chk.split:
        det.eng.overflow_count()
    with torch.no_grad():
        dense = det.forward_dense(img, valid)
    torch.cuda.synchronize()
    print(chk.summary(time.time() - t0))
    assert not chk.escaped, "%s: launches outside a checked call: %s" % (name, chk.escaped)
    assert chk.checked == chk.low and chk.checked > 0
    assert chk.gcb_checked == 13                                        # c3-c5 of R-50: 4 + 6 + 3 blocks
    if chk.split:
        assert det.eng.overflow_count() == 0, name
    if chk.split and not test_scale:
        tbl._tiles_vs_fp64(det, sd, lambda s, x: cr.forward_dense(s, x, lay), img, dense, name)
    monkeypatch.setattr(tbl, "PARITY", tbl.PARITY + GCB_PARITY)
    tbl._signatures_pinned(chk)
    del det, chk, dense
    torch.cuda.empty_cache()
