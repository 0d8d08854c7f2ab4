"""Generalized attention on the H100 (include/orp_b200_attention.h): every attention launch of R-50 with the published c4-c5
layout at 1024^2 and 960^2 tiles against fp64 in all three formats, a peaked softmax, every attention_type the engine builds as
a whole block, whole R-50 graphs with '1111' / '0010' blocks (with and without DCN) against the fp64 graph, CUDA-graph capture,
two input shapes, init_detector from a checkpoint, and the entry points on a side stream and from two host threads."""
import ctypes
import itertools
import threading

import pytest
import torch

from orientedreppoints_b200 import _lib
from orientedreppoints_b200 import gen_attention as ga
from orientedreppoints_b200.detector import EngineF32, OrientedRepPointsDetector
from orientedreppoints_b200.weights import gen_attention_layout, gen_attention_spec, random_state_dict
import gen_attention_ref as gr

pytestmark = pytest.mark.gpu
FORMATS = ["f16x3", "bf16", "fp32"]


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
    """t (fp32, [.., C]) in the engine's format, and the exact values it holds (fp64)"""
    x = t.reshape((1, 1) + t.shape[-2:]) if t.dim() == 2 else t
    if e.name == "fp32":
        y = x.to(e.device).contiguous()
        return y, y.double().reshape(t.shape)
    y = e.from_float(x)
    return y, e.to_float(y).double().reshape(t.shape)


def _ref(qc, qp, k, v, px, py, h, w, hk, wk, s, heads):
    """the kernel's contract in fp64: qc / qp [N, H W, C] or None, k / v [N, Hk Wk, C], px [Rx, C], py [Ry, C]"""
    n, _, c = v.shape
    d = c // heads
    hd = lambda t: t.reshape(t.shape[0], -1, heads, d).transpose(1, 2)                   # noqa: E731
    e = torch.zeros(n, heads, h * w, hk * wk, dtype=torch.float64, device=v.device)
    if qc is not None:
        e = e + hd(qc) @ hd(k).transpose(2, 3)
    if qp is not None:
        ix = (torch.arange(w)[:, None] - s * torch.arange(wk)[None, :] + s * (wk - 1)).to(v.device)
        iy = (torch.arange(h)[:, None] - s * torch.arange(hk)[None, :] + s * (hk - 1)).to(v.device)
        fx, fy = px.reshape(-1, heads, d)[ix], py.reshape(-1, heads, d)[iy]                 # [W, Wk, heads, d]
        q5 = hd(qp).reshape(n, heads, h, w, d)
        ex = torch.einsum('nhyxd,xkhd->nhyxk', q5, fx)
        ey = torch.einsum('nhyxd,ykhd->nhyxk', q5, fy)
        e = e + (ey[..., :, None] + ex[..., None, :]).reshape(n, heads, h * w, hk * wk)
    return (torch.softmax(e, -1) @ hd(v)).transpose(1, 2).reshape(n, h * w, c), e


def _launch(e, fmt, n, h, w, c, heads, s, seed, content=True, position=True, q_gain=1.0):
    g = torch.Generator().manual_seed(seed)
    hk, wk = -(-h // s), -(-w // s)
    d = c // heads
    q = torch.randn(n, h, w, 2 * c, generator=g) * (q_gain / d ** 0.25)
    kv = torch.randn(n, hk, wk, 2 * c, generator=g) / d ** 0.25
    kv[..., c:] *= d ** 0.25
    px = torch.randn(w + s * (wk - 1), c, generator=g) / d ** 0.25
    py = torch.randn(h + s * (hk - 1), c, generator=g) / d ** 0.25
    qd, q64 = _held(e, q)
    kvd, kv64 = _held(e, kv)
    tabs = [_held(e, t) for t in (px, py)]
    out = ga.attend(e, qd, 0 if content else None, c if position else None, kvd, 0 if content else None, c,
                    (tabs[0][0], tabs[1][0]) if position else None, n, h, w, hk, wk, s, c, heads)
    got = (e.to_float(out) if fmt != "fp32" else out).double().reshape(n, h * w, c)
    q64, kv64 = q64.reshape(n, h * w, 2 * c), kv64.reshape(n, hk * wk, 2 * c)
    ref, energy = _ref(q64[..., :c] if content else None, q64[..., c:] if position else None, kv64[..., :c], kv64[..., c:],
                       tabs[0][1], tabs[1][1], h, w, hk, wk, s, heads)
    return got, ref, energy


# (tile, map side, channels): stage 3 and stage 4 of R-50 at 1024^2 and 960^2
LAUNCHES = [(1024, 64, 256), (1024, 32, 512), (960, 60, 256), (960, 30, 512)]
TOL = {"f16x3": 1e-4, "fp32": 1e-4, "bf16": None}


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("tile, h, c", LAUNCHES)
def test_published_launches_vs_fp64(dev, fmt, tile, h, c):
    e = _engine(fmt, dev)
    got, ref, energy = _launch(e, fmt, 2, h, h, c, 8, 2, seed=tile + h)
    err = float((got - ref).abs().max() / ref.abs().max())
    if fmt == "bf16":
        # bf16 holds Q, K, V and the tables to 2^-9 relative; an energy of spread sigma then moves by ~2^-8 sigma sqrt(d)-
        # fold summed, and the probabilities by that times themselves.  The seeded energies have unit spread (|E| <~ 6).
        sigma = float(energy.std())
        assert sigma < 2.0
        tol = 0.02 * max(1.0, sigma)
    else:
        tol = TOL[fmt]
    assert err < tol, (err, tol)


@pytest.mark.parametrize("fmt", ["f16x3", "fp32"])
def test_peaked_softmax(dev, fmt):
    e = _engine(fmt, dev)
    got, ref, energy = _launch(e, fmt, 1, 33, 31, 256, 8, 2, seed=5, q_gain=12.0)
    assert float(energy.abs().max()) > 100                              # rows dominated by a few keys
    assert float((got - ref).abs().max() / ref.abs().max()) < 2e-4


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("content, position", [(True, False), (False, True), (False, False)])
def test_terms_and_stride1_odd(dev, fmt, content, position):
    e = _engine(fmt, dev)
    got, ref, _ = _launch(e, fmt, 2, 13, 9, 512, 8, 1, seed=7, content=content, position=position)
    assert float((got - ref).abs().max() / ref.abs().max()) < (0.03 if fmt == "bf16" else 1e-4)


TYPES = ["".join(b) for b in itertools.product("01", repeat=4) if not (b[1] == "1" and b[3] == "0")]


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("t", TYPES)
def test_block_every_attention_type(dev, fmt, t):
    """the whole block (Q / KV / proj convolutions, tables, the launch, the '0010' shortcut) against gen_attention_ref.block"""
    cfg = dict(gr.PUBLISHED, attention_type=t)
    stages = [[], [], [0], []]
    sd = random_state_dict(50, seed=11, reference_init=False, gen_attention=cfg, stage_with_gen_attention=stages,
                           gen_attention_gamma=0.7)
    spec = gen_attention_spec(cfg, 256)
    e = _engine(fmt, dev)
    blk = ga.GenAttentionBlock(sd, "backbone.layer3.0", spec, dev)
    x = torch.randn(2, 11, 14, 256, generator=torch.Generator().manual_seed(3))
    xd, x64 = _held(e, x)
    y = blk(e, xd)
    got = (e.to_float(y) if fmt != "fp32" else y).double()
    p64 = {k: v.double() for k, v in gr.block_params(sd, "backbone.layer3.0").items()}
    ref = gr.block(spec, p64, x64.cpu().permute(0, 3, 1, 2)).permute(0, 2, 3, 1).to(dev)
    assert float((got - x64).abs().max()) > 0.05                       # the block acts
    err = float((got - ref).abs().max() / ref.abs().max())
    assert err < (0.03 if fmt == "bf16" else 1e-4), err


def _tame(sd, f=0.03):
    """scale every block's Qc / Qp / K sources by f, so energies scale by f^2: with the seeded graphs' activations (up to ~100
    at c4 / c5) the energies of the draws reach std ~3000, a softmax that is an argmax of near-ties which 1e-6 changes of its
    input flip; at f = 0.03 their std stays within about 0.01..3 (0.0009 times the std of the unscaled draws, measured per block
    on the H100 at 128^2 input: 8.9 .. 2900)"""
    for k in list(sd):
        if ".gen_attention_block." in k and k.split(".gen_attention_block.")[1] in (
                "query_conv.weight", "key_conv.weight", "appr_geom_fc_x.weight", "appr_geom_fc_y.weight", "appr_bias", "geom_bias"):
            sd[k] = sd[k] * f
    return sd


def _graph_case(t, dcn, fmt, dev, size=128):
    stages = gr.PUBLISHED_STAGES
    cfg = dict(gr.PUBLISHED, attention_type=t)
    dcfg = dict(type='DCN', deformable_groups=1, fallback_on_stride=False) if dcn else None
    swd = (False, True, True, True) if dcn else (False,) * 4
    # with DCN, residual_gain 0.3 as in tests/test_dcn_backbone_gpu.py: larger activations make larger offsets, and the fp64 graph
    # itself then amplifies fp32 rounding differences of its input beyond 1e-4
    sd = random_state_dict(50, seed=21, reference_init=False, residual_gain=0.3 if dcn else 0.5, dcn=dcfg, stage_with_dcn=swd,
                           dcn_offset_scale=0.5 if dcn else 0.0, gen_attention=cfg, stage_with_gen_attention=stages,
                           gen_attention_gamma=0.7)
    _tame(sd)
    from orientedreppoints_b200.weights import dcn_layout
    lay = dcn_layout(50, dcfg, swd) if dcn else None
    gal = gen_attention_layout(50, cfg, stages)
    det = OrientedRepPointsDetector(sd, 50, dev, fmt, dcn=lay, gen_attention=gal)
    img = torch.randn(2, 3, size, size, generator=torch.Generator().manual_seed(4))
    return det, sd, img, lay, gal


@pytest.mark.parametrize("t", ["1111", "0010"])
@pytest.mark.parametrize("dcn", [False, True])
@pytest.mark.parametrize("fmt", ["f16x3", "fp32"])
def test_whole_graph_vs_fp64(dev, t, dcn, fmt):
    det, sd, img, lay, gal = _graph_case(t, dcn, fmt, dev)
    (outs, feats) = det.forward_dense(img.to(dev))
    sd64 = {k: v.double() for k, v in sd.items()}
    ref_outs, ref_feats = gr.forward_dense(sd64, img.double(), lay, gal)
    for f, r in zip(feats, ref_feats):
        got = (det.eng.to_float(f) if fmt != "fp32" else f).double().cpu().permute(0, 3, 1, 2)
        err = float((got - r).abs().max() / r.abs().max())
        assert err < 1e-4, err
    for (c, i, rf), (rc, ri, rr) in zip(outs, ref_outs):          # head outputs as tests/test_dcn_backbone_gpu.py measures them
        for a, b in ((c, rc), (i, ri), (rf, rr)):
            a = a.double().cpu().permute(0, 3, 1, 2)
            assert float((a - b).abs().max()) / max(1.0, float(b.abs().max())) < 1e-4
    if fmt == "f16x3":
        assert det.eng.overflow_count() == 0
    dets = det.simple_test(img.to(dev), rescale=False)
    assert len(dets) == 2


@pytest.mark.parametrize("t", ["1111", "0010"])
def test_capture_and_two_shapes(dev, t):
    det, sd, img, lay, gal = _graph_case(t, False, "f16x3", dev, size=256)
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
    res = det.aug_test([img, small], metas)
    assert len(res) == 2
    blk = det.blocks[2][0]["att"]
    if blk.qp_off is not None:
        assert {k[1:] for k in blk._tables} == {(16, 16), (8, 8)}                  # one table pair per map size


def test_init_detector_with_checkpoint(dev, tmp_path):
    import os
    from orientedreppoints_b200.apis import Config, init_detector
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = Config.fromfile(os.path.join(root, "configs", "dota", "orientedrepoints_r50_demo.py"))
    cfg['model']['backbone'] = dict(cfg['model']['backbone'], gen_attention=dict(gr.PUBLISHED, attention_type='1111'),
                                    stage_with_gen_attention=gr.PUBLISHED_STAGES)
    cfg['model']['pretrained'] = None
    sd = _tame(random_state_dict(50, seed=8, reference_init=False, residual_gain=0.5, gen_attention=dict(gr.PUBLISHED),
                                 stage_with_gen_attention=gr.PUBLISHED_STAGES, gen_attention_gamma=0.7))
    ck = tmp_path / "ck.pth"
    torch.save(dict(state_dict=sd), str(ck))
    m = init_detector(cfg, str(ck), device="cuda:0")
    assert torch.equal(m.state_dict()["backbone.layer4.2.gen_attention_block.gamma"].cpu(), sd["backbone.layer4.2.gen_attention_block.gamma"])
    img = torch.randn(1, 3, 128, 128, generator=torch.Generator().manual_seed(1)).to(dev)
    feats = m.extract_feat(img)
    sd64 = {k: v.double() for k, v in sd.items()}
    ref = gr.forward_dense(sd64, img.double().cpu(), None, gen_attention_layout(50, dict(gr.PUBLISHED), gr.PUBLISHED_STAGES))[1]
    got = m.engine().eng.to_float(feats[0]).double().cpu().permute(0, 3, 1, 2)
    assert float((got - ref[0]).abs().max() / ref[0].abs().max()) < 1e-4


def _busy(dev):
    a = torch.randn(4096, 4096, device=dev)
    for _ in range(8):
        a = a @ a
        a = a / a.norm()
    return a


@pytest.mark.parametrize("fmt", FORMATS)
def test_side_stream_and_threads(dev, fmt):
    e = _engine(fmt, dev)
    c, h, n = 256, 24, 2
    x = torch.randn(n, h, h, c, generator=torch.Generator().manual_seed(9))
    cfg = dict(gr.PUBLISHED, attention_type='1111')
    sd = random_state_dict(50, seed=12, reference_init=False, gen_attention=cfg, stage_with_gen_attention=[[], [], [0], []],
                           gen_attention_gamma=0.7)
    blk = ga.GenAttentionBlock(sd, "backbone.layer3.0", gen_attention_spec(cfg, c), dev)
    sal = ga.GenAttentionBlock(random_state_dict(50, seed=13, gen_attention=dict(cfg, attention_type='0010'),
                                                 stage_with_gen_attention=[[], [], [0], []], gen_attention_gamma=0.7),
                               "backbone.layer3.0", gen_attention_spec(dict(cfg, attention_type='0010'), c), dev)
    xd, _ = _held(e, x)
    want = [blk(e, xd).clone(), sal(e, xd).clone()]
    torch.cuda.synchronize()
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _busy(dev)
        got = [blk(e, xd), sal(e, xd)]
    torch.cuda.current_stream().wait_stream(side)
    for a, b in zip(want, got):
        assert torch.equal(a, b)
    res, errs = [None, None], []

    def work(i):
        try:
            with torch.cuda.device(dev):
                s = torch.cuda.Stream(device=dev)
                with torch.cuda.stream(s):
                    r = [blk(e, xd), sal(e, xd)]
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
        for a, b in zip(want, r):
            assert torch.equal(a, b)


def test_refusals_on_device(dev):
    a = _lib.GenAttentionArgs()
    lib = _lib.lib()
    assert lib.orp_gen_attention_f16x3(ctypes.byref(a), None) == -1                   # ORP_EINVAL before any launch
    x = torch.zeros(1, 4, 4, 2, 256, dtype=torch.float16, device=dev)
    assert lib.orp_gen_attention_bcast_add_f16x3(_lib.ptr(x), 1, 4, 4, 256, None, _lib.ptr(x), None) == -1
