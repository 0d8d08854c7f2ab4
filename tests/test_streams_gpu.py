"""GPU: every compute entry point of the library on a PyTorch side stream, and the detector from two host threads.

Every entry point takes a `stream`, and the Python wrappers pass torch.cuda.current_stream().  The benchmark does not run
on the default stream only (detector.capture warms up on a side stream, bench_tile uploads on a copy stream), and ctypes
releases the GIL, so two threads can be inside the library at once.  PyTorch's pool streams are created non-blocking: the
legacy default stream does not order them, so work the library put on stream 0 (a synchronous cudaMemcpy, a symbol copy)
would run out of order with the caller's work.

- Side-stream equivalence: each case runs once on the default stream (its result is pinned to fp64 or to the reference by
  the rest of the suite), then on a fresh torch.cuda.Stream behind a torch.cuda._sleep spin, with its inputs written by a
  copy kernel after the spin into buffers that held NaN (zero for integers).  An entry point that reads inputs or scratch
  out of stream order sees the stale values.  Outputs the case allocates go into NaN-filled guarded buffers.  Results
  must be bitwise equal, except GroupNorm sums (fp64 atomics) and what is computed from them: REPLAY_TOL.
- ENTRY_POINTS maps every compute symbol of _lib.SIGNATURES to its cases; NOT_STREAM_ORDERED lists the rest with a reason.
- The f16x3 overflow counter is read in stream order and its reset loses no events.
- Two detectors in two threads, each on its own stream, give their serial results; one replays a graph meanwhile."""
import ctypes
import threading

import numpy as np
import pytest
import torch

from orientedreppoints_b200 import _lib

gpu = pytest.mark.gpu

SPIN = 50_000_000          # torch.cuda._sleep cycles ahead of the inputs: ~25 ms at the H100's 1.98 GHz boost clock
REPLAY_TOL = 1e-5          # tests/test_production_launches_gpu.py: GroupNorm sums are atomics, bits may differ
GUARD = 4096               # bytes before and after every guarded output
FILL = -1                  # int16 fill of guarded outputs: NaN as fp32, fp16 and bf16; -1 as integers

# compute symbol -> the cases of this file that run it on a side stream
ENTRY_POINTS = {
    "orp_conv2d_bf16": ["test_conv_side_stream"],
    "orp_conv2d_f16x3": ["test_conv_side_stream", "test_overflow_count_side_stream"],
    "orp_conv2d_tc_splitk": ["test_conv_side_stream"],
    "orp_stem_s2d_bf16": ["test_conv_side_stream"],
    "orp_stem_s2d_f16x3": ["test_conv_side_stream"],
    "orp_stem_conv_s2d_bf16": ["test_conv_side_stream"],
    "orp_stem_conv_s2d_f16x3": ["test_conv_side_stream"],
    "orp_stem_s2d_u8_bf16": ["test_stem_u8_side_stream"],
    "orp_stem_s2d_u8_f16x3": ["test_stem_u8_side_stream"],
    "orp_stem_s2d_u8_padded_bf16": ["test_stem_u8_side_stream"],
    "orp_stem_s2d_u8_padded_f16x3": ["test_stem_u8_side_stream"],
    "orp_stem_im2col_bf16": ["test_stem_u8_side_stream"],
    "orp_gn_stats_bf16": ["test_gn_maxpool_side_stream", "test_conv_side_stream"],
    "orp_gn_stats_f16x3": ["test_gn_maxpool_side_stream", "test_conv_side_stream"],
    "orp_gn_apply_bf16_multi": ["test_gn_maxpool_side_stream"],
    "orp_gn_apply_f16x3_multi": ["test_gn_maxpool_side_stream"],
    "orp_maxpool3x3s2_bf16": ["test_gn_maxpool_side_stream"],
    "orp_maxpool3x3s2_f16x3": ["test_gn_maxpool_side_stream"],
    "orp_split_from_f32": ["test_layout_side_stream"],
    "orp_split_to_f32": ["test_layout_side_stream"],
    "orp_transpose_f32": ["test_layout_side_stream"],
    "orp_nchw_f32_to_split": ["test_layout_side_stream"],
    "orp_dcn_offsets_multi": ["test_layout_side_stream"],
    "orp_layernorm_bf16": ["test_swin_side_stream"],
    "orp_layernorm_f16x3": ["test_swin_side_stream"],
    "orp_window_attention_bf16": ["test_swin_side_stream"],
    "orp_window_attention_f16x3": ["test_swin_side_stream"],
    "orp_patch_embed_rows_bf16": ["test_swin_side_stream"],
    "orp_patch_embed_rows_f16x3": ["test_swin_side_stream"],
    "orp_patch_embed_rows_u8_bf16": ["test_swin_side_stream"],
    "orp_patch_embed_rows_u8_f16x3": ["test_swin_side_stream"],
    "orp_patch_embed_rows_u8_padded_bf16": ["test_swin_side_stream"],
    "orp_patch_embed_rows_u8_padded_f16x3": ["test_swin_side_stream"],
    "orp_patch_merge_gather_bf16": ["test_swin_side_stream"],
    "orp_patch_merge_gather_f16x3": ["test_swin_side_stream"],
    "orp_subsample2_bf16": ["test_swin_side_stream"],
    "orp_subsample2_f16x3": ["test_swin_side_stream"],
    "orp_rnms": ["test_rnms_side_stream"],
    "orp_head_postprocess": ["test_postprocess_merge_eval_side_stream"],
    "orp_head_postprocess_aug": ["test_postprocess_merge_eval_side_stream"],
    "orp_pack_detections": ["test_postprocess_merge_eval_side_stream"],
    "orp_result_merge": ["test_postprocess_merge_eval_side_stream"],
    "orp_dota_eval_task1": ["test_postprocess_merge_eval_side_stream"],
    "orp_dota_eval_aoe": ["test_postprocess_merge_eval_side_stream"],
    "orp_poly2rbox_v3": ["test_postprocess_merge_eval_side_stream"],
    "orp_resize_u8": ["test_resize_split_side_stream"],
    "orp_split_tiles_u8": ["test_resize_split_side_stream"],
    "orp_minarearect": ["test_geometry_side_stream"],
    "orp_box_iou_rotated": ["test_geometry_side_stream"],
    "orp_quad_iou_matrix": ["test_geometry_side_stream"],
    "orp_poly_overlaps": ["test_geometry_side_stream"],
    "orp_iou_poly_f64_pairs": ["test_geometry_side_stream"],
    "orp_convex_iou": ["test_geometry_side_stream"],
    "orp_convex_giou": ["test_geometry_side_stream"],
    "orp_conv2d_f32": ["test_f32_engine_side_stream"],
    "orp_deform_conv2d_f32": ["test_f32_engine_side_stream"],
    "orp_gn_apply_f32": ["test_f32_engine_side_stream"],
    "orp_maxpool3x3s2_f32": ["test_f32_engine_side_stream"],
    "orp_f16x3_overflow_count": ["test_overflow_count_side_stream", "test_overflow_count_reset_keeps_running_launch"],
}

# symbols without a stream to order: host-side state and the blocking host-buffer drop-ins
NOT_STREAM_ORDERED = {
    "orp_last_error": "thread-local message of the last failure",
    "orp_version": "constant",
    "orp_compiled_sm": "constant",
    "orp_launch_count": "host counter (atomic)",
    "orp_reset_launch_count": "host counter (atomic)",
    "orp_rnms_last_stats": "host copy of the last NMS counters; documented to need the caller's stream synchronised",
    "orp_rnms_last_plan": "thread-local host record, checked per thread by test_two_threads_two_detectors",
    "orp_set_timing": "host switch",
    "orp_rnms_last_sweep_ms": "waits on the call's own events",
    "orp_tc_timing_collect": "waits on the calls' own events",
    "orp_tc_last_plan": "thread-local host record, checked per thread by test_two_threads_two_detectors",
    "orp_tc_plan_conv": "dry run on the host, no device work",
    "orp_poly_nms_host": "host buffers, blocking: runs on a non-blocking stream of its own and synchronises it",
    "orp_poly_overlaps_host": "host buffers, blocking: runs on a stream of its own and synchronises it",
}


def test_every_entry_point_is_covered_or_listed():
    """each symbol of _lib.SIGNATURES (every symbol the header declares, tests/test_abi.py) names an existing case of this
    file or a reason why it has no stream to order"""
    assert not set(ENTRY_POINTS) & set(NOT_STREAM_ORDERED)
    assert set(ENTRY_POINTS) | set(NOT_STREAM_ORDERED) == set(_lib.SIGNATURES), \
        sorted(set(_lib.SIGNATURES) ^ (set(ENTRY_POINTS) | set(NOT_STREAM_ORDERED)))
    for name, cases in ENTRY_POINTS.items():
        assert cases, name
        for c in cases:
            assert callable(globals().get(c)), (name, c)


# ------------------------------------------------------------------------------------------------------------ harness
class Guarded:
    """an output tensor carved out of a larger buffer with guard regions on both sides"""

    def __init__(self, shape, dtype, dev):
        n = 1
        for v in shape:
            n *= v
        self.nbytes = n * torch.empty((), dtype=dtype).element_size()
        self.buf = torch.empty(2 * GUARD + self.nbytes + (self.nbytes & 1), dtype=torch.uint8, device=dev)
        self.t = self.buf[GUARD:GUARD + self.nbytes].view(dtype).view(shape)
        self.buf.view(torch.int16).fill_(FILL)

    def guards_intact(self):
        w = self.buf.view(torch.int16)
        return bool((w[:GUARD // 2] == FILL).all()) and bool((w[(GUARD + self.nbytes + 1) // 2:] == FILL).all())


class Run:
    """one run of a case: the guarded outputs it made (filled on the stream current when they are made)"""

    def __init__(self, dev):
        self.dev, self.guarded = dev, []

    def out(self, shape, dtype):
        g = Guarded(tuple(shape), dtype, self.dev)
        self.guarded.append(g)
        return g.t


def _bits(t):
    t = t.contiguous()
    if t.dtype == torch.bool:
        return t.view(torch.uint8)
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _stale(t):
    s = torch.empty_like(t)
    if s.is_floating_point():
        s.fill_(float("nan"))
    else:
        s.zero_()
    return s


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / (b.double().abs().max() + 1e-30))


def side_stream_check(dev, src, fn, tol=()):
    """fn(inputs, run) -> list of output tensors.  Once on the default stream, once on a fresh side stream whose inputs
    are copied in behind a spin; outputs bitwise equal (indices in `tol`: within REPLAY_TOL).  Returns the reference."""
    r0 = Run(dev)
    ref = [o.clone() for o in fn({k: v.clone() for k, v in src.items()}, r0)]
    stale = {k: _stale(v) for k, v in src.items()}
    torch.cuda.synchronize(dev)
    s = torch.cuda.Stream(device=dev)
    r1 = Run(dev)
    with torch.cuda.stream(s):
        torch.cuda._sleep(SPIN)
        for k, v in stale.items():
            v.copy_(src[k])
        got = [o.clone() for o in fn(stale, r1)]
    s.synchronize()
    torch.cuda.synchronize(dev)
    for g in r0.guarded + r1.guarded:
        assert g.guards_intact(), "a store landed outside its output"
    assert len(ref) == len(got)
    for i, (a, b) in enumerate(zip(ref, got)):
        assert a.shape == b.shape and a.dtype == b.dtype, i
        if i in tol:
            assert bool(torch.isfinite(b.double()).all()), "output %d: not finite on the side stream" % i
            assert _rel(b, a) < REPLAY_TOL, (i, _rel(b, a))
        else:
            assert torch.equal(_bits(a), _bits(b)), "output %d differs on the side stream" % i
    return ref


def _engine(prec, dev):
    from orientedreppoints_b200.engine_tc import EngineTC, EngineTCSplit
    return EngineTCSplit(dev) if prec == "f16x3" else EngineTC(dev)


def _act(run, eng, n, h, w, c):
    return run.out((n, h, w, 2, c) if eng.name == "f16x3" else (n, h, w, c), eng.act_dtype)


def _nhwc(g, *shape):
    """fp32 NHWC random tensor of NCHW shape"""
    return torch.randn(*shape, generator=g).permute(0, 2, 3, 1).contiguous()


# --------------------------------------------------------------------------------------------------- tensor-core conv
@gpu
@pytest.mark.parametrize("prec", ["f16x3", "bf16"])
@pytest.mark.parametrize("kind", ["residual_relu", "head_f32", "gn_fused", "splitk", "splitk_gn", "deform", "deform_mask",
                                  "stem"])
def test_conv_side_stream(cuda, prec, kind):
    from orientedreppoints_b200.detector import ConvLayer
    eng = _engine(prec, cuda)
    g = torch.Generator().manual_seed(sum(map(ord, prec + kind)))
    st = _lib.current_stream_ptr
    tol = ()
    if kind == "stem":
        L = ConvLayer(torch.randn(64, 3, 7, 7, generator=g) * 0.1, torch.randn(64, generator=g) * 0.1, 2, 3, cuda, pad_cin_to=4)
        src = {"img": torch.randn(2, 3, 96, 160, generator=g).to(cuda)}

        def fn(inp, run):
            n, _, h, w = inp["img"].shape
            xs = eng._s2d_input(n, h, w)
            eng._call("orp_stem_s2d_%s", _lib.ptr(inp["img"]), n, h, w, _lib.ptr(xs), st())
            ws, scale = eng._stem_s2d_operands(L)
            y = _act(run, eng, n, h // 2, w // 2, 64)
            eng._call("orp_stem_conv_s2d_%s", _lib.ptr(xs), n, h, w, _lib.ptr(ws), _lib.ptr(L.bias), *scale, 1, _lib.ptr(y), st())
            return [y]
    elif kind in ("splitk", "splitk_gn"):
        cin, hw = (2048, 32) if kind == "splitk" else (512, 16)
        L = ConvLayer(torch.randn(256, cin, 3, 3, generator=g) * (1.0 / (cin * 9) ** 0.5),
                      torch.randn(256, generator=g) if kind == "splitk" else None, 2, 1, cuda)
        src = {"x": eng.from_float(_nhwc(g, 1, cin, hw, hw).to(cuda))}
        torch.cuda.synchronize()
        ho = hw // 2
        assert eng._ksplit(1, ho, ho, L, 1, kind == "splitk", None, False, None) > 1

        def fn(inp, run):
            y = _act(run, eng, 1, ho, ho, 256)
            stats = torch.zeros((1, 32, 2), dtype=torch.float64, device=cuda) if kind == "splitk_gn" else None
            eng._conv_splitk(inp["x"], y, eng._tc(L), L, kind == "splitk", eng._ksplit(1, ho, ho, L, 1, True, None, False, None),
                             stats, prec == "f16x3")
            return [y] if stats is None else [y, stats]
        tol = (1,)
    elif kind in ("deform", "deform_mask"):
        L = ConvLayer(torch.randn(256, 256, 3, 3, generator=g) * 0.02, None, 1, 1, cuda)
        shapes = [(2, 24, 40), (2, 12, 20), (2, 6, 10)]
        src = {}
        for i, (n, h, w) in enumerate(shapes):
            src["x%d" % i] = eng.from_float(_nhwc(g, n, 256, h, w).to(cuda))
            src["o%d" % i] = (_nhwc(g, n, 18, h, w) * 2.5).to(cuda)
            if kind == "deform_mask":
                src["m%d" % i] = torch.rand(n, h, w, 9, generator=g).to(cuda)
        torch.cuda.synchronize()

        def fn(inp, run):
            ys = [_act(run, eng, n, h, w, 256) for (n, h, w) in shapes]
            k = range(len(shapes))
            eng._launch([inp["x%d" % i] for i in k], ys, eng._tc(L), 256, 3, 3, 256, 1, 1, None, True, False, True,
                        offsets=[inp["o%d" % i] for i in k], masks=[inp["m%d" % i] for i in k] if kind == "deform_mask" else None)
            return ys
    else:
        cin, cout, k = {"residual_relu": (128, 256, 3), "head_f32": (256, 18, 1), "gn_fused": (256, 256, 3)}[kind]
        L = ConvLayer(torch.randn(cout, cin, k, k, generator=g) * (1.0 / (cin * k * k) ** 0.5),
                      torch.randn(cout, generator=g) if kind != "gn_fused" else None, 1, k // 2, cuda)
        shapes = [(2, 40, 56), (2, 20, 28)] if kind != "residual_relu" else [(2, 40, 56)]
        src = {}
        for i, (n, h, w) in enumerate(shapes):
            src["x%d" % i] = eng.from_float(_nhwc(g, n, cin, h, w).to(cuda))
            if kind == "residual_relu":
                src["r%d" % i] = eng.from_float(_nhwc(g, n, cout, h, w).to(cuda))
            if kind == "head_f32":
                src["r%d" % i] = _nhwc(g, n, cout, h, w).to(cuda)
        torch.cuda.synchronize()
        idx = range(len(shapes))

        def fn(inp, run):
            xs = [inp["x%d" % i] for i in idx]
            if kind == "head_f32":
                ys = [run.out((n, h, w, cout), torch.float32) for (n, h, w) in shapes]
                eng._launch(xs, ys, eng._tc(L), cout, 1, 1, cin, 1, 0, L.bias, False, True, False, res32=[inp["r%d" % i] for i in idx])
                return ys
            ys = [_act(run, eng, n, h, w, cout) for (n, h, w) in shapes]
            if kind == "residual_relu":
                eng._launch(xs, ys, eng._tc(L), cout, k, k, cin, 1, k // 2, L.bias, True, False, False,
                            res=[inp["r%d" % i] for i in idx])
                return ys
            stats = [torch.zeros((n, 32, 2), dtype=torch.float64, device=cuda) for (n, _, _) in shapes]
            eng._launch(xs, ys, eng._tc(L), cout, k, k, cin, 1, k // 2, None, False, False, False, stats=stats)
            return ys + stats
        if kind == "gn_fused":
            tol = (2, 3)
    side_stream_check(cuda, src, fn, tol)
    if prec == "f16x3":
        assert eng.overflow_count() == 0


@gpu
@pytest.mark.parametrize("prec", ["f16x3", "bf16"])
def test_stem_u8_side_stream(cuda, prec):
    """the uint8 stem inputs (Normalize, and Pad when valid_hw is given, fused into the space-to-depth transform) and the
    bf16 im2col stem"""
    from orientedreppoints_b200.detector import ConvLayer
    eng = _engine(prec, cuda)
    g = torch.Generator().manual_seed(31)
    L = ConvLayer(torch.randn(64, 3, 7, 7, generator=g) * 0.1, torch.randn(64, generator=g) * 0.1, 2, 3, cuda, pad_cin_to=4)
    cfg = dict(mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375], to_rgb=True)
    src = {"img": torch.randint(0, 256, (2, 96, 128, 3), generator=g, dtype=torch.uint8).to(cuda),
           "valid": torch.tensor([[96, 128], [71, 93]], dtype=torch.int32).to(cuda),
           "nchw": torch.randn(2, 3, 64, 80, generator=g).to(cuda)}
    torch.cuda.synchronize()

    def fn(inp, run):
        outs = [eng.stem_u8(inp["img"], L, cfg), eng.stem_u8(inp["img"], L, cfg, valid_hw=inp["valid"])]
        if prec == "bf16":
            outs.append(eng.stem(inp["nchw"], L, mode="im2col"))
        return outs
    side_stream_check(cuda, src, fn)


# -------------------------------------------------------------------------------------------- GroupNorm, max-pool
@gpu
@pytest.mark.parametrize("prec", ["f16x3", "bf16"])
def test_gn_maxpool_side_stream(cuda, prec):
    """GroupNorm statistics (atomics: REPLAY_TOL) and the apply pass over two tensors with the FPN's upsampled add, the apply
    again from fixed statistics (bitwise), and the stem's max-pool"""
    eng = _engine(prec, cuda)
    g = torch.Generator().manual_seed(41)
    shapes = [(2, 34, 46), (2, 17, 23)]
    src = {"x0": eng.from_float((_nhwc(g, 2, 256, 34, 46) * 3 + 1).to(cuda)),
           "x1": eng.from_float((_nhwc(g, 2, 256, 17, 23) * 3 + 1).to(cuda)),
           "up0": eng.from_float(_nhwc(g, 2, 256, 17, 23).to(cuda)),
           "gamma": torch.randn(256, generator=g).to(cuda), "beta": torch.randn(256, generator=g).to(cuda),
           "s1": torch.zeros(2, 32, 2, dtype=torch.float64),
           "p": eng.from_float(_nhwc(g, 2, 64, 33, 41).to(cuda))}
    stat = torch.zeros(2, 32, 2, dtype=torch.float64, device=cuda)
    n, h, w = shapes[1]
    eng._call("orp_gn_stats_%s", _lib.ptr(src["x1"]), n, h * w, 256, 32, _lib.ptr(stat), _lib.current_stream_ptr())
    src["s1"] = stat
    torch.cuda.synchronize()

    def apply(inp, run, xs, stats, ups):
        ys = [_act(run, eng, n, h, w, 256) for (n, h, w) in [shapes[i] for i in xs]]
        arr = (_lib.GnProblem * len(xs))()
        for j, i in enumerate(xs):
            x = inp["x%d" % i]
            arr[j].x, arr[j].N, arr[j].H, arr[j].W = x.data_ptr(), shapes[i][0], shapes[i][1], shapes[i][2]
            arr[j].stats, arr[j].up_src, arr[j].y = stats[j].data_ptr(), ups[j], ys[j].data_ptr()
        eng._call("orp_gn_apply_%s_multi", len(xs), arr, 256, 32, _lib.ptr(inp["gamma"]), _lib.ptr(inp["beta"]), 1e-5, 1,
                  _lib.current_stream_ptr())
        return ys

    def fn(inp, run):
        st = _lib.current_stream_ptr()
        stats = [torch.zeros((n, 32, 2), dtype=torch.float64, device=cuda) for (n, _, _) in shapes]
        for i, (n, h, w) in enumerate(shapes):
            eng._call("orp_gn_stats_%s", _lib.ptr(inp["x%d" % i]), n, h * w, 256, 32, _lib.ptr(stats[i]), st)
        ys = apply(inp, run, [0, 1], stats, [inp["up0"].data_ptr(), None])
        fixed = apply(inp, run, [1], [inp["s1"]], [None])
        y = _act(run, eng, 2, 17, 21, 64)
        eng._call("orp_maxpool3x3s2_%s", _lib.ptr(inp["p"]), 2, 33, 41, 64, _lib.ptr(y), st)
        return stats + ys + fixed + [y]
    side_stream_check(cuda, src, fn, tol=(0, 1, 2, 3))


# ---------------------------------------------------------------------------------------------- layouts, DCN offsets
@gpu
def test_layout_side_stream(cuda):
    """the boundary conversions of the split format, the NCHW <-> NHWC transpose and the head's DCN offsets"""
    g = torch.Generator().manual_seed(51)
    src = {"x": torch.randn(2, 13, 17, 96, generator=g).to(cuda), "nchw": torch.randn(2, 96, 13, 17, generator=g).to(cuda),
           "p0": torch.randn(2, 20, 28, 18, generator=g).to(cuda), "p1": torch.randn(2, 10, 14, 18, generator=g).to(cuda)}
    src["s"] = torch.empty(2, 13, 17, 2, 96, dtype=torch.float16, device=cuda)
    _lib.check(_lib.lib().orp_split_from_f32(_lib.ptr(src["x"]), 2 * 13 * 17, 96, _lib.ptr(src["s"]), _lib.current_stream_ptr()), "split")
    torch.cuda.synchronize()
    base = (ctypes.c_float * 18)(*[float(v) for v in np.stack([np.repeat([-1., 0., 1.], 3), np.tile([-1., 0., 1.], 3)], 1).reshape(-1)])

    def fn(inp, run):
        l, st = _lib.lib(), _lib.current_stream_ptr()
        a = run.out((2, 13, 17, 2, 96), torch.float16)
        _lib.check(l.orp_split_from_f32(_lib.ptr(inp["x"]), 2 * 13 * 17, 96, _lib.ptr(a), st), "orp_split_from_f32")
        b = run.out((2, 13, 17, 96), torch.float32)
        _lib.check(l.orp_split_to_f32(_lib.ptr(inp["s"]), 2 * 13 * 17, 96, _lib.ptr(b), st), "orp_split_to_f32")
        c = run.out((2, 13 * 17, 96), torch.float32)
        _lib.check(l.orp_transpose_f32(_lib.ptr(inp["nchw"]), 2, 96, 13 * 17, _lib.ptr(c), st), "orp_transpose_f32")
        d = run.out((2, 13, 17, 2, 96), torch.float16)
        _lib.check(l.orp_nchw_f32_to_split(_lib.ptr(inp["nchw"]), 2, 96, 13 * 17, _lib.ptr(d), st), "orp_nchw_f32_to_split")
        offs = [run.out(inp[k].shape, torch.float32) for k in ("p0", "p1")]
        pa = (ctypes.c_void_p * 2)(inp["p0"].data_ptr(), inp["p1"].data_ptr())
        po = (ctypes.c_void_p * 2)(*[o.data_ptr() for o in offs])
        ne = (ctypes.c_longlong * 2)(inp["p0"].numel(), inp["p1"].numel())
        _lib.check(l.orp_dcn_offsets_multi(2, pa, po, ne, 0.3, base, st), "orp_dcn_offsets_multi")
        return [a, b, c, d] + offs
    side_stream_check(cuda, src, fn)


# ---------------------------------------------------------------------------------------------------------- Swin-T
@gpu
@pytest.mark.parametrize("prec", ["f16x3", "bf16"])
def test_swin_side_stream(cuda, prec):
    """the Swin-T backbone (patch embedding from float, uint8 and padded uint8 images, LayerNorm, shifted-window
    attention, patch merging, GELU MLPs) and the P6 / P7 subsampling: no GroupNorm, so bitwise"""
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    from orientedreppoints_b200.swin import random_swin_state_dict
    det = OrientedRepPointsDetector(random_swin_state_dict(0), "swin_tiny", cuda, prec)
    sw = det.swin
    g = torch.Generator().manual_seed(61)
    src = {"img": torch.randint(0, 256, (2, 128, 192, 3), generator=g, dtype=torch.uint8).to(cuda),
           "valid": torch.tensor([[128, 192], [101, 77]], dtype=torch.int32).to(cuda),
           "f": torch.randn(1, 3, 96, 128, generator=g).to(cuda)}
    torch.cuda.synchronize()

    def fn(inp, run):
        a = sw.forward(inp["img"], det.img_norm_cfg)
        b = sw.forward(inp["img"], det.img_norm_cfg, inp["valid"])
        c = sw.forward(inp["f"])
        return a + b + c + [sw.subsample2(a[2]), sw.subsample2(sw.subsample2(a[1]))]
    side_stream_check(cuda, src, fn)
    if prec == "f16x3":
        assert det.eng.overflow_count() == 0


# ---------------------------------------------------------------------------------------------------------- NMS
@gpu
@pytest.mark.parametrize("mode,order,union,seg", [
    ("exact64", _lib.ORP_ORDER_INDEX_ASC, _lib.ORP_UNION_NAN_KEEPS, False),
    ("exact64", _lib.ORP_ORDER_SCORE_DESC, _lib.ORP_UNION_GUARD, True),
    ("exact64", _lib.ORP_ORDER_SCORE_DESC, _lib.ORP_UNION_NAN_SUPPRESSES, True),
    ("exact64", _lib.ORP_ORDER_INDEX_ASC, _lib.ORP_UNION_NAN_SUPPRESSES_ALL, False),
    ("compat32", _lib.ORP_ORDER_INDEX_ASC, _lib.ORP_UNION_NAN_KEEPS, True),
    ("compat32", _lib.ORP_ORDER_SCORE_DESC, _lib.ORP_UNION_GUARD, False),
])
def test_rnms_side_stream(cuda, golden, mode, order, union, seg):
    """orp_rnms over the clustered golden set (dense overlaps: the candidate list outgrows its first allocation, so the
    call's one host round trip - on the caller's stream - is taken); the flags / no-sync paths run inside
    orp_head_postprocess and orp_result_merge (test_postprocess_merge_eval_side_stream)"""
    from orientedreppoints_b200.ops import rnms_indices
    dets = torch.from_numpy(golden("nms_clustered.npz")["dets"]).to(cuda)
    n = dets.shape[0]
    src = {"dets": dets, "seg": (torch.arange(n, device=cuda, dtype=torch.int32) % 3)}

    def fn(inp, run):
        keep, cnt = rnms_indices(inp["dets"], 0.3, segments=inp["seg"] if seg else None, mode=mode, union_mode=union,
                                 order=order, return_count_tensor=True)
        plan = _lib.rnms_last_plan()
        assert plan["order"] == order and plan["union_mode"] == union and plan["n"] == n
        return [cnt, keep[:int(cnt.item())]]
    side_stream_check(cuda, src, fn)


# ------------------------------------------------------------------------------- post-processing, merge, evaluation
def _head_outputs(g, b, sizes, dev):
    cls = [(torch.randn(b, h, w, 15, generator=g) * 2 - 3).to(dev) for (h, w) in sizes]
    ref = [(torch.randn(b, h, w, 18, generator=g) * 1.5).to(dev) for (h, w) in sizes]
    return cls, ref


@gpu
def test_postprocess_merge_eval_side_stream(cuda):
    """the detection tail of the benchmark on a side stream: orp_head_postprocess (its NMS runs without host sync), the
    aug variant over two views, packing, ResultMerge (flags-out NMS), Task1 and mAOE evaluation, poly2rbox_v3"""
    from orientedreppoints_b200.core.get_bboxes import get_bboxes_aug_fused, get_bboxes_fused
    from orientedreppoints_b200.detector import STRIDES
    from orientedreppoints_b200.dota import aoe_evaluation, evaluation
    from orientedreppoints_b200.dota.result_merge import merge_packed
    from orientedreppoints_b200.gather import pack
    g = torch.Generator().manual_seed(71)
    sizes = [(32, 40), (16, 20), (8, 10), (4, 5), (2, 3)]
    cfg = dict(nms_pre=1000, min_bbox_size=0, score_thr=0.05, nms=dict(type='rnms', iou_thr=0.4), max_per_img=300)
    b = 3
    cls, ref = _head_outputs(g, b, sizes, cuda)
    cls2, ref2 = _head_outputs(g, b, sizes, cuda)
    src = {"c%d" % i: t for i, t in enumerate(cls + cls2)}
    src.update({"r%d" % i: t for i, t in enumerate(ref + ref2)})
    metas = [dict(scale_factor=0.75) for _ in range(b)]
    metas2 = [dict(scale_factor=0.75, flip=True, img_shape=(320, 300, 3)) for _ in range(b)]
    L = len(sizes)

    def post(inp, run):
        d, l, c = get_bboxes_fused([inp["c%d" % i] for i in range(L)], [inp["r%d" % i] for i in range(L)], STRIDES, metas, cfg, True)
        da, la, ca = get_bboxes_aug_fused([[inp["c%d" % i] for i in range(L)], [inp["c%d" % (L + i)] for i in range(L)]],
                                          [[inp["r%d" % i] for i in range(L)], [inp["r%d" % (L + i)] for i in range(L)]],
                                          STRIDES, [metas, metas2], cfg, False)
        plan = _lib.rnms_last_plan()
        assert plan["no_sync"] == 1
        buf, _ = pack(d, l, c)
        return [d, l, c, da, la, ca, buf]
    d, l, c, _, _, _, packed = side_stream_check(cuda, src, post)
    counts = c.cpu().tolist()
    assert min(counts) > 0, counts

    tn = b
    xy = torch.tensor([[0, 0], [824, 0], [0, 824]], dtype=torch.int32).to(cuda)
    src = {"packed": packed, "slot": torch.arange(tn, dtype=torch.int32).to(cuda), "xy": xy,
           "rate": torch.ones(tn, dtype=torch.float64).to(cuda), "img": torch.tensor([0, 0, 1], dtype=torch.int32).to(cuda)}

    def merge(inp, run):
        m = merge_packed(inp["packed"], inp["slot"], inp["xy"], inp["rate"], inp["img"], 2, max_rows=tn * (packed.shape[1] - 1))
        return [m.cls, m.img, m.score, m.quad, m.src_row]
    merged = side_stream_check(cuda, src, merge)
    m_cls, m_img, m_score, m_quad = merged[:4]
    nd = m_cls.shape[0]
    assert nd > 0

    # ground truth: a perturbed half of the survivors plus boxes of their own, difficult flags alternating
    sel = torch.arange(0, nd, 2, device=cuda)
    gq = torch.cat([m_quad[sel] + torch.randn(sel.shape[0], 8, generator=g, dtype=torch.float64).to(cuda),
                    torch.rand(7, 8, generator=g, dtype=torch.float64).to(cuda) * 900])
    gc = torch.cat([m_cls[sel], torch.randint(0, 15, (7,), generator=g, dtype=torch.int32).to(cuda)])
    gi = torch.cat([m_img[sel], torch.randint(0, 2, (7,), generator=g, dtype=torch.int32).to(cuda)])
    gd = (torch.arange(gc.shape[0], device=cuda) % 3 == 0).to(torch.uint8)
    src = {"dc": m_cls, "di": m_img, "ds": m_score, "dq": m_quad, "gc": gc, "gi": gi, "gq": gq, "gd": gd}
    torch.cuda.synchronize()

    def evals(inp, run):
        ins = [inp[k] for k in ("dc", "di", "ds", "dq", "gc", "gi", "gq", "gd")]
        t1, _ = evaluation._launch(ins, 15, 2, 0.5, True, cuda)
        t2, _ = evaluation._launch(ins, 15, 2, 0.5, False, cuda)
        ao, _ = aoe_evaluation._launch(ins[:7], 15, 2, 0.5, cuda)
        rb = run.out((nd, 5), torch.float64)
        _lib.check(_lib.lib().orp_poly2rbox_v3(_lib.ptr(inp["dq"]), nd, _lib.ptr(rb), _lib.current_stream_ptr()), "orp_poly2rbox_v3")
        return [t1, t2, ao, rb]
    side_stream_check(cuda, src, evals)


# ------------------------------------------------------------------------------------------------ resize, split tiles
@gpu
def test_resize_split_side_stream(cuda):
    """the test pipeline's resize (+ flip, + pad) and the DOTA tiling of a large image"""
    from orientedreppoints_b200.datasets.pipelines import device_tables
    g = torch.Generator().manual_seed(81)
    src = {"img": torch.randint(0, 256, (2, 301, 417, 3), generator=g, dtype=torch.uint8).to(cuda),
           "big": torch.randint(0, 256, (1500, 1300, 3), generator=g, dtype=torch.uint8).to(cuda),
           "org": torch.tensor([[0, 0], [824, 0], [0, 476], [824, 476]], dtype=torch.int32).to(cuda)}
    xt, yt = device_tables(cuda, (301, 417), (480, 664))
    torch.cuda.synchronize()

    def fn(inp, run):
        l, st = _lib.lib(), _lib.current_stream_ptr()
        outs = []
        for flip in (0, 1):
            y = run.out((2, 512, 672, 3), torch.uint8)
            _lib.check(l.orp_resize_u8(_lib.ptr(inp["img"]), 2, 301, 417, 3, _lib.ptr(y), 480, 664, 512, 672, flip, _lib.ptr(xt),
                                       _lib.ptr(yt), st), "orp_resize_u8")
            outs.append(y)
        t = run.out((4, 1024, 1024, 3), torch.uint8)
        _lib.check(l.orp_split_tiles_u8(_lib.ptr(inp["big"]), 1500, 1300, 3, _lib.ptr(inp["org"]), 4, 1024, _lib.ptr(t), st),
                   "orp_split_tiles_u8")
        return outs + [t]
    side_stream_check(cuda, src, fn)


# ------------------------------------------------------------------------------------------------------- geometry
@gpu
def test_geometry_side_stream(cuda):
    from oracle import pyoracle as po
    g = torch.Generator().manual_seed(91)
    n, k = 700, 90
    quads = torch.from_numpy(po.gen_rotated_boxes(n, seed=3)[:, :8].astype(np.float32)).to(cuda)
    src = {"pts": (torch.randn(n, 18, generator=g) * 4 + 100).to(cuda), "ctr": (torch.rand(n, 2, generator=g) * 500).to(cuda),
           "b5": torch.cat([torch.rand(n, 2, generator=g) * 300, torch.rand(n, 2, generator=g) * 40 + 2,
                            torch.rand(n, 1, generator=g) * 3.1], 1).to(cuda),
           "qa": quads, "p8": quads[:k].double().contiguous(), "q8": quads[k:2 * k].double().contiguous()}
    src["q18"] = (src["pts"][:, :8] + torch.randn(n, 8, generator=g).to(cuda) * 3).contiguous()
    torch.cuda.synchronize()

    def fn(inp, run):
        l, st = _lib.lib(), _lib.current_stream_ptr()
        r = run.out((n, 8), torch.float32)
        hull = run.out((n, 9), torch.int32)
        _lib.check(l.orp_minarearect(_lib.ptr(inp["pts"]), n, _lib.ptr(r), _lib.ptr(hull), 8.0, _lib.ptr(inp["ctr"]), st), "minarearect")
        bi = run.out((n, k), torch.float32)
        _lib.check(l.orp_box_iou_rotated(_lib.ptr(inp["b5"]), n, _lib.ptr(inp["b5"]), k, _lib.ptr(bi), st), "box_iou_rotated")
        po_ = run.out((n, k), torch.float32)
        _lib.check(l.orp_poly_overlaps(_lib.ptr(inp["b5"]), n, _lib.ptr(inp["b5"]), k, _lib.ptr(po_), st), "poly_overlaps")
        outs = [r, hull, bi, po_]
        for mode in (_lib.ORP_NMS_EXACT64, _lib.ORP_NMS_COMPAT32):
            q = run.out((n, k), torch.float32)
            _lib.check(l.orp_quad_iou_matrix(_lib.ptr(inp["qa"]), n, _lib.ptr(inp["qa"]), k, mode, _lib.ORP_UNION_GUARD, _lib.ptr(q), st),
                       "quad_iou_matrix")
            outs.append(q)
        f = run.out((k,), torch.float64)
        _lib.check(l.orp_iou_poly_f64_pairs(_lib.ptr(inp["p8"]), _lib.ptr(inp["q8"]), k, _lib.ptr(f), st), "iou_poly_f64_pairs")
        ci = run.out((n, k), torch.float32)
        _lib.check(l.orp_convex_iou(_lib.ptr(inp["pts"]), n, _lib.ptr(inp["qa"]), k, _lib.ptr(ci), st), "convex_iou")
        gi = run.out((n, 19), torch.float32)
        _lib.check(l.orp_convex_giou(_lib.ptr(inp["pts"]), _lib.ptr(inp["q18"]), n, _lib.ptr(gi), st), "convex_giou")
        return outs + [f, ci, gi]
    side_stream_check(cuda, src, fn)


# ------------------------------------------------------------------------------------------------------ fp32 engine
@gpu
def test_f32_engine_side_stream(cuda):
    """the CUDA-core engine: convolution with residual and GroupNorm statistics (atomics), DCNv1 / DCNv2, GroupNorm apply
    with the upsampled add from fixed statistics, max-pool"""
    g = torch.Generator().manual_seed(101)
    n, h, w, cin, cout = 2, 21, 27, 64, 128
    src = {"x": torch.randn(n, h, w, cin, generator=g).to(cuda),
           "w": (torch.randn(cout, 3, 3, cin, generator=g) * 0.05).to(cuda), "b": torch.randn(cout, generator=g).to(cuda),
           "res": torch.randn(n, h, w, cout, generator=g).to(cuda), "off": (torch.randn(n, h, w, 18, generator=g) * 2).to(cuda),
           "mask": torch.rand(n, h, w, 9, generator=g).to(cuda),
           "gx": torch.randn(n, 18, 26, 256, generator=g).to(cuda), "up": torch.randn(n, 9, 13, 256, generator=g).to(cuda),
           "gamma": torch.randn(256, generator=g).to(cuda), "beta": torch.randn(256, generator=g).to(cuda),
           "stats": torch.cat([torch.randn(n, 32, 1, generator=g, dtype=torch.float64) * 100,
                               torch.rand(n, 32, 1, generator=g, dtype=torch.float64) * 1e4 + 2e4], 2).to(cuda)}
    torch.cuda.synchronize()

    def fn(inp, run):
        l, st = _lib.lib(), _lib.current_stream_ptr()
        y = run.out((n, h, w, cout), torch.float32)
        stats = torch.zeros((n, 32, 2), dtype=torch.float64, device=cuda)
        _lib.check(l.orp_conv2d_f32(_lib.ptr(inp["x"]), n, h, w, cin, _lib.ptr(inp["w"]), cout, 3, 3, 1, 1, _lib.ptr(inp["b"]),
                                    _lib.ptr(inp["res"]), 1, _lib.ptr(y), _lib.ptr(stats), 32, st), "orp_conv2d_f32")
        outs = [y, stats]
        for m in (None, inp["mask"]):
            d = run.out((n, h, w, cout), torch.float32)
            _lib.check(l.orp_deform_conv2d_f32(_lib.ptr(inp["x"]), n, h, w, cin, _lib.ptr(inp["off"]), _lib.ptr(m), _lib.ptr(inp["w"]),
                                               cout, 3, 3, 1, 1, 1, _lib.ptr(inp["b"]), 1, _lib.ptr(d), st), "orp_deform_conv2d_f32")
            outs.append(d)
        gy = run.out((n, 18, 26, 256), torch.float32)
        _lib.check(l.orp_gn_apply_f32(_lib.ptr(inp["gx"]), n, 18, 26, 256, _lib.ptr(inp["stats"]), 32, _lib.ptr(inp["gamma"]),
                                      _lib.ptr(inp["beta"]), 1e-5, 1, _lib.ptr(inp["up"]), _lib.ptr(gy), st), "orp_gn_apply_f32")
        mp = run.out((n, 9, 13, 256), torch.float32)
        _lib.check(l.orp_maxpool3x3s2_f32(_lib.ptr(inp["gx"]), n, 18, 26, 256, _lib.ptr(mp), st), "orp_maxpool3x3s2_f32")
        return outs + [gy, mp]
    side_stream_check(cuda, src, fn, tol=(1,))


# ------------------------------------------------------------------------------------------ f16x3 overflow counter
def _saturating_case(cuda):
    """test_conv_f16x3_small_weights_and_overflow_flag's overflow launch: weights * 3e4 on inputs * 100"""
    from orientedreppoints_b200.detector import ConvLayer
    from orientedreppoints_b200.engine_tc import EngineTCSplit
    eng = EngineTCSplit(cuda)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(1, 256, 24, 24, generator=g)
    wt = torch.randn(256, 256, 3, 3, generator=g) * 0.01
    L = ConvLayer(wt * 3e4, None, 1, 1, cuda)
    xs = eng.from_float((x * 100).permute(0, 2, 3, 1).contiguous())
    eng.overflow_count()                             # the counter is one per process: start from zero
    eng.conv(xs, L)                                  # weight upload, and the number of events one launch records
    want = eng.overflow_count()
    assert want > 0
    return eng, L, xs, want


@gpu
def test_overflow_count_side_stream(cuda):
    """a saturating f16x3 launch on a side stream behind a spin, then overflow_count() with no synchronisation: the read
    is ordered after the launch, so it reports the launch's events (a read on the legacy default stream returns 0
    here, before the launch has run)"""
    eng, L, xs, want = _saturating_case(cuda)
    s = torch.cuda.Stream(device=cuda)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(SPIN)
        eng.conv(xs, L)
        got = eng.overflow_count()
        after = eng.overflow_count()
    assert got == want, (got, want)
    assert after == 0


@gpu
def test_overflow_count_reset_keeps_running_launch(cuda):
    """a reset issued on one stream while a saturating launch is still queued on another loses none of its events: they
    are in the next read"""
    eng, L, xs, want = _saturating_case(cuda)
    s = torch.cuda.Stream(device=cuda)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(SPIN)
        eng.conv(xs, L)
    early = eng.overflow_count()                     # on the default stream: not ordered after s
    s.synchronize()
    late = eng.overflow_count()
    assert early + late == want, (early, late, want)


# ----------------------------------------------------------------------------------------------------- host threads
_NMS_PLAN_FIELDS = ("lazy", "R", "seg_limit", "no_sync", "flags_out", "union_mode", "order", "n", "cap_first")


def _step(det, img, rec, graph):
    """one simple_test(return_tensors="padded") of det on the current stream -> (dense outputs, padded detections,
    get_bboxes_fused of those dense outputs, last NMS plan of this thread, last convolution plan of this thread)"""
    from orientedreppoints_b200.core.get_bboxes import get_bboxes_fused
    from orientedreppoints_b200.detector import STRIDES
    padded = det.simple_test(img, return_tensors="padded")
    nms = _lib.rnms_last_plan()
    tc = None if graph else _lib.tc_last_plan()        # a replay launches no convolution from this thread
    outs = det._g_out[0] if graph else rec["outs"]
    again = get_bboxes_fused([o[0] for o in outs], [o[2] for o in outs], STRIDES, [dict(scale_factor=1.0)] * img.shape[0],
                             det.test_cfg, False)
    dense = [t.clone() for lvl in outs for t in lvl]
    return dense, [t.clone() for t in padded], [t.clone() for t in again], {k: nms[k] for k in _NMS_PLAN_FIELDS}, tc


@gpu
def test_two_threads_two_detectors(cuda):
    """two f16x3 R-50 detectors, batch 2 at 1024^2, each on its own stream in its own host thread, simple_test at the same
    time: each thread's dense outputs are its serial ones (REPLAY_TOL: GroupNorm sums), its padded detections are
    get_bboxes_fused of its own dense outputs bit for bit, and the library's per-thread plan records describe that thread's
    own last NMS and convolution (the detectors differ in nms_pre, so their NMS plans differ).  Then one detector runs
    eagerly while the other replays its captured graph."""
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    from orientedreppoints_b200.weights import random_state_dict
    dets, recs = [], []
    for i in range(2):
        d = OrientedRepPointsDetector(random_state_dict(50, seed=i, reference_init=False), 50, cuda, "f16x3",
                                      test_cfg=dict(score_thr=0.02, nms_pre=(2000, 1000)[i]))
        rec = {}

        def fwd(img, valid_hw, _eager=d._forward_dense_opt, _rec=rec):
            r = _eager(img, valid_hw)
            _rec["outs"] = r[0]
            return r
        d._forward_dense_opt = fwd                     # keep the dense outputs simple_test post-processes
        dets.append(d)
        recs.append(rec)
    imgs = [torch.randn(2, 3, 1024, 1024, generator=torch.Generator().manual_seed(7 + i)).to(cuda) for i in range(2)]
    serial = [_step(dets[i], imgs[i], recs[i], False) for i in range(2)]
    torch.cuda.synchronize()
    assert serial[0][3] != serial[1][3]
    for dense, padded, again, _, tc in serial:
        assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(padded, again))
        assert tc["Cout"] == 18 and tc["nprob"] == 5 and tc["residual"] == 2, tc     # the refine head closes the graph
    iters = 3

    def worker(i, res, graph):
        try:
            s = torch.cuda.Stream(device=cuda)
            with torch.cuda.device(cuda), torch.cuda.stream(s):
                res[i] = [_step(dets[i], imgs[i], recs[i], graph) for _ in range(iters)]
                s.synchronize()
        except BaseException as e:                       # raised again in the main thread
            res[i] = e

    def run_pair(graph_second):
        res = [None, None]
        ts = [threading.Thread(target=worker, args=(i, res, graph_second and i == 1)) for i in range(2)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        for i, r in enumerate(res):
            if isinstance(r, BaseException):
                raise r
            assert len(r) == iters
            for dense, padded, again, nms, tc in r:
                for a, b in zip(dense, serial[i][0]):
                    assert _rel(a, b) < REPLAY_TOL, (i, _rel(a, b))
                for a, b in zip(padded, again):
                    assert torch.equal(_bits(a), _bits(b)), i
                assert nms == serial[i][3], (i, nms, serial[i][3])
                assert tc is None or tc == serial[i][4], (i, tc)
    run_pair(False)
    dets[1].capture(tuple(imgs[1].shape))
    torch.cuda.synchronize()
    run_pair(True)
    assert dets[0].eng.overflow_count() == 0
