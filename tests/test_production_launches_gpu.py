"""GPU: every tensor-core convolution launch of the benchmark workloads checked at its production shape against fp64, and
the benchmarked step (16 uint8 tiles -> stem_u8 -> the dense graph replayed as a CUDA graph -> fused post-processing) tile
by tile against the fp64 reference graph.

tests/test_conv_plans_gpu.py checks one case per launch plan at the smallest shape that reaches it.  At production size a
persistent CTA walks 60+ tiles, M tiles cross up to 15 image boundaries, addresses into the ~1 GiB f16x3 activations reach
values no small case reaches, and the head's deformable convolution samples learned offsets.  This file checks the launches
where they happen.

- test_every_conv_launch_vs_fp64: one eager forward_dense per benchmark workload (R-50 f16x3 x16 and x1, R-101 f16x3 x4,
  Swin-T f16x3 / bf16 x8, R-50 bf16 x16, and R-101 x4 / Swin-T x8 at the test scale: 1024^2 uint8 tiles through the
  config's test pipeline to 960^2, with the valid extents), the input the bench's own seeded uint8 tiles.  The weights are
  random_state_dict(reference_init=False) (randomised norm scales, so that no conv3 launch is trivially zero) and the Swin-T
  state dict of the bench; the launch plans must be those of the bench's detector, launch for launch.  The engine's
  conv_multi, deform_conv_multi, _stem_conv_s2d and group_conv are wrapped; after each real call the output is compared with an fp64
  reference built from the exact operands (the input as the engine holds it, raw fp32 weights in f16x3 or bf16-rounded
  ones in bf16, bias, the 16-bit or fp32 residual, the activation, the production DCN offsets through deform_conv_ref, the
  stem's image decoded from its space-to-depth operand and convolved at the stem layer's stride and padding: ResNet's 7x7 or
  HRNet's 3x3 conv1), image by image relative to that image's max, with the tolerances
  of test_conv_plans_gpu.py; GroupNorm sums against fp64 sums.  The references are computed one image at a time on the
  device, so that the fp64 im2col of a 16 x 128^2 deformable convolution is never resident at once.  Then the call is
  launched twice more into guarded outputs prefilled with two NaN patterns: both results bitwise equal to the first output,
  guards untouched.  Counters on _launch, _conv_splitk and the stem and grouped entry points make sure that no launch
  escapes the checker.  tests/test_backbone_launches_gpu.py runs the same checker on the ResNeXt, HRNet, DCN-stage and
  GeneralizedAttention graphs.
- test_benchmarked_step_r50_x16: the headline configuration exactly as bench_tile.run builds it, with the reference's
  initialisation and with randomised norm scales.  Graph replays equal the eager pass (1e-5) and each other; every tile
  of the 16-tile replay is within north_star's 1e-4 of the fp64 graph run on that tile alone (normalised in fp64 on the
  host); the padded detections of the bench's call equal the fused post-processing of the frozen dense outputs bit for bit
  and, on tiles 0 and 15, the op-by-op mirror (labels and scores exact, coordinates 1e-3 px).  With randomised norm scales
  tiles 0 and 15 also match the oracle post-processing of the fp64 graph's outputs.  (With the reference's initialisation
  the network is near-degenerate: 2.8 % of tile 0's detections, at scores within 2e-8 of the oracle's, fall the other way
  in the NMS, so that content match is not made there.)
- test_benchmarked_step_other_workloads: R-101 f16x3 x4 and Swin-T f16x3 x8 as bench_tile.run_config builds them, every
  tile of the replay against the fp64 graph."""
import ctypes
import time

import pytest
import torch
import torch.nn.functional as F

from orientedreppoints_b200 import _lib

from conv_plan_cases import signature
from test_conv_plans_gpu import (BF16_F32_TOL, BF16_TOL, DCN_BF16_TOL, DCN_F16X3_TOL, GN_TOL, OP_TOL, PATTERNS, WORKLOADS,
                                 Guarded, _rel)

pytestmark = pytest.mark.gpu

DENSE_TOL = 1e-4                                  # north_star: dense outputs within 1e-4 of the fp64 reference graph
REPLAY_TOL = 1e-5                                 # graph replay against eager: GroupNorm sums are atomics, bits may differ
GROUP_BF16_TOL = 1.5e-2                           # bf16 grouped conv2: the launch tolerance of tests/test_resnext_gpu.py
TEST_SCALE = [("r101", "f16x3", 4), ("swin_tiny", "f16x3", 8)]     # bench_tile.run_test_scale


# ------------------------------------------------------------------------------------------------------------- helpers
def _nchw64(t):
    """NHWC fp32 -> NCHW fp64"""
    return t.permute(0, 3, 1, 2).double()


def _act(v, act):
    return torch.relu(v) if act is True or act == 1 else (F.gelu(v) if act == 2 else v)


def _hrnet_names(hr, names):
    """HRNetGraph's layers by the reference's module paths (hrnet.py), HRFPN's reduction slices and fpn_convs"""
    names[id(hr.conv2)] = "conv2"
    for b, blk in enumerate(hr.layer1):
        for k, L in enumerate(blk["convs"]):
            names[id(L)] = "layer1.%d.conv%d" % (b, k + 1)
        if blk["ds"] is not None:
            names[id(blk["ds"])] = "layer1.%d.downsample" % b
    for s, (trans, mods) in enumerate(zip(hr.transitions, hr.stages), 1):
        for i, chain in enumerate(trans):
            for j, L in enumerate(chain or ()):
                names[id(L)] = "transition%d.%d.%d" % (s, i, j)
        for m, (branches, fuse) in enumerate(mods):
            p = "stage%d.%d." % (s + 1, m)
            for br, blocks in enumerate(branches):
                for k, (c1, c2) in enumerate(blocks):
                    names[id(c1)], names[id(c2)] = p + "branches.%d.%d.conv1" % (br, k), p + "branches.%d.%d.conv2" % (br, k)
            for i, row in enumerate(fuse):
                for j, path in enumerate(row):
                    for k, L in enumerate(path or ()):
                        names[id(L)] = p + "fuse_layers.%d.%d.%d" % (i, j, k)
    for i, L in enumerate(hr.reduce):
        names[id(L)] = "reduction_conv.%d" % i
    for i, L in enumerate(hr.fpn):
        names[id(L)] = "fpn_convs.%d" % i


def _layer_names(det):
    """id(ConvLayer) -> the layer's name, for every convolution of the detector: ResNet / ResNeXt (with deformable conv2 and
    their conv_offset, and GeneralizedAttention blocks), Swin, HRNet + HRFPN, the FPN and the head"""
    names = {}
    if getattr(det, "swin", None) is not None:
        sw = det.swin
        names[id(sw.embed)] = "patch_embed"
        for i, stage in enumerate(sw.blocks):
            for j, blk in enumerate(stage):
                for k in ("qkv", "proj", "fc1", "fc2"):
                    names[id(blk[k])] = "stage%d.%d.%s" % (i, j, k)
        for i, m in enumerate(sw.merges):
            names[id(m["red"])] = "merge%d" % i
    else:
        names[id(det.stem)] = "stem"
    if getattr(det, "hrnet", None) is not None:
        _hrnet_names(det.hrnet, names)
    for li, stage in enumerate(getattr(det, "blocks", ())):
        for b, blk in enumerate(stage):
            for k in ("c1", "c2", "c3", "ds", "off"):
                if blk.get(k) is not None:
                    names[id(blk[k])] = "layer%d.%d.%s" % (li + 1, b, k)
            att = blk.get("att")
            for k in ("q", "kv", "proj"):
                if att is not None and getattr(att, k) is not None:
                    names[id(getattr(att, k))] = "layer%d.%d.att.%s" % (li + 1, b, k)
    for i, (L, _) in enumerate(getattr(det, "lat", ())):
        names[id(L)] = "lateral%d" % i
    for i, (L, _) in enumerate(getattr(det, "fpn", ())):
        names[id(L)] = "fpn%d" % i
    for i, ((lc, _), (lr, _)) in enumerate(zip(det.cls_convs, det.reg_convs)):
        names[id(lc)], names[id(lr)] = "cls_convs%d" % i, "reg_convs%d" % i
    for k in ("cls_dcn", "cls_out", "init_conv", "init_out", "ref_dcn", "ref_out"):
        names[id(getattr(det, k))] = k
    return names


def _where(y, ref, tol):
    """(channel, row, column) of the first element past tol x max, and of the largest error"""
    d = (y - ref).abs()[0]
    bad = (d > tol * float(ref.abs().max())).reshape(-1).nonzero()
    shape = d.shape

    def unravel(i):
        c, r = divmod(i, shape[1] * shape[2])
        return (c,) + divmod(r, shape[2])
    return unravel(int(bad[0])) if bad.numel() else None, unravel(int(d.reshape(-1).argmax()))


class LaunchChecker:
    """wraps the tensor-core convolution methods of one detector's engine; every call is checked against fp64 and for
    write-once stores as it happens (see the module docstring)"""
    conv_margin = 1.0                         # factor on the f16x3 convolution tolerance OP_TOL * max(1, K / 4096)

    def __init__(self, det, name):
        self.det, self.eng, self.name = det, det.eng, name
        self.split = self.eng.name == "f16x3"
        self.names = _layer_names(det)
        self.inside = False                   # within a checked call
        self.replaying = False                # re-launching a checked call into guarded outputs
        self.rec = []                         # low-level launches of the current checked call
        self.low = 0                          # low-level launches of the forward pass
        self.escaped = []                     # ... made outside a checked call
        self.checked = 0
        self.sigs = []                        # plan signature of every checked orp_conv2d / stem launch, in order
        self.layers = []                      # ... and the name of its layer
        self.worst = {}                       # kind -> (rel err, tol, where)
        e = self.eng
        self.orig = {m: getattr(e, m) for m in ("conv_multi", "deform_conv_multi", "_stem_conv_s2d", "group_conv", "_launch",
                                                "_conv_splitk", "_call")}
        e.conv_multi, e.deform_conv_multi, e._stem_conv_s2d = self._conv_multi, self._deform_conv_multi, self._stem_conv_s2d
        e.group_conv = self._group_conv
        e._launch, e._conv_splitk, e._call = self._counted("_launch"), self._counted("_conv_splitk"), self._call

    # ----------------------------------------------------------------------------------------------- counters
    def _saw(self, kind, a, kw):
        if self.replaying:
            return
        self.low += 1
        if self.inside:
            self.rec.append((kind, a, kw))
        else:
            self.escaped.append(kind)

    def _counted(self, kind):
        fn = self.orig[kind]

        def wrapper(*a, **kw):
            self._saw(kind, a, kw)
            return fn(*a, **kw)
        return wrapper

    def _call(self, name, *args):
        if name in ("orp_stem_conv_s2d_%s", "orp_group_conv2d_%s"):
            self._saw("stem" if name == "orp_stem_conv_s2d_%s" else "group", (name,) + args, {})
        return self.orig["_call"](name, *args)

    def _run(self, method, *a):
        assert not self.inside, "a checked call inside another"
        self.inside, self.rec = True, []
        try:
            out = self.orig[method](*a)
        finally:
            self.inside = False
        plan = _lib.tc_last_plan()
        torch.cuda.synchronize()
        assert len(self.rec) == 1, "%s: %d low-level launches in one call" % (method, len(self.rec))
        return out, plan, self.rec[0]

    # --------------------------------------------------------------------------------------------- checked calls
    def _conv_multi(self, xs, L, relu=False, residual=None, out_f32=False, residual_f32=None, stats=None):
        ys, plan, low = self._run("conv_multi", xs, L, relu, residual, out_f32, residual_f32, stats)
        wd, bias = self._weights(L), None if L.bias is None else L.bias.double().view(1, -1, 1, 1)
        K = L.w_raw.shape[1] * L.w_raw.shape[2] * L.w_raw.shape[3]

        def ref(i, j):
            r = F.conv2d(self._held(xs[i][j:j + 1]), wd, None, L.stride, L.pad)
            if bias is not None:
                r = r + bias
            if residual is not None:
                r = r + self._held(residual[i][j:j + 1])
            if residual_f32 is not None:
                r = r + _nchw64(residual_f32[i][j:j + 1])
            return _act(r, relu)
        if self.split:
            tol = OP_TOL * max(1.0, K / 4096.0) * self.conv_margin
        else:
            tol = BF16_F32_TOL if out_f32 else BF16_TOL
        kind = "split-K" if low[0] == "_conv_splitk" else ("fp32-out" if out_f32 else "conv")
        self._check(kind, L, ys, ref, tol, plan, low, stats=stats, K=K, out_f32=out_f32)
        return ys

    def _deform_conv_multi(self, xs, offsets, L, relu=False, masks=None):
        from oracle import torch_reference as tr
        ys, plan, low = self._run("deform_conv_multi", xs, offsets, L, relu, masks)
        wd, bias = self._weights(L), None if L.bias is None else L.bias.double().view(1, -1, 1, 1)

        def ref(i, j):
            off = offsets[i][j:j + 1].permute(0, 3, 1, 2).double()
            m = None if masks is None else masks[i][j:j + 1].permute(0, 3, 1, 2).double()
            r = tr.deform_conv_ref(self._held(xs[i][j:j + 1]), off, wd, stride=L.stride, padding=L.pad, mask=m)
            return _act(r if bias is None else r + bias, relu)
        self._check("DCN", L, ys, ref, DCN_F16X3_TOL if self.split else DCN_BF16_TOL, plan, low)
        return ys

    def _stem_conv_s2d(self, xs, L, n, h, w):
        y, plan, low = self._run("_stem_conv_s2d", xs, L, n, h, w)
        wd, bias = self._weights(L), L.bias.double()

        def ref(i, j):                        # ResNet's 7x7 / s2 / pad 3 conv1, or HRNet's 3x3 / s2 / pad 1
            return torch.relu(F.conv2d(self._s2d_image(xs, n, h, w, j), wd, bias, L.stride, L.pad))
        self._check("stem", L, [y], ref, OP_TOL if self.split else BF16_TOL, plan, low)
        return y

    def _group_conv(self, x, L, groups, relu=False):
        """ResNeXt's grouped conv2: its own walk over the groups (not an orp_conv2d plan, so no signature is recorded)"""
        y, plan, low = self._run("group_conv", x, L, groups, relu)
        wd, bias = self._weights(L), L.bias.double()

        def ref(i, j):
            return _act(F.conv2d(self._held(x[j:j + 1]), wd, bias, L.stride, 1, groups=groups), relu)
        K = 9 * L.w_raw.shape[3]
        self._check("grouped", L, [y], ref, OP_TOL * max(1.0, K / 4096.0) if self.split else GROUP_BF16_TOL, plan, low)
        return y

    # --------------------------------------------------------------------------------------------- operands
    def _weights(self, L):
        """[Cout, Cin, KH, KW] fp64: what the tensor core multiplies"""
        w = L.w_raw.permute(0, 3, 1, 2).to(self.eng.device)
        return w.double() if self.split else w.bfloat16().double()

    def _held(self, x):
        """an activation tensor as the engine holds it (hi + lo in f16x3, the bf16 value), NCHW fp64"""
        return _nchw64(self.eng.to_float(x))

    def _s2d_image(self, xs, n, h, w, j):
        """image j decoded from the space-to-depth stem operand: cell (Y, X) channel (dy * 2 + dx) * 3 + c holds pixel
        (2 (Y - 2) + dy, 2 (X - 2) + dx) of channel c; the two outer cells of each side and channels 12..15 are zero"""
        hp, wp = h // 2 + 3, w // 2 + 3
        if self.split:
            planes = xs.reshape(-1).view(2, n, hp, wp, 16)                 # hi plane, then lo plane
            s = planes[0, j].double() + planes[1, j].double()
        else:
            s = xs[j].double()
        rest = s.clone()
        rest[2:2 + h // 2, 2:2 + w // 2, :12] = 0
        assert not bool(rest.any()), "%s: the stem operand is not zero outside the image" % self.name
        img = s[2:2 + h // 2, 2:2 + w // 2, :12].reshape(h // 2, w // 2, 2, 2, 3)
        return img.permute(4, 0, 2, 1, 3).reshape(1, 3, h, w)

    # --------------------------------------------------------------------------------------------- checks
    def _check(self, kind, L, ys, ref, tol, plan, low, stats=None, K=None, out_f32=False):
        k = self.checked
        what = "%s launch %d %s (%s, BN %d, %d tiles on %d CTAs)" % (self.name, k, self.names.get(id(L), "?"), kind, plan["BN"],
                                                                  plan["num_tiles"], plan["grid"])
        if kind != "grouped":
            self.sigs.append(signature(plan))
            self.layers.append(self.names.get(id(L), "?"))
        self._values(kind, what, ys, ref, tol, stats, K, out_f32, plan)
        if self.split:
            assert self.eng.overflow_count() == 0, "%s: f16 overflow" % what
        self._write_once(what, ys, low)
        self.checked += 1

    def _result(self, y, out_f32):
        return _nchw64(y) if out_f32 else self._held(y)

    def _values(self, kind, what, ys, ref, tol, stats, K, out_f32, plan):
        for i, y in enumerate(ys):
            n = y.shape[0]
            for j in range(n):
                r = ref(i, j)
                got = self._result(y[j:j + 1], out_f32)
                assert got.shape == r.shape, (what, got.shape, r.shape)
                assert bool(torch.isfinite(got).all()), "%s: problem %d image %d: non-finite output" % (what, i, j)
                err = _rel(got, r)
                if err >= tol:
                    first, worst = _where(got, r, tol)
                    raise AssertionError("%s: problem %d image %d of %d: rel err %.3e >= %.1e; first wrong element (c, y, x) %s, "
                                         "largest error at %s; plan %s" % (what, i, j, n, err, tol, first, worst, plan))
                if err > self.worst.get(kind, (-1.0,))[0]:
                    self.worst[kind] = (err, tol, "%s problem %d image %d" % (what, i, j))
                if stats is not None:
                    self._gn(what, stats[i][j], r if (self.split or plan["gn_fused"]) else got, K, i, j)

    def _gn(self, what, st, src, K, i, j):
        """GroupNorm(32) sums of the epilogue (or of the split-K finishing pass) against fp64 sums: of the fp64 reference, or
        in bf16 without the fused epilogue of the stored output (as test_conv_plans_gpu._check_gn).  The fused sums see the
        tensor core's accumulator truncation, which is biased towards zero: a relative bias d of the outputs moves the sum of
        squares by 2 d.  On P6 (fpn3, K = 18432) the production input is the post-ReLU C5, every activation of one sign, and
        the bias stops averaging out: the sums of squares measured 5.3e-5 (f16x3) and 4.7e-5 (bf16) off on an H100 at
        K = 18432, the plain sums 1.6e-5.  So the sums of squares are held to twice the bound of the sums."""
        tol = GN_TOL * max(1.0, K / 4096.0)
        r = src.reshape(32, -1)
        s_err = float(((st[:, 0] - r.sum(1)).abs() / r.abs().sum(1)).max())
        q_err = float(((st[:, 1] - (r * r).sum(1)).abs() / (r * r).sum(1)).max())
        assert s_err < tol and q_err < 2 * tol, "%s: problem %d image %d: GroupNorm sums off by %.2e / %.2e (tol %.1e / %.1e)" % (
            what, i, j, s_err, q_err, tol, 2 * tol)
        for kind, err, bound in (("GN sums", s_err, tol), ("GN squares", q_err, 2 * tol)):
            if err > self.worst.get(kind, (-1.0,))[0]:
                self.worst[kind] = (err, bound, "%s problem %d image %d" % (what, i, j))

    def _relaunch(self, low, outs):
        """the recorded low-level launch again, into the guarded outputs, with fresh GroupNorm sums"""
        kind, a, kw = low
        fresh = (lambda s: None if s is None else torch.zeros_like(s))
        self.replaying = True
        try:
            if kind == "_launch":
                kw = dict(kw)
                if kw.get("stats") is not None:
                    kw["stats"] = [fresh(s) for s in kw["stats"]]
                self.orig["_launch"](a[0], [g.t for g in outs], *a[2:], **kw)
            elif kind == "_conv_splitk":
                (g,) = outs
                self.orig["_conv_splitk"](a[0], g.t, *a[2:6], fresh(a[6]), *a[7:])
            elif kind == "group":                                 # the same problem, its output the guarded buffer
                (g,) = outs
                q = _lib.TcProblem()
                ctypes.pointer(q)[0] = a[1]._obj
                q.out = g.t.data_ptr()
                self.orig["_call"](a[0], ctypes.byref(q), *a[2:])
            else:
                (g,) = outs
                self.orig["_call"](*a[:-2], _lib.ptr(g.t), a[-1])
        finally:
            self.replaying = False

    def _write_once(self, what, ys, low):
        """two launches into NaN-prefilled guarded outputs: both bitwise equal to the first output, guards untouched"""
        outs = [Guarded(tuple(y.shape), y.dtype, y.device) for y in ys]
        for pat in PATTERNS:
            for g in outs:
                g.fill(pat)
            self._relaunch(low, outs)
            torch.cuda.synchronize()
            for i, (g, y) in enumerate(zip(outs, ys)):
                assert g.guards_intact(pat), "%s: problem %d: a store landed outside the output (fill %#x)" % (what, i, pat & 0xFFFF)
                iv = torch.int32 if y.dtype == torch.float32 else torch.int16
                if not torch.equal(g.t.view(iv), y.view(iv)):
                    diff = (g.t.view(iv) != y.view(iv)).reshape(y.shape[0], -1).any(1).nonzero().reshape(-1).tolist()
                    raise AssertionError("%s: problem %d: the re-launch into a buffer filled with %#x differs from the first "
                                         "launch in images %s (an element not written, or not reproducible)"
                                         % (what, i, pat & 0xFFFF, diff))
        del outs

    def summary(self, seconds):
        kinds = ", ".join("%s %.2e (tol %.1e)" % (k, v[0], v[1]) for k, v in sorted(self.worst.items()))
        return "%s: %d launches checked (counters %d, %d outside a checked call); worst %s; %.1f s" % (
            self.name, self.checked, self.low, len(self.escaped), kinds, seconds)


def _inputs(backbone, batch, test_scale, dev):
    """the bench's input: seeded uint8 tiles; at the test scale through the config's test pipeline (+ valid extents)"""
    if not test_scale:
        g = torch.Generator().manual_seed(1000)                       # bench_tile.run / run_config, rank 0
        return torch.randint(0, 256, (batch, 1024, 1024, 3), generator=g, dtype=torch.uint8).to(dev), None
    from orientedreppoints_b200.bench_tile import _config_test_pipeline
    from orientedreppoints_b200.datasets.pipelines import run_test_pipeline
    g = torch.Generator().manual_seed(2000)                           # bench_tile.run_test_scale, rank 0
    tiles = torch.randint(0, 256, (batch, 1024, 1024, 3), generator=g, dtype=torch.uint8).to(dev)
    data = run_test_pipeline(_config_test_pipeline(backbone), tiles, device=dev)
    (view,), (valid,) = data["img"], data["valid_hw"]
    return view, valid


def _bench_signatures(backbone, prec, dev, img, valid):
    """plan signature of every convolution launch of the bench's own detector, in order"""
    from orientedreppoints_b200.bench_tile import build_detector
    _, det = build_detector(backbone, prec, dev)
    sigs, eng = [], det.eng

    def recorded(fn):
        def wrapper(*a, **kw):
            out = fn(*a, **kw)
            sigs.append(signature(_lib.tc_last_plan()))
            return out
        return wrapper
    for m in ("_launch", "_conv_splitk", "_stem_conv_s2d"):
        setattr(eng, m, recorded(getattr(eng, m)))
    with torch.no_grad():
        det.forward_dense(img, valid)
    torch.cuda.synchronize()
    del det, eng
    torch.cuda.empty_cache()
    return sigs


def _checked_detector(backbone, prec, dev):
    """random weights whose every launch carries signal: randomised norm scales (no zero_init_residual) for the ResNets,
    with a modest residual gain over R-101's 33 blocks (as tests/test_f16x3_gpu.py), the bench's Swin-T state dict"""
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    if backbone == "swin_tiny":
        from orientedreppoints_b200.swin import random_swin_state_dict
        return OrientedRepPointsDetector(random_swin_state_dict(0), "swin_tiny", dev, prec, test_cfg=dict(score_thr=0.0))
    from orientedreppoints_b200.weights import random_state_dict
    depth = int(backbone[1:])
    sd = random_state_dict(depth, seed=0, reference_init=False, residual_gain=1.0 if depth == 50 else 0.3)
    return OrientedRepPointsDetector(sd, depth, dev, prec, test_cfg=dict(score_thr=0.0))


def _run_workload(dev, backbone, prec, batch, test_scale):
    t0 = time.time()
    name = "%s %s x%d%s" % (backbone, prec, batch, " at 960^2" if test_scale else "")
    img, valid = _inputs(backbone, batch, test_scale, dev)
    bench_sigs = _bench_signatures(backbone, prec, dev, img, valid)
    det = _checked_detector(backbone, prec, dev)
    chk = LaunchChecker(det, name)
    if chk.split:
        det.eng.overflow_count()                                      # the counter is global: start from zero
    with torch.no_grad():
        det.forward_dense(img, valid)
    torch.cuda.synchronize()
    line = chk.summary(time.time() - t0)
    print(line)
    assert not chk.escaped, "%s: launches outside a checked call: %s" % (name, chk.escaped)
    assert chk.checked == chk.low and chk.checked > 0, line
    assert chk.sigs == bench_sigs, "%s: the checked detector launches other plans than the bench's" % name
    del det, chk
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------- A: every launch
LAUNCH_WORKLOADS = [w + (False,) for w in WORKLOADS] + [w + (True,) for w in TEST_SCALE]


@pytest.mark.parametrize("backbone,prec,batch,test_scale", LAUNCH_WORKLOADS,
                         ids=["%s-%s-x%d%s" % (b, p, n, "-960" if t else "") for b, p, n, t in LAUNCH_WORKLOADS])
def test_every_conv_launch_vs_fp64(cuda, backbone, prec, batch, test_scale):
    _run_workload(cuda, backbone, prec, batch, test_scale)


# ---------------------------------------------------------------------------------------------- B: the benchmarked step
def _state_dict(backbone, reference_init):
    """the state dict bench_tile.build_detector builds"""
    if backbone == "swin_tiny":
        from orientedreppoints_b200.swin import random_swin_state_dict
        return random_swin_state_dict(0)
    from orientedreppoints_b200.weights import random_state_dict
    return random_state_dict(int(backbone[1:]), seed=0, reference_init=reference_init)


def _host_normalised64(tile, cfg, dev):
    """one uint8 HWC tile -> Normalize (to_rgb, (x - mean) / std) in fp64 on the host, NCHW [1,3,H,W]"""
    x = tile.cpu().double()
    if cfg["to_rgb"]:
        x = x.flip(-1)
    x = (x - torch.tensor(cfg["mean"], dtype=torch.float64)) / torch.tensor(cfg["std"], dtype=torch.float64)
    return x.permute(2, 0, 1).unsqueeze(0).contiguous().to(dev)


def _fp64_dense(sd, depth, img):
    from oracle import torch_reference as tr
    from oracle import torch_swin as ts
    from orientedreppoints_b200.weights import STAGE_BLOCKS
    sdg = {k: v.to(img.device).double() for k, v in sd.items()}
    with torch.no_grad():
        if depth == "swin_tiny":
            fpn = ts.swin_fpn(sdg, ts.swin_forward(sdg, img))
            return [tr.head_single(sdg, f)[:3] for f in fpn], fpn
        return tr.forward_dense(sdg, img, blocks=STAGE_BLOCKS[depth])


def _clone_dense(dense):
    outs, feats = dense
    return [tuple(t.clone() for t in o) for o in outs], [f.clone() for f in feats]


def _replays_agree(eng, a, b, n, what):
    """dense outputs a and b, tile by tile: the five FPN levels and cls / init / refine of every level within REPLAY_TOL"""
    (oa, fa), (ob, fb) = a, b
    for t in range(n):
        for lvl in range(5):
            e = _rel(eng.to_float(fa[lvl][t:t + 1]), eng.to_float(fb[lvl][t:t + 1]))
            assert e < REPLAY_TOL, (what, "tile %d feat%d" % (t, lvl), e)
            for k, nm in enumerate(("cls", "init", "refine")):
                e = _rel(oa[lvl][k][t:t + 1], ob[lvl][k][t:t + 1])
                assert e < REPLAY_TOL, (what, "tile %d %s%d" % (t, nm, lvl), e)


def _tile_vs_fp64(det, sd, depth, img, dense, t):
    """tile t of the replayed dense outputs against the fp64 graph run on that tile alone; returns (errors, fp64 outputs)"""
    outs, feats = dense
    ref_outs, ref_feats = _fp64_dense(sd, depth, _host_normalised64(img[t], det.img_norm_cfg, img.device))
    errs = {}
    for lvl in range(5):
        errs["feat%d" % lvl] = _rel(_nchw64(det.eng.to_float(feats[lvl][t:t + 1])), ref_feats[lvl])
        for k, nm in enumerate(("cls", "init", "refine")):
            a, b = _nchw64(outs[lvl][k][t:t + 1]), ref_outs[lvl][k]
            assert a.shape == b.shape
            errs["%s%d" % (nm, lvl)] = float((a - b).abs().max()) / max(1.0, float(b.abs().max()))
    return errs, ref_outs


def _check_tiles(det, sd, depth, img, dense, tiles, what):
    refs = {}
    for t in tiles:
        errs, refs[t] = _tile_vs_fp64(det, sd, depth, img, dense, t)
        worst = max(errs, key=errs.get)
        print("%s tile %d: max rel err %.2e (%s) vs the fp64 graph" % (what, t, errs[worst], worst))
        for k, v in errs.items():
            assert v < DENSE_TOL, (what, "tile %d" % t, k, v)
    return refs


def _oracle_detections(det, dense, ref_outs, t, what):
    """tile t's detections against the oracle post-processing of the fp64 graph's outputs, matched by content as in
    tests/test_f16x3_gpu.py::test_dense_graph_f16x3_1024_and_detections, at its score_thr 0.02"""
    from oracle import torch_reference as tr
    from orientedreppoints_b200.core.get_bboxes import get_bboxes_fused
    from orientedreppoints_b200.detector import STRIDES
    outs, _ = dense
    thr = 0.02
    cfg = dict(det.test_cfg, score_thr=thr)
    dets, labels, counts = get_bboxes_fused([o[0][t:t + 1] for o in outs], [o[2][t:t + 1] for o in outs], STRIDES,
                                            [dict(scale_factor=1.0)], cfg, True)
    c = int(counts[0])
    d, lab = dets[0, :c].cpu(), labels[0, :c].cpu()
    rd, rl = tr.get_bboxes_single([o[0][0].float() for o in ref_outs], [o[2][0].float().cpu() for o in ref_outs], score_thr=thr)
    assert c > 0 and rd.shape[0] > 0, (what, t, c, rd.shape)
    dist = torch.cdist(d[:, :26].double(), rd[:, :26].double(), p=float("inf"))
    dist = dist + (lab[:, None] != rl[None, :]).double() * 1e6
    best, arg = dist.min(dim=1)
    matched = best < 1e-2
    frac = float(matched.float().mean())
    back = float((dist.min(dim=0).values < 1e-2).float().mean())
    sdelta = float((d[matched, 26] - rd[arg[matched], 26]).abs().max())
    print("%s tile %d: %d detections at score_thr %.6f (oracle %d): %.4f found in the oracle's, %.4f of the oracle's found; "
          "max score delta %.2e" % (what, t, c, thr, rd.shape[0], frac, back, sdelta))
    assert frac > 0.98 and back > 0.98, (what, t, frac, back)
    assert sdelta < 1e-4, (what, t, sdelta)


def _bench_step(backbone, batch, dev, reference_init=True):
    """the detector and input of bench_tile.run / run_config, the graph captured, and the padded output of one step"""
    from orientedreppoints_b200.bench_tile import build_detector
    depth, det = build_detector(backbone, "f16x3", dev, reference_init)
    g = torch.Generator().manual_seed(1000)
    img = torch.randint(0, 256, (batch, 1024, 1024, 3), generator=g, dtype=torch.uint8).to(dev)
    det.eng.overflow_count()
    with torch.no_grad():
        eager = _clone_dense(det.forward_dense(img))
    det.capture(img.shape, img.dtype)
    step = det.simple_test(img, return_tensors="padded")
    replay = _clone_dense(det._g_out)
    torch.cuda.synchronize()
    return depth, det, img, eager, replay, step


@pytest.mark.parametrize("reference_init", [True, False], ids=["reference-init", "random-norm-scales"])
def test_benchmarked_step_r50_x16(cuda, reference_init):
    from orientedreppoints_b200.core.get_bboxes import get_bboxes, get_bboxes_fused
    from orientedreppoints_b200.detector import STRIDES
    t0 = time.time()
    what = "r50 f16x3 x16 step (%s)" % ("reference init" if reference_init else "random norm scales")
    depth, det, img, eager, replay, (dets, labels, counts) = _bench_step("r50", 16, cuda, reference_init)
    _replays_agree(det.eng, replay, eager, 16, what + ": replay vs eager")
    det.forward_dense_graph(img)
    _replays_agree(det.eng, det._g_out, replay, 16, what + ": replay vs replay")
    refs = _check_tiles(det, _state_dict("r50", reference_init), depth, img, replay, range(16), what)
    assert det.eng.overflow_count() == 0
    # detections: the bench's padded output is the fused post-processing of the replayed dense outputs it came from
    outs, _ = replay
    metas = [dict(scale_factor=1.0) for _ in range(16)]
    d2, l2, c2 = get_bboxes_fused([o[0] for o in outs], [o[2] for o in outs], STRIDES, metas, det.test_cfg, False)
    assert torch.equal(counts, c2) and torch.equal(labels, l2)
    for t in range(16):
        c = int(counts[t])
        assert c > 0 and torch.equal(dets[t, :c].view(torch.int32), d2[t, :c].view(torch.int32)), (what, t)
    # ... and agrees with the op-by-op mirror of get_bboxes / multiclass_rnms (labels and scores exact, coordinates 1e-3 px
    # as in tests/test_dense_gpu.py::test_fused_postprocess_equals_torch_mirror_and_oracle) on the first and last tile
    for t in (0, 15):
        (md, ml), = get_bboxes([o[0][t:t + 1] for o in outs], [o[2][t:t + 1] for o in outs], STRIDES, metas[:1], det.test_cfg, False)
        c = int(counts[t])
        assert md.shape[0] == c and torch.equal(labels[t, :c], ml), (what, t, c, md.shape)
        assert torch.equal(dets[t, :c, 26], md[:, 26]) and float((dets[t, :c] - md).abs().max()) < 1e-3, (what, t)
    for t in (0, 15) if not reference_init else ():
        _oracle_detections(det, replay, refs[t], t, what)
    print("%s: %.1f s" % (what, time.time() - t0))
    del det
    torch.cuda.empty_cache()


@pytest.mark.parametrize("backbone,batch", [("r101", 4), ("swin_tiny", 8)])
def test_benchmarked_step_other_workloads(cuda, backbone, batch):
    t0 = time.time()
    what = "%s f16x3 x%d step" % (backbone, batch)
    depth, det, img, eager, replay, _ = _bench_step(backbone, batch, cuda)
    _replays_agree(det.eng, replay, eager, batch, what + ": replay vs eager")
    _check_tiles(det, _state_dict(backbone, True), depth, img, replay, range(batch), what)
    assert det.eng.overflow_count() == 0
    print("%s: %.1f s" % (what, time.time() - t0))
    del det
    torch.cuda.empty_cache()
