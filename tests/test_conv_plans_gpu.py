"""GPU: the wgmma convolution kernel (csrc/dense_tc.cu) against fp64, once per launch plan the detector uses.

For every launch the host code of conv2d_tc picks a plan from the shapes: accumulator width BN, TMA or staged
epilogue, the ncat / dcat / res_mma / b_resident / epi_merge / gn_fused variants, output staging buffers, pipeline stages
and how many tiles each persistent CTA processes.  orp_tc_last_plan reports the plan as launched.  The cases (PARITY) live
in tests/conv_plan_cases.py.

- test_production_plans_are_covered runs the benchmark workloads once and reduces every convolution launch to a plan
  signature (SIG_FIELDS); each one must be pinned by a case of PARITY, so a heuristic change that moves production onto an
  untested plan fails here.
- test_conv_plan_vs_fp64: one case per signature.  It asserts the plan it reaches (and that the dry run orp_tc_plan_conv
  plans the same launch, field for field), compares with an fp64 reference, and
  launches twice into outputs pre-filled with different NaN patterns between guard regions: the two results must be
  bitwise equal and the guards untouched (every output element written exactly once, nothing outside).
- test_deform_edges: the production DCN plans with zero offsets, samples exactly on the image border and DCNv2 masks."""
import pytest
import torch
import torch.nn.functional as F

from orientedreppoints_b200 import _lib

from conv_plan_cases import PARITY, SIG_FIELDS, case_id, planned, signature

pytestmark = pytest.mark.gpu

# tolerances of tests/test_f16x3_gpu.py and tests/test_dense_gpu.py
OP_TOL = 8e-6           # f16x3, one layer, scaled by max(1, K / 4096)
DCN_F16X3_TOL = 2.5e-5  # f16x3 deformable: (tap, block, term) walk, the loss of 3K/16 accumulator steps
BF16_F32_TOL = 2e-5     # bf16 operands, fp32 output: fp32 accumulation of exact bf16 products
BF16_TOL = 6e-3         # bf16 output: one rounding to bf16 (2^-8 of the largest value)
DCN_BF16_TOL = 1.5e-2   # bf16 deformable: the sample is rounded to bf16 before the MMA, the output again
GN_TOL = 1e-5           # GroupNorm statistics and f16x3 GroupNorm output

# ------------------------------------------------------------------------------------------------------------- helpers
@pytest.fixture(scope="module")
def engines(cuda):
    from orientedreppoints_b200.engine_tc import EngineTC, EngineTCSplit
    return {"f16x3": EngineTCSplit(cuda), "bf16": EngineTC(cuda)}


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / (b.double().abs().max() + 1e-30))


GUARD = 4096                                    # bytes before and after every output
PATTERNS = (-1, 0x7FC0)                          # int16 fills: NaN as fp32, fp16 and bf16 alike


class Guarded:
    """an output tensor carved out of a larger buffer with guard regions on both sides"""

    def __init__(self, shape, dtype, dev):
        n = 1
        for v in shape:
            n *= v
        self.nbytes = n * torch.empty((), dtype=dtype).element_size()
        self.buf = torch.empty(2 * GUARD + self.nbytes, dtype=torch.uint8, device=dev)
        self.t = self.buf[GUARD:GUARD + self.nbytes].view(dtype).view(shape)

    def fill(self, pattern):
        self.buf.view(torch.int16).fill_(pattern)

    def guards_intact(self, pattern):
        w = self.buf.view(torch.int16)
        return bool((w[:GUARD // 2] == pattern).all()) and bool((w[(GUARD + self.nbytes) // 2:] == pattern).all())

    def bits(self):
        return self.t.view(torch.int32 if self.t.dtype == torch.float32 else torch.int16).clone()


def _nchw(y):
    return y.permute(0, 3, 1, 2)


def _act(v, act):
    return torch.relu(v) if act == 1 else (F.gelu(v) if act == 2 else v)


class Case:
    """inputs, fp64 references and guarded outputs of one PARITY entry"""

    def __init__(self, c, eng, dev, seed, offsets="random", masks=None):
        self.sig, self.prec, self.kind, cin, cout, k, s, bias, act, out_f32, res, gn, probs = c
        self.eng, self.dev = eng, dev
        self.cin, self.cout, self.k, self.s, self.act, self.out_f32, self.res, self.gn = cin, cout, k, s, act, out_f32, res, gn
        self.pad = k // 2
        self.split = self.prec == "f16x3"
        g = torch.Generator().manual_seed(seed)
        from orientedreppoints_b200.detector import ConvLayer
        rq = (lambda t: t.double()) if self.split else (lambda t: t.bfloat16().double())   # what the tensor core multiplies
        if self.kind == "stem":
            wt = torch.randn(64, 3, 7, 7, generator=g) * 0.1
            b = torch.randn(64, generator=g) * 0.1
            self.L = ConvLayer(wt, b, 2, 3, dev, pad_cin_to=4)
            self.imgs = [torch.randn(n, 3, h, w, generator=g).to(dev) for (n, h, w) in probs]
            self.refs = [torch.relu(F.conv2d(rq(x), rq(wt.to(dev)), b.double().to(dev), 2, 3)) for x in self.imgs]
            self.tol = OP_TOL if self.split else BF16_TOL
            self.outs = [Guarded((n, h // 2, w // 2) + ((2, 64) if self.split else (64,)), torch.float16 if self.split else torch.bfloat16, dev)
                         for (n, h, w) in probs]
            self.stats = None
            return
        wt = torch.randn(cout, cin, k, k, generator=g) * (1.0 / (cin * k * k) ** 0.5)
        b = torch.randn(cout, generator=g) if bias else None
        self.L = ConvLayer(wt, b, s, self.pad, dev)
        wd = rq(wt.to(dev))
        self.xs, self.res16, self.res32, self.offs, self.masks, self.refs, self.outs = [], [], [], [], [], [], []
        for (n, h, w) in probs:
            ho, wo = (h + 2 * self.pad - k) // s + 1, (w + 2 * self.pad - k) // s + 1
            x = torch.randn(n, cin, h, w, generator=g).to(dev)
            self.xs.append(eng.from_float(x.permute(0, 2, 3, 1)))
            if self.kind == "deform":
                from oracle import torch_reference as tr
                off = _offsets(offsets, n, h, w, g).to(dev)
                m = None if masks is None else _masks(masks, n, h, w, g).to(dev)
                self.offs.append(off.permute(0, 2, 3, 1).contiguous())
                self.masks.append(None if m is None else m.permute(0, 2, 3, 1).contiguous())
                ref = tr.deform_conv_ref(rq(x), off.double(), wd, mask=None if m is None else m.double())
            else:
                ref = F.conv2d(rq(x), wd, None, s, self.pad)
            if b is not None:
                ref = ref + b.double().to(dev).view(1, -1, 1, 1)
            if res:
                r = torch.randn(n, cout, ho, wo, generator=g).to(dev)
                if res == 1:
                    self.res16.append(eng.from_float(r.permute(0, 2, 3, 1)))
                    ref = ref + rq(r)
                else:
                    self.res32.append(r.permute(0, 2, 3, 1).contiguous())
                    ref = ref + r.double()
            self.refs.append(_act(ref, act))
            if out_f32:
                self.outs.append(Guarded((n, ho, wo, cout), torch.float32, dev))
            else:
                self.outs.append(Guarded((n, ho, wo) + ((2, cout) if self.split else (cout,)),
                                         torch.float16 if self.split else torch.bfloat16, dev))
        self.stats = [torch.zeros((n, 32, 2), dtype=torch.float64, device=dev) for (n, _, _) in probs] if gn else None
        K = cin * k * k
        if self.kind == "deform":
            self.tol = DCN_F16X3_TOL if self.split else DCN_BF16_TOL
        elif self.split:
            self.tol = OP_TOL * max(1.0, K / 4096.0)
        else:
            self.tol = BF16_F32_TOL if out_f32 else BF16_TOL

    def launch(self):
        """the launch the engine makes for this layer, into the guarded outputs; returns the reported plan"""
        e, st = self.eng, _lib.current_stream_ptr()
        ys = [o.t for o in self.outs]
        if self.kind == "stem":
            for img, y in zip(self.imgs, ys):
                n, _, h, w = img.shape
                if self.split:
                    ws = e._stem_s2d_tc(self.L)
                    xs = torch.empty((2, n, h // 2 + 3, w // 2 + 3, 16), dtype=torch.float16, device=self.dev)
                    _lib.check(e.lib.orp_stem_s2d_f16x3(_lib.ptr(img), n, h, w, _lib.ptr(xs), st), "orp_stem_s2d_f16x3")
                    _lib.check(e.lib.orp_stem_conv_s2d_f16x3(_lib.ptr(xs), n, h, w, _lib.ptr(ws["w"]), _lib.ptr(self.L.bias), ws["s"],
                                                             1, _lib.ptr(y), st), "orp_stem_conv_s2d_f16x3")
                else:
                    ws = e._stem_s2d_tc(self.L)
                    xs = torch.empty((n, h // 2 + 3, w // 2 + 3, 16), dtype=torch.bfloat16, device=self.dev)
                    _lib.check(e.lib.orp_stem_s2d_bf16(_lib.ptr(img), n, h, w, _lib.ptr(xs), st), "orp_stem_s2d_bf16")
                    _lib.check(e.lib.orp_stem_conv_s2d_bf16(_lib.ptr(xs), n, h, w, _lib.ptr(ws), _lib.ptr(self.L.bias), 1,
                                                            _lib.ptr(y), st), "orp_stem_conv_s2d_bf16")
            return _lib.tc_last_plan()
        tc = e._tc(self.L, out16=self.kind == "conv" and not self.out_f32)     # the weights conv_multi packs for this layer
        if self.stats is not None:
            for t in self.stats:
                t.zero_()
        if self.kind == "deform":
            e._launch(self.xs, ys, tc, self.cout, 3, 3, self.cin, 1, 1, self.L.bias, self.act, False, True, offsets=self.offs,
                      masks=None if self.masks[0] is None else self.masks)
            return _lib.tc_last_plan()
        n, ho, wo = ys[0].shape[:3]
        ks = e._ksplit(n, ho, wo, self.L, len(ys), self.act, self.res16 or None, bool(self.out_f32), self.res32 or None)
        if ks > 1:
            e._conv_splitk(self.xs[0], ys[0], tc, self.L, self.act, ks, None if self.stats is None else self.stats[0], self.split)
        else:
            e._launch(self.xs, ys, tc, self.cout, self.k, self.k, self.cin, self.s, self.pad, self.L.bias, self.act,
                      bool(self.out_f32), False, res=self.res16 or None, res32=self.res32 or None, stats=self.stats)
        return _lib.tc_last_plan()

    def result(self, i):
        y = self.outs[i].t
        if self.out_f32:
            return _nchw(y)
        return _nchw(self.eng.to_float(y) if self.split else y.float())


def _offsets(mode, n, h, w, g):
    """[N, 18, H, W] (dy, dx) per tap of a 3x3 / pad 1 / stride 1 DCN.  "edges": every sample lands exactly on a row of
    {-1, -0.5, 0, 0.5, H-1.5, H-1, H-0.5, H} or an interior point, and likewise for columns - the validity and corner tests of
    the bilinear sample at their boundaries"""
    if mode == "random":
        return torch.randn(n, 18, h, w, generator=g) * 2.5
    if mode == "zero":
        return torch.zeros(n, 18, h, w)
    assert mode == "edges"

    def targets(size, shape):
        pick = torch.tensor([-1.0, -0.5, 0.0, 0.5, size - 1.5, size - 1.0, size - 0.5, float(size)])
        t = pick[torch.randint(0, len(pick), shape, generator=g)]
        inner = torch.randint(0, 2 * size, shape, generator=g).float() * 0.5 - 0.5      # half-integer grid inside
        return torch.where(torch.rand(shape, generator=g) < 0.75, t, inner)

    off = torch.empty(n, 18, h, w)
    hh = torch.arange(h).view(1, h, 1).float()
    ww = torch.arange(w).view(1, 1, w).float()
    for t in range(9):
        kh, kw = divmod(t, 3)
        off[:, 2 * t] = targets(h, (n, h, w)) - (hh - 1 + kh)
        off[:, 2 * t + 1] = targets(w, (n, h, w)) - (ww - 1 + kw)
    return off


def _masks(mode, n, h, w, g):
    if mode == "binary":
        return torch.randint(0, 2, (n, 9, h, w), generator=g).float()
    return torch.rand(n, 9, h, w, generator=g)


def _check_written_once(case):
    """two launches into differently NaN-filled outputs: bitwise equal results, untouched guards; returns the plan"""
    bits, plan = [], None
    for pat in PATTERNS:
        for o in case.outs:
            o.fill(pat)
        plan = case.launch()
        torch.cuda.synchronize()
        for o in case.outs:
            assert o.guards_intact(pat), "a store landed outside the output"
        bits.append([o.bits() for o in case.outs])
    for i, (a, b) in enumerate(zip(*bits)):
        assert torch.equal(a, b), "problem %d: outputs differ between launches (an element not written, or not reproducible)" % i
    return plan


def _check_values(case, plan):
    errs = []
    for i, ref in enumerate(case.refs):
        y = case.result(i)
        assert bool(torch.isfinite(y).all()), "problem %d: non-finite output" % i
        errs.append(_rel(y, ref))
    assert max(errs) < case.tol, (errs, case.tol)
    if case.gn:
        _check_gn(case, plan)
    if case.split:
        assert case.eng.overflow_count() == 0
    return max(errs)


def _check_gn(case, plan):
    """the GroupNorm(32) statistics the launch produced against fp64 sums, and conv_gn's normalised output against
    F.group_norm.  The fused epilogue sums the fp32 results, so its reference is the fp64 convolution; its error is the
    tensor core's accumulator truncation, which is linear in the K steps and biased towards zero (the sums of squares
    see twice the bias): the bound scales with K beyond 4096 as OP_TOL does (measured 3.6e-5 at K = 18432 in bf16).
    The separate pass (split-K launches) sums the stored outputs: in bf16 its reference is the bf16 output itself."""
    g = torch.Generator().manual_seed(99)
    gamma = (torch.rand(256, generator=g) + 0.5).to(case.dev)
    beta = (torch.randn(256, generator=g) * 0.1).to(case.dev)
    tol = GN_TOL * max(1.0, case.cin * case.k * case.k / 4096.0)
    for i, (st, ref) in enumerate(zip(case.stats, case.refs)):
        n = ref.shape[0]
        src = ref if (case.split or plan["gn_fused"]) else case.result(i).double()
        r = src.reshape(n, 32, -1)
        s_err = (st[..., 0] - r.sum(2)).abs() / r.abs().sum(2)
        q_err = (st[..., 1] - (r * r).sum(2)).abs() / (r * r).sum(2)
        assert float(s_err.max()) < tol and float(q_err.max()) < tol, (float(s_err.max()), float(q_err.max()), tol)

    class _Norm:
        pass
    nm = _Norm()
    nm.gamma, nm.beta = gamma, beta
    ys = case.eng.gn_multi([o.t for o in case.outs], nm, stats=case.stats)
    for y, ref in zip(ys, case.refs):
        want = F.group_norm(ref, 32, gamma.double(), beta.double(), 1e-5)
        got = _nchw(case.eng.to_float(y) if case.split else y.float())
        # bf16: the convolution output and the normalised output are each rounded to bf16
        assert _rel(got, want) < (GN_TOL if case.split else 2 * BF16_TOL)


# ---------------------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("c", PARITY, ids=[case_id(c) for c in PARITY])
def test_conv_plan_vs_fp64(cuda, engines, c):
    case = Case(c, engines[c[1]], cuda, seed=sum(c[3:7]) + len(c[-1]))
    plan = _check_written_once(case)
    assert signature(plan) == c[0], "the case left its plan: %s" % dict(zip(SIG_FIELDS, signature(plan)))
    assert plan == planned(c), "the dry run plans another launch: %s" % planned(c)
    err = _check_values(case, plan)
    print("%s: grid %d, %d tiles (%.1f per CTA), %d N tiles, rel err %.2e (tol %.1e)"
          % (case_id(c), plan["grid"], plan["num_tiles"], plan["num_tiles"] / plan["grid"], plan["n_tiles_n"], err, case.tol))


DCN_CASES = [c for c in PARITY if c[2] == "deform"]
DCN_IDS = [case_id(c) if c[7] else c[1] for c in DCN_CASES]    # the head's DCN (no bias) by its format, the backbone's by its case


@pytest.mark.parametrize("mode", ["zero", "edges", "mask_binary", "mask_random", "edges_mask_random"])
@pytest.mark.parametrize("c", DCN_CASES, ids=DCN_IDS)
def test_deform_edges(cuda, engines, c, mode):
    offsets = "zero" if mode == "zero" else ("edges" if mode.startswith("edges") else "random")
    masks = "binary" if mode == "mask_binary" else ("random" if "mask_random" in mode else None)
    case = Case(c, engines[c[1]], cuda, seed=7, offsets=offsets, masks=masks)
    plan = _check_written_once(case)
    assert signature(plan) == c[0]
    assert plan == planned(c)
    if mode == "zero":
        # zero offsets: every sample is the input pixel itself - the plain 3x3 convolution
        for i, ref in enumerate(case.refs):
            x = case.eng.to_float(case.xs[i]) if case.split else case.xs[i].float()
            plain = torch.relu(F.conv2d(_nchw(x).double(), case.L.w_raw.permute(0, 3, 1, 2).to(cuda).double()
                                        if case.split else case.L.w_raw.permute(0, 3, 1, 2).to(cuda).bfloat16().double(),
                                        None if case.L.bias is None else case.L.bias.double(), 1, 1))
            assert _rel(ref, plain) < 1e-6                      # the fp64 references agree (x rounded as the engine holds it)
    err = _check_values(case, plan)
    print("%s %s: %d tiles on %d CTAs, %d stages, rel err %.2e" % (c[1], mode, plan["num_tiles"], plan["grid"], plan["stages"], err))


# ------------------------------------------------------------------------------------------------ production inventory
WORKLOADS = [("r50", "f16x3", 16), ("r50", "f16x3", 1), ("r101", "f16x3", 4), ("swin_tiny", "f16x3", 8), ("swin_tiny", "bf16", 8),
             ("r50", "bf16", 16)]


def test_production_plans_are_covered(cuda):
    """the bench workloads, one forward_dense each with random weights: every convolution launch's plan signature must be
    one that PARITY pins"""
    from orientedreppoints_b200.bench_tile import build_detector
    seen = {}
    for backbone, prec, batch in WORKLOADS:
        name = "%s %s x%d" % (backbone, prec, batch)
        _, det = build_detector(backbone, prec, cuda)
        eng = det.eng

        def recorded(fn):
            def wrapper(*a, **kw):
                out = fn(*a, **kw)
                p = _lib.tc_last_plan()
                e = seen.setdefault(signature(p), dict(launches=0, workloads=set(), tpc=0.0))
                e["launches"] += 1
                e["workloads"].add(name)
                e["tpc"] = max(e["tpc"], p["num_tiles"] / p["grid"])
                return out
            return wrapper
        for m in ("_launch", "_conv_splitk", "stem", "stem_u8"):
            setattr(eng, m, recorded(getattr(eng, m)))
        img = torch.randint(0, 256, (batch, 1024, 1024, 3), generator=torch.Generator().manual_seed(1), dtype=torch.uint8)
        with torch.no_grad():
            det.forward_dense(img.to(cuda))
        torch.cuda.synchronize()
        del det, eng
        torch.cuda.empty_cache()
    pinned = {c[0] for c in PARITY}
    print("\n%-6s %s  launches  max tiles/CTA  workloads" % ("pinned", " ".join(SIG_FIELDS)))
    for sig, e in sorted(seen.items(), key=lambda kv: str(kv[0])):
        print("%-6s %s  %4d  %6.1f  %s" % ("yes" if sig in pinned else "NO", sig, e["launches"], e["tpc"], ", ".join(sorted(e["workloads"]))))
    missing = [s for s in seen if s not in pinned]
    assert not missing, "production plans without a parity case: %s" % [dict(zip(SIG_FIELDS, s)) for s in missing]
