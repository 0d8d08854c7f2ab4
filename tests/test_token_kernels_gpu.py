"""GPU: the memory-bound and token kernels of the benchmarked graphs against fp64 or bitwise against torch, once per
launch signature the detector reaches.

Kernels: csrc/dense_misc.cu (GroupNorm apply for up to 8 problems with the FPN top-down add and ReLU, GroupNorm
statistics, the 3x3/2 max-pool, the stem's space-to-depth input from float, uint8 or uint8 with per-image extents) and
csrc/swin.cu (LayerNorm into a plain or 7-padded grid, the mma.sync window attention,
the patch-embed rows, the patch-merge gather, the stride-2 subsample of Swin P6 / P7).

- A signature per kernel family reduces a launch to what selects code paths (`call_signature` reads it from the
  arguments of the C entry point).  CASES holds one case per production signature plus edge cases.
- test_token_kernel: every case launches twice into outputs pre-filled with different NaN patterns between guard regions;
  the guards stay untouched, the two results are bitwise equal, and the result matches its reference.  GroupNorm
  statistics use double atomics, so the GroupNorm cases repeat the apply step with fixed statistics.
- test_production_signatures_are_covered runs the bench workloads, records every call to these entry points and fails
  when one reaches a signature no case pins.
- test_invalid_launches_are_refused: shapes the kernels cannot run return ORP_EINVAL before anything is launched."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from orientedreppoints_b200 import _lib

pytestmark = pytest.mark.gpu

ORP_EINVAL = -1
NUM_SMS = 132                                     # kNumSMs of csrc/common.cuh: the GroupNorm statistics grid cap

# relative to the reference's largest magnitude
GN_APPLY_TOL = {"f16x3": 1e-5, "bf16": 4e-3}     # exact statistics: fp32 normalise + one output rounding (bf16: 2^-8)
GN_E2E_TOL = {"f16x3": 1e-4, "bf16": 6e-3}       # statistics summed by the kernels, |mean| / std <= 16
# |mean| / std = 64: the statistics are fp32 partial sums of x and x^2 added in double, and var = E[x^2] - mean^2 loses
# the digits the partials rounded away.  The measured envelope, not a target (DESIGN.md section 2).
GN_E2E_R64_TOL = 5e-4
LN_TOL = {"f16x3": 2e-6, "bf16": 8e-3}
ATTN_TOL = {"f16x3": 5e-6, "bf16": 6e-3}

GUARD = 4096                                      # bytes before and after every output
PATTERNS = (-1, 0x7FC0)                           # int16 fills: NaN in fp16 and bf16 alike


# ------------------------------------------------------------------------------------------------------------ signatures
def sig_gn_apply(fmt, probs, relu):
    """probs: (N, H, W, has top-down source) per problem.  A block covers 1024 (f16x3) or 2048 (bf16) 16-byte items of an
    image; the top-down source is read at ceil(H / 2) x ceil(W / 2)"""
    items = 1024 if fmt == "f16x3" else 2048
    return ("gn_apply", fmt, len(probs), int(any(p[3] for p in probs)), int(bool(relu)), int(any(p[0] > 1 for p in probs)),
            int(any(p[1] * p[2] * 32 % items for p in probs)), int(any(p[3] and (p[1] % 2 or p[2] % 2) for p in probs)))


def gn_stats_grid(n, hw):
    """(slab count capped, HW % slab != 0) as orp_gn_stats_* sizes its grid"""
    slabs = -(-hw // 64)
    maxs = (NUM_SMS * 4 + n - 1) // n
    capped = slabs > maxs
    slab = -(-hw // min(slabs, maxs))
    return int(capped), int(hw % slab != 0)


def sig_gn_stats(fmt, n, hw):
    return ("gn_stats", fmt) + gn_stats_grid(n, hw)


def sig_maxpool(fmt, h, w):
    return ("maxpool", fmt, h % 2, w % 2)


def sig_stem(fmt, src, h, w, valid):
    """src: f32 (normalised NCHW), u8 (HWC tiles), u8v (with per-image extents)"""
    below = int(any(vh < h or vw < w for vh, vw in valid)) if valid else 0
    odd = int(any(min(vw, w) % 2 for _, vw in valid)) if valid else 0
    return ("stem", fmt, src, below, odd)


def ln_plan(c):
    """(chunks per lane, lanes per token G, tokens per block) of layernorm_impl"""
    k = 3 if c <= 768 else 6
    g = 1
    while g < 32 and g * k < c // 8:
        g *= 2
    return k, g, 8 * (32 // g)


def sig_ln(fmt, b, h, w, c, hp, wp):
    k, g, tpb = ln_plan(c)
    return ("layernorm", fmt, k, g, int((hp, wp) != (h, w)), int(b * h * w % tpb != 0))


def sig_attn(fmt, h, w, hp, wp, heads, shift):
    return ("attention", fmt, heads, int(shift > 0), int(hp > h), int(wp > w), int(hp == 7 or wp == 7))


def sig_embed(fmt, src, h, w):
    return ("patch_embed", fmt, src, int(h % 4 != 0 or w % 4 != 0))


def sig_gather(kind, fmt, h, w):
    return (kind, fmt, h % 2, w % 2)


_VALID = {}                                       # device address -> the (h, w) extents it holds


def _addr(p):
    return p.value if isinstance(p, ctypes.c_void_p) else int(p or 0)


def call_signature(name, a):
    """the signature of one call to an entry point of ENTRY_POINTS, from its arguments"""
    fmt = "f16x3" if "f16x3" in name else "bf16"
    base = name[len("orp_"):]
    if base.startswith("gn_apply"):
        return sig_gn_apply(fmt, [(a[1][i].N, a[1][i].H, a[1][i].W, bool(a[1][i].up_src)) for i in range(a[0])], a[7])
    if base.startswith("gn_stats"):
        return sig_gn_stats(fmt, a[1], a[2])
    if base.startswith("maxpool3x3s2"):
        return sig_maxpool(fmt, a[2], a[3])
    if base.startswith("stem_s2d_u8_padded"):
        return sig_stem(fmt, "u8v", a[2], a[3], _VALID[_addr(a[7])])
    if base.startswith("stem_s2d_u8"):
        return sig_stem(fmt, "u8", a[2], a[3], None)
    if base.startswith("stem_s2d"):
        return sig_stem(fmt, "f32", a[2], a[3], None)
    if base.startswith("layernorm"):
        return sig_ln(fmt, a[1], a[2], a[3], a[4], a[8], a[9])
    if base.startswith("window_attention"):
        return sig_attn(fmt, a[2], a[3], a[4], a[5], a[7], a[8])
    if base.startswith("patch_embed_rows_u8_padded"):
        return sig_embed(fmt, "u8v", a[2], a[3])
    if base.startswith("patch_embed_rows_u8"):
        return sig_embed(fmt, "u8", a[2], a[3])
    if base.startswith("patch_embed_rows"):
        return sig_embed(fmt, "f32", a[2], a[3])
    if base.startswith("patch_merge_gather"):
        return sig_gather("merge", fmt, a[2], a[3])
    assert base.startswith("subsample2"), name
    return sig_gather("subsample2", fmt, a[2], a[3])


ENTRY_POINTS = ["orp_%s_%s" % (k, f) for f in ("f16x3", "bf16")
                for k in ("gn_stats", "maxpool3x3s2", "stem_s2d", "stem_s2d_u8", "stem_s2d_u8_padded", "layernorm",
                          "window_attention", "patch_embed_rows", "patch_embed_rows_u8", "patch_embed_rows_u8_padded",
                          "patch_merge_gather", "subsample2")] + ["orp_gn_apply_f16x3_multi", "orp_gn_apply_bf16_multi"]


def _call(name, *args):
    """one launch through the library; returns its signature"""
    _lib.check(getattr(_lib.lib(), name)(*args), name)
    return call_signature(name, args)


# ------------------------------------------------------------------------------------------------------------ cases
# (kind, fmt, spec).  The production shapes come from the bench workloads: R-50 x16 and x1, R-101 x4, Swin-T x8 at 1024^2,
# and the test scale (R-101 x4, Swin-T x8 resized to 960^2 with extents).  FPN levels at 1024^2: 128, 64, 32, 16, 8; at
# 960^2: 120, 60, 30, 15, 8.  Swin-T stages at 1024^2: 256, 128, 64, 32 (windows padded to 259, 133, 70, 35); at 960^2:
# 240, 120, 60, 30 (245, 126, 63, 35).
FMTS = ("f16x3", "bf16")
LEVELS = {1024: (128, 64, 32, 16, 8), 960: (120, 60, 30, 15, 8)}
STAGES = {1024: (256, 128, 64, 32), 960: (240, 120, 60, 30)}
HEADS = (3, 6, 12, 24)
STD_RGB = dict(mean=(123.675, 116.28, 103.53), std=(58.395, 57.12, 57.375))


def _build_cases():
    cases = []
    for fmt in FMTS:
        # GroupNorm apply with exact statistics: the head towers (5 levels in one launch, ReLU), the FPN laterals with the
        # top-down add, the FPN outputs
        for n, size in ((16, 1024), (1, 1024), (4, 960), (8, 960)):
            lv = LEVELS[size]
            cases.append(("gn_apply", fmt, dict(probs=[(n, s, s, False) for s in lv], relu=1)))
            cases.append(("gn_apply", fmt, dict(probs=[(n, lv[1], lv[1], True)], relu=0)))
            cases.append(("gn_apply", fmt, dict(probs=[(n, lv[2], lv[2], False)], relu=0)))
        cases.append(("gn_apply", fmt, dict(probs=[(4, 120, 120, True)], relu=0)))
        cases.append(("gn_apply", fmt, dict(probs=[(4, 15, 15, False)], relu=0)))
        # odd top-down pairs, ReLU with the add, eight problems of mixed sizes
        cases.append(("gn_apply", fmt, dict(probs=[(2, 25, 25, True)], relu=0)))
        cases.append(("gn_apply", fmt, dict(probs=[(2, 15, 15, True)], relu=1)))
        cases.append(("gn_apply", fmt, dict(probs=[(1, 15, 26, True), (3, 9, 9, False), (1, 1, 1, True), (2, 7, 5, False),
                                                   (1, 64, 33, True), (1, 8, 8, False), (2, 3, 40, True), (1, 16, 16, False)],
                                            relu=1)))
        # GroupNorm end to end: statistics from orp_gn_stats_* at per-group |mean| / std = r, then the apply step
        for hw in (8, 15, 128):
            for r in (0, 4, 16, 64):
                cases.append(("gn_e2e", fmt, dict(src="stats", N=2, H=hw, W=hw, r=r)))
        cases.append(("gn_e2e", fmt, dict(src="stats", N=16, H=128, W=128, r=4)))    # capped slab count, ragged slabs
        cases.append(("gn_e2e", fmt, dict(src="stats", N=16, H=8, W=8, r=4)))
        cases.append(("gn_e2e", fmt, dict(src="stats", N=4, H=15, W=15, r=4)))
        # max-pool after the stem: 16 x 512^2, and odd sizes
        cases.append(("maxpool", fmt, dict(N=16, H=512, W=512, C=64)))
        for h, w in ((33, 41), (34, 41), (33, 40)):
            cases.append(("maxpool", fmt, dict(N=2, H=h, W=w, C=64)))
        # stems: 16 x 1024^2 uint8, 4 x 960^2 uint8 with full extents, float input, extents with an odd width and an empty image
        cases.append(("stem", fmt, dict(src="u8", N=16, H=1024, W=1024, to_rgb=1)))
        cases.append(("stem", fmt, dict(src="u8v", N=4, H=960, W=960, valid=[(960, 960)] * 4, to_rgb=1)))
        cases.append(("stem", fmt, dict(src="f32", N=2, H=106, W=130)))
        cases.append(("stem", fmt, dict(src="u8v", N=3, H=64, W=70, valid=[(64, 37), (0, 70), (51, 70)], to_rgb=1)))
        cases.append(("stem", fmt, dict(src="u8v", N=2, H=64, W=70, valid=[(40, 56), (64, 70)], to_rgb=0)))
        # LayerNorm: every Swin-T norm at 8 x 1024^2 and 8 x 960^2 (norm1 into the padded grid, norm2 / out norms, merge
        # norms at 4C), widths that are not Swin's and token counts that leave the last block partial
        for size in (1024, 960):
            for i, s in enumerate(STAGES[size]):
                c, sp = 96 << i, -(-s // 7) * 7
                cases.append(("ln", fmt, dict(B=8, H=s, W=s, C=c, Hp=sp, Wp=sp)))
                cases.append(("ln", fmt, dict(B=8, H=s, W=s, C=c, Hp=s, Wp=s)))
                if i < 3:
                    cases.append(("ln", fmt, dict(B=8, H=s // 2, W=s // 2, C=4 * c, Hp=s // 2, Wp=s // 2)))
        for c in (8, 40, 776, 1000, 1536, 96):
            cases.append(("ln", fmt, dict(B=3, H=5, W=7, C=c, Hp=5, Wp=7)))
            cases.append(("ln", fmt, dict(B=2, H=9, W=6, C=c, Hp=14, Wp=7)))
        # window attention: every (stage, shift) at 8 x 1024^2 and 8 x 960^2; grids without padding, H <= 7, a sharp softmax
        for size in (1024, 960):
            for s, heads in zip(STAGES[size], HEADS):
                for shift in (0, 3):
                    cases.append(("attn", fmt, dict(B=8, H=s, W=s, heads=heads, shift=shift)))
        for h, w, heads, shift in ((14, 21, 3, 3), (14, 21, 2, 0), (7, 7, 4, 3), (5, 6, 2, 3), (7, 12, 1, 3), (12, 7, 3, 0),
                                   (19, 9, 12, 3)):
            cases.append(("attn", fmt, dict(B=2, H=h, W=w, heads=heads, shift=shift)))
        for shift in (0, 3):
            cases.append(("attn", fmt, dict(B=2, H=20, W=23, heads=6, shift=shift, sharp=True)))
        # patch-embed rows: 8 x 1024^2 uint8, 8 x 960^2 with extents, float input and uint8 at H % 4 = 1, 2, 3
        cases.append(("embed", fmt, dict(src="u8", B=8, H=1024, W=1024)))
        cases.append(("embed", fmt, dict(src="u8v", B=8, H=960, W=960, valid=[(960, 960)] * 8)))
        cases.append(("embed", fmt, dict(src="f32", B=2, H=64, W=64)))
        for h, w in ((37, 50), (38, 49), (39, 52)):
            cases.append(("embed", fmt, dict(src="f32", B=2, H=h, W=w)))
            cases.append(("embed", fmt, dict(src="u8", B=2, H=h, W=w)))
            cases.append(("embed", fmt, dict(src="u8v", B=3, H=h, W=w, valid=[(h, w), (h - 5, w - 3), (0, w)])))
        # merge gathers of Swin-T at 8 x 1024^2 and 8 x 960^2, P6 / P7 subsampling 32 -> 16 -> 8 and 30 -> 15 -> 8, odd sizes
        for size in (1024, 960):
            for i, s in enumerate(STAGES[size][:3]):
                cases.append(("merge", fmt, dict(B=8, H=s, W=s, C=96 << i)))
            p5 = STAGES[size][3]
            cases.append(("subsample2", fmt, dict(B=8, H=p5, W=p5, C=256)))
            cases.append(("subsample2", fmt, dict(B=8, H=(p5 + 1) // 2, W=(p5 + 1) // 2, C=256)))
        for h, w in ((9, 11), (10, 11), (9, 10)):
            cases.append(("merge", fmt, dict(B=2, H=h, W=w, C=96)))
            cases.append(("subsample2", fmt, dict(B=2, H=h, W=w, C=256)))
    # the fused GroupNorm statistics of a convolution epilogue (f16x3: bf16 sums the fp32 accumulator but normalises the
    # rounded output, so its reference is not the stored tensor)
    for hw in (15, 128):
        for r in (0, 4, 16, 64):
            cases.append(("gn_e2e", "f16x3", dict(src="conv", N=2, H=hw, W=hw, r=r)))
    return cases


CASES = _build_cases()


def case_signature(c):
    kind, fmt, s = c
    if kind == "gn_apply":
        return sig_gn_apply(fmt, s["probs"], s["relu"])
    if kind == "gn_e2e":
        return sig_gn_stats(fmt, s["N"], s["H"] * s["W"]) if s["src"] == "stats" else ("gn_fused_conv", fmt)
    if kind == "maxpool":
        return sig_maxpool(fmt, s["H"], s["W"])
    if kind == "stem":
        return sig_stem(fmt, s["src"], s["H"], s["W"], s.get("valid"))
    if kind == "ln":
        return sig_ln(fmt, s["B"], s["H"], s["W"], s["C"], s["Hp"], s["Wp"])
    if kind == "attn":
        return sig_attn(fmt, s["H"], s["W"], -(-s["H"] // 7) * 7, -(-s["W"] // 7) * 7, s["heads"], s["shift"])
    if kind == "embed":
        return sig_embed(fmt, s["src"], s["H"], s["W"])
    return sig_gather(kind, fmt, s["H"], s["W"])


def _case_id(c):
    kind, fmt, s = c
    if kind == "gn_apply":
        body = "+".join("%dx%dx%d%s" % (n, h, w, "up" if u else "") for n, h, w, u in s["probs"]) + ("-relu" if s["relu"] else "")
    else:
        body = "-".join("%s%s" % (k, v if not isinstance(v, list) else "x".join("%d.%d" % t for t in v[:3]))
                        for k, v in s.items())
    return "%s-%s-%s" % (kind, fmt, body)


# ------------------------------------------------------------------------------------------------------------ helpers
def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / (b.double().abs().max() + 1e-30))


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
        return self.t.view(torch.int16).clone()


def _twice(launch, outs, prepare=None):
    """launch into outputs filled with each NaN pattern in turn (prepare() may then overwrite parts, e.g. a zero border):
    the guards stay untouched and both results are bitwise equal.  Returns the launch's signature."""
    bits, sig = [], None
    for pat in PATTERNS:
        for o in outs:
            o.fill(pat)
        if prepare is not None:
            prepare()
        sig = launch()
        torch.cuda.synchronize()
        for o in outs:
            assert o.guards_intact(pat), "a store landed outside the output"
        bits.append([o.bits() for o in outs])
    for i, (a, b) in enumerate(zip(*bits)):
        assert torch.equal(a, b), "output %d differs between launches (an element not written, or not reproducible)" % i
    return sig


def _split(v):
    """fp32 values -> (hi, lo) fp16 as the kernels split them: saturate, round to nearest, round the remainder"""
    a = v.float().clamp(-65504.0, 65504.0)
    hi = a.half()
    return hi, (a - hi.float()).half()


def _act(fmt, x):
    """fp32 [..., C] -> the activation format: bf16 [..., C] or split fp16 [..., 2, C]"""
    if fmt == "bf16":
        return x.bfloat16().contiguous()
    return torch.stack(_split(x), dim=-2).contiguous()


def _val(fmt, t):
    """the fp64 values of an activation tensor"""
    return t.double() if fmt == "bf16" else t[..., 0, :].double() + t[..., 1, :].double()


def _out(fmt, dev, *shape):
    """a guarded activation tensor [..., C] in the format"""
    shape = shape if fmt == "bf16" else shape[:-1] + (2, shape[-1])
    return Guarded(shape, torch.bfloat16 if fmt == "bf16" else torch.float16, dev)


def _bits(t):
    return t.contiguous().view(torch.int16)


def _st():
    return _lib.current_stream_ptr()


def _valid_tensor(valid, dev):
    t = torch.tensor(valid, dtype=torch.int32, device=dev).contiguous()
    _VALID[t.data_ptr()] = [tuple(v) for v in valid]
    return t


def _normalise_u8(img, to_rgb, valid, stdinv):
    """uint8 HWC [N,H,W,3] -> fp32 NCHW as mmcv.imnormalize computes it ((x - mean) * stdinv in fp32, model channel c from
    image channel 2 - c with to_rgb), zero outside the extents (Pad after Normalize)"""
    x = img.permute(0, 3, 1, 2).float()
    if to_rgb:
        x = x.flip(1)
    mean = torch.tensor(STD_RGB["mean"], dtype=torch.float32, device=img.device).view(1, 3, 1, 1)
    x = (x - mean) * stdinv.view(1, 3, 1, 1)
    if valid is not None:
        n, _, h, w = x.shape
        yy = torch.arange(h, device=img.device).view(1, h, 1)
        xx = torch.arange(w, device=img.device).view(1, 1, w)
        v = torch.tensor(valid, device=img.device)
        keep = (yy < v[:, 0].view(n, 1, 1)) & (xx < v[:, 1].view(n, 1, 1))
        x = torch.where(keep.unsqueeze(1), x, torch.zeros((), device=img.device))     # +0.0, as the kernels write
    return x


# ------------------------------------------------------------------------------------------------------------ GroupNorm
def _gn_params(dev, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(256, generator=g) + 0.5).to(dev), (torch.randn(256, generator=g) * 0.1).to(dev)


def _gn_launch(fmt, xs, stats, ups, ys, gamma, beta, relu):
    arr = (_lib.GnProblem * len(xs))()
    for i, x in enumerate(xs):
        arr[i].x, arr[i].N, arr[i].H, arr[i].W = x.data_ptr(), x.shape[0], x.shape[1], x.shape[2]
        arr[i].stats = stats[i].data_ptr()
        arr[i].up_src = ups[i].data_ptr() if ups[i] is not None else None
        arr[i].y = ys[i].data_ptr()
    return _call("orp_gn_apply_%s_multi" % fmt, len(xs), arr, 256, 32, _lib.ptr(gamma), _lib.ptr(beta), 1e-5, int(relu), _st())


def _gn_ref(v, gamma, beta, relu, up):
    """F.group_norm in fp64 (+ ReLU) + the nearest-upsampled top-down source, NHWC"""
    y = F.group_norm(v.permute(0, 3, 1, 2), 32, gamma.double(), beta.double(), 1e-5)
    if relu:
        y = torch.relu(y)
    if up is not None:
        y = y + F.interpolate(up.permute(0, 3, 1, 2), size=tuple(v.shape[1:3]), mode="nearest")
    return y.permute(0, 2, 3, 1)


def _exact_stats(v):
    r = v.reshape(v.shape[0], -1, 32, 8).transpose(1, 2).reshape(v.shape[0], 32, -1)
    return torch.stack([r.sum(2), (r * r).sum(2)], dim=2).contiguous()


def _check_gn_apply(fmt, xs, stats, ups, gamma, beta, relu, tol):
    dev = xs[0].device
    outs = [_out(fmt, dev, *x.shape[:3], 256) for x in xs]
    sig = _twice(lambda: _gn_launch(fmt, xs, stats, ups, [o.t for o in outs], gamma, beta, relu), outs)
    err = 0.0
    for x, up, o in zip(xs, ups, outs):
        y = _val(fmt, o.t)
        assert bool(torch.isfinite(y).all()), "an output element was not written"
        err = max(err, _rel(y, _gn_ref(_val(fmt, x), gamma, beta, relu, None if up is None else _val(fmt, up))))
    assert err < tol, (err, tol)
    return sig, err


def run_gn_apply(fmt, s, dev, g):
    xs, ups = [], []
    for n, h, w, up in s["probs"]:
        off = torch.randn(1, 1, 1, 256, generator=g) * 2                   # per-channel offsets: |mean| / std up to ~4
        xs.append(_act(fmt, (torch.randn(n, h, w, 256, generator=g) * 1.5 + off).to(dev)))
        ups.append(_act(fmt, torch.randn(n, (h + 1) // 2, (w + 1) // 2, 256, generator=g).to(dev)) if up else None)
    stats = [_exact_stats(_val(fmt, x)) for x in xs]
    gamma, beta = _gn_params(dev, 5)
    return _check_gn_apply(fmt, xs, stats, ups, gamma, beta, s["relu"], GN_APPLY_TOL[fmt])


def run_gn_e2e(fmt, s, dev, g):
    """statistics computed by the library at per-group |mean| / std = r, normalised by gn_apply, against F.group_norm of
    the stored values in fp64"""
    n, h, w, r = s["N"], s["H"], s["W"], s["r"]
    sign = torch.where(torch.rand(32, generator=g) < 0.5, -1.0, 1.0).repeat_interleave(8)
    off = (r * sign + torch.randn(256, generator=g) * 0.05).view(1, 1, 1, 256)
    stats = torch.zeros((n, 32, 2), dtype=torch.float64, device=dev)
    if s["src"] == "stats":
        x = _act(fmt, (torch.randn(n, h, w, 256, generator=g) + off).to(dev))
        sig = _call("orp_gn_stats_%s" % fmt, _lib.ptr(x), n, h * w, 256, 32, _lib.ptr(stats), _st())
    else:
        from orientedreppoints_b200.detector import ConvLayer
        from orientedreppoints_b200.engine_tc import EngineTCSplit
        # the epilogue fuses the statistics only without bias: input channel 0 is 1.0 and its weights carry the offsets
        wt = torch.randn(256, 192, 1, 1, generator=g) / 191 ** 0.5
        wt[:, 0, 0, 0] = off.view(256)
        xin = torch.randn(n, h, w, 192, generator=g)
        xin[..., 0] = 1.0
        x = EngineTCSplit(dev).conv_multi([_act(fmt, xin.to(dev))], ConvLayer(wt, None, 1, 0, dev), stats=[stats])[0]
        assert _lib.tc_last_plan()["gn_fused"] == 1, "the convolution did not fuse the statistics"
        sig = ("gn_fused_conv", fmt)
    torch.cuda.synchronize()
    gamma, beta = _gn_params(dev, 6)
    tol = GN_E2E_R64_TOL if (fmt == "f16x3" and r > 16) else GN_E2E_TOL[fmt]
    _, err = _check_gn_apply(fmt, [x], [stats], [None], gamma, beta, 0, tol)
    v = _val(fmt, x)
    ex = _exact_stats(v)
    mean = ex[..., 0] / (h * w * 8)
    var = ex[..., 1] / (h * w * 8) - mean * mean
    print("r=%d: |mean|/std %.1f, GroupNorm output rel err %.2e" % (r, float((mean.abs() / var.sqrt()).max()), err))
    return sig, err


# ------------------------------------------------------------------------------------------------------------ others
def run_maxpool(fmt, s, dev, g):
    n, h, w, c = s["N"], s["H"], s["W"], s["C"]
    x = _act(fmt, torch.randn(n, h, w, c, generator=g).to(dev))
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    out = _out(fmt, dev, n, ho, wo, c)
    sig = _twice(lambda: _call("orp_maxpool3x3s2_%s" % fmt, _lib.ptr(x), n, h, w, c, _lib.ptr(out.t), _st()), [out])
    ref = F.max_pool2d(_val(fmt, x).permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    assert torch.equal(_bits(out.t), _bits(_act(fmt, ref.float())))
    return sig, 0.0


def run_stem(fmt, s, dev, g):
    n, h, w, src = s["N"], s["H"], s["W"], s["src"]
    hp, wp = h // 2 + 3, w // 2 + 3
    out = Guarded((2, n, hp, wp, 16) if fmt == "f16x3" else (n, hp, wp, 16), torch.float16 if fmt == "f16x3" else torch.bfloat16, dev)
    if src == "f32":
        v = torch.randn(n, 3, h, w, generator=g).to(dev)
        launch = lambda: _call("orp_stem_s2d_%s" % fmt, _lib.ptr(v), n, h, w, _lib.ptr(out.t), _st())   # noqa: E731
    else:
        img = torch.randint(0, 256, (n, h, w, 3), generator=g, dtype=torch.uint8).to(dev)
        mean, std = (ctypes.c_float * 3)(*STD_RGB["mean"]), (ctypes.c_float * 3)(*STD_RGB["std"])
        stdinv = torch.tensor([1.0 / float(ctypes.c_float(v).value) for v in STD_RGB["std"]], dtype=torch.float32, device=dev)
        valid = s.get("valid")
        v = _normalise_u8(img, s["to_rgb"], valid, stdinv)
        if src == "u8":
            launch = lambda: _call("orp_stem_s2d_u8_%s" % fmt, _lib.ptr(img), n, h, w, mean, std, s["to_rgb"],   # noqa: E731
                                   _lib.ptr(out.t), _st())
        else:
            vt = _valid_tensor(valid, dev)
            launch = lambda: _call("orp_stem_s2d_u8_padded_%s" % fmt, _lib.ptr(img), n, h, w, mean, std,   # noqa: E731
                                   s["to_rgb"], _lib.ptr(vt), _lib.ptr(out.t), _st())
    sig = _twice(launch, [out])
    # out[n][Y][X][(dy * 2 + dx) * 3 + c] = v[n][c][2 (Y - 2) + dy][2 (X - 2) + dx], zero outside, channels 12..15 zero
    t = F.pad(v, (4, 2, 4, 2)).view(n, 3, hp, 2, wp, 2).permute(0, 2, 4, 3, 5, 1).reshape(n, hp, wp, 12)
    ref = F.pad(t, (0, 4))
    want = torch.stack(_split(ref)) if fmt == "f16x3" else ref.bfloat16()
    assert torch.equal(_bits(out.t), _bits(want))
    return sig, 0.0


def run_ln(fmt, s, dev, g):
    b, h, w, c, hp, wp = s["B"], s["H"], s["W"], s["C"], s["Hp"], s["Wp"]
    x = _act(fmt, (torch.randn(b, h, w, c, generator=g) * 2 + torch.randn(b, h, w, 1, generator=g) * 3).to(dev))
    gamma = (torch.rand(c, generator=g) + 0.5).to(dev)
    beta = torch.randn(c, generator=g).to(dev)
    out = _out(fmt, dev, b, hp, wp, c)

    def zero_border():
        out.t[:, h:].zero_()
        out.t[:, :, w:].zero_()
    padded = (hp, wp) != (h, w)
    sig = _twice(lambda: _call("orp_layernorm_%s" % fmt, _lib.ptr(x), b, h, w, c, _lib.ptr(gamma), _lib.ptr(beta), 1e-5, hp, wp,
                               _lib.ptr(out.t), _st()), [out], zero_border if padded else None)
    if padded:
        assert not bool(_bits(out.t[:, h:]).any()) and not bool(_bits(out.t[:, :, w:]).any()), "the padding was written"
    y = _val(fmt, out.t[:, :h, :w])
    assert bool(torch.isfinite(y).all()), "a token was not written"
    err = _rel(y, F.layer_norm(_val(fmt, x), (c,), gamma.double(), beta.double(), 1e-5))
    assert err < LN_TOL[fmt], (err, LN_TOL[fmt])
    return sig, err


def run_attn(fmt, s, dev, g):
    from oracle import torch_swin as ts
    b, h, w, heads, shift = s["B"], s["H"], s["W"], s["heads"], s["shift"]
    c, hp, wp = heads * 32, -(-h // 7) * 7, -(-w // 7) * 7
    if s.get("sharp"):
        # q and k scaled so the logits span about +-30, bias entries up to +-10: most probabilities far below fp16's normal range
        qkv = torch.randn(b, hp, wp, 3, c, generator=g) * torch.tensor([3.2, 3.2, 1.0]).view(1, 1, 1, 3, 1)
        table = (torch.rand(169, heads, generator=g) * 20 - 10).to(dev)
    else:
        qkv = torch.randn(b, hp, wp, 3, c, generator=g)
        table = (torch.randn(169, heads, generator=g) * 0.5).to(dev)
    x = _act(fmt, qkv.reshape(b, hp, wp, 3 * c).to(dev))
    scale = float(ctypes.c_float(32 ** -0.5).value)
    out = _out(fmt, dev, b, h, w, c)
    sig = _twice(lambda: _call("orp_window_attention_%s" % fmt, _lib.ptr(x), b, h, w, hp, wp, c, heads, shift, _lib.ptr(table),
                               scale, _lib.ptr(out.t), _st()), [out])
    y = _val(fmt, out.t)
    assert bool(torch.isfinite(y).all()), "a token was not written"
    xv = _val(fmt, x)
    del x
    sx = torch.roll(xv, shifts=(-shift, -shift), dims=(1, 2)) if shift else xv
    q, k, v = ts.window_partition(sx, 7).view(-1, 49, 3, heads, 32).permute(2, 0, 3, 1, 4)
    del sx
    mask = ts.shift_mask(hp, wp, shift, dev).double() if shift else None
    aw = ts.attention_core(q * (scale / 32 ** -0.5), k, v, table.double(), heads, mask).view(-1, 7, 7, c)
    del q, k, v
    ref = ts.window_reverse(aw, 7, hp, wp)
    ref = (torch.roll(ref, shifts=(shift, shift), dims=(1, 2)) if shift else ref)[:, :h, :w]
    err = _rel(y, ref)
    assert err < ATTN_TOL[fmt], (err, ATTN_TOL[fmt])
    return sig, err


def run_embed(fmt, s, dev, g):
    b, h, w, src = s["B"], s["H"], s["W"], s["src"]
    ho, wo = (h + 3) // 4, (w + 3) // 4
    out = _out(fmt, dev, b, ho, wo, 64)
    if src == "f32":
        v = torch.randn(b, 3, h, w, generator=g).to(dev)
        launch = lambda: _call("orp_patch_embed_rows_%s" % fmt, _lib.ptr(v), b, h, w, _lib.ptr(out.t), _st())   # noqa: E731
    else:
        img = torch.randint(0, 256, (b, h, w, 3), generator=g, dtype=torch.uint8).to(dev)
        mean = (ctypes.c_float * 3)(*STD_RGB["mean"])
        stdinv = (ctypes.c_float * 3)(*[1.0 / v for v in STD_RGB["std"]])
        valid = s.get("valid")
        v = _normalise_u8(img, 1, valid, torch.tensor(list(stdinv), dtype=torch.float32, device=dev))
        if src == "u8":
            launch = lambda: _call("orp_patch_embed_rows_u8_%s" % fmt, _lib.ptr(img), b, h, w, mean, stdinv, 1,   # noqa: E731
                                   _lib.ptr(out.t), _st())
        else:
            vt = _valid_tensor(valid, dev)
            launch = lambda: _call("orp_patch_embed_rows_u8_padded_%s" % fmt, _lib.ptr(img), b, h, w, mean, stdinv, 1,   # noqa: E731
                                   _lib.ptr(vt), _lib.ptr(out.t), _st())
    sig = _twice(launch, [out])
    # rows[b, oh, ow, c * 16 + kh * 4 + kw] = v[b, c, 4 oh + kh, 4 ow + kw], zero beyond the image and for k >= 48
    ip = F.pad(v, (0, 4 * wo - w, 0, 4 * ho - h))
    ref = F.pad(ip.unfold(2, 4, 4).unfold(3, 4, 4).permute(0, 2, 3, 1, 4, 5).reshape(b, ho, wo, 48), (0, 16))
    assert torch.equal(_bits(out.t), _bits(_act(fmt, ref)))
    return sig, 0.0


def run_gather(kind, fmt, s, dev, g):
    b, h, w, c = s["B"], s["H"], s["W"], s["C"]
    x = _act(fmt, torch.randn(b, h, w, c, generator=g).to(dev))
    if kind == "merge":
        ho, wo = (h + 1) // 2, (w + 1) // 2
        out = _out(fmt, dev, b, ho, wo, 4 * c)
        sig = _twice(lambda: _call("orp_patch_merge_gather_%s" % fmt, _lib.ptr(x), b, h, w, c, _lib.ptr(out.t), _st()), [out])
        xp = torch.zeros((b, 2 * ho, 2 * wo) + tuple(x.shape[3:]), dtype=x.dtype, device=dev)
        xp[:, :h, :w] = x
        # PatchMerging: x(0::2, 0::2) | x(1::2, 0::2) | x(0::2, 1::2) | x(1::2, 1::2), per plane
        ref = torch.cat([xp[:, 0::2, 0::2], xp[:, 1::2, 0::2], xp[:, 0::2, 1::2], xp[:, 1::2, 1::2]], -1)
    else:
        ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        out = _out(fmt, dev, b, ho, wo, c)
        sig = _twice(lambda: _call("orp_subsample2_%s" % fmt, _lib.ptr(x), b, h, w, c, _lib.ptr(out.t), _st()), [out])
        ref = x[:, ::2, ::2]                                            # max_pool2d(kernel 1, stride 2)
    assert torch.equal(_bits(out.t), _bits(ref))
    return sig, 0.0


RUNNERS = dict(gn_apply=run_gn_apply, gn_e2e=run_gn_e2e, maxpool=run_maxpool, stem=run_stem, ln=run_ln, attn=run_attn,
               embed=run_embed)


# ------------------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("c", CASES, ids=[_case_id(c) for c in CASES])
def test_token_kernel(cuda, c):
    kind, fmt, s = c
    g = torch.Generator().manual_seed(CASES.index(c) + 11)
    run = RUNNERS.get(kind)
    sig, err = run(fmt, s, cuda, g) if run is not None else run_gather(kind, fmt, s, cuda, g)
    assert sig == case_signature(c), "the case left its signature: %s" % (sig,)
    print("%s: %s rel err %.2e" % (_case_id(c), sig, err))
    torch.cuda.empty_cache()


WORKLOADS_TEST_SCALE = [("r101", "f16x3", 4), ("swin_tiny", "f16x3", 8)]


def test_production_signatures_are_covered(cuda, monkeypatch):
    """one forward_dense of each bench workload (test_conv_plans_gpu.WORKLOADS at 1024^2, and the test-scale workloads through
    the config's test pipeline with extents): every call to the entry points above must reach a signature CASES pins"""
    from test_conv_plans_gpu import WORKLOADS

    from orientedreppoints_b200 import engine_tc
    from orientedreppoints_b200.bench_tile import _config_test_pipeline, build_detector
    from orientedreppoints_b200.datasets.pipelines import run_test_pipeline
    seen = {}
    name = [None]

    def note(sig):
        e = seen.setdefault(sig, dict(calls=0, workloads=set()))
        e["calls"] += 1
        e["workloads"].add(name[0])

    lib = _lib.lib()
    for ep in ENTRY_POINTS:
        fn = getattr(lib, ep)

        def recorded(*a, _fn=fn, _ep=ep):
            note(call_signature(_ep, a))
            return _fn(*a)
        monkeypatch.setattr(lib, ep, recorded)
    valid_fn = engine_tc._valid

    def valid(valid_hw, n, device):
        t = valid_fn(valid_hw, n, device)
        _VALID[t.data_ptr()] = [tuple(v) for v in t.tolist()]
        return t
    monkeypatch.setattr(engine_tc, "_valid", valid)

    runs = [(b, p, n, False) for b, p, n in WORKLOADS] + [(b, p, n, True) for b, p, n in WORKLOADS_TEST_SCALE]
    for backbone, prec, batch, test_scale in runs:
        name[0] = "%s %s x%d%s" % (backbone, prec, batch, " test scale" if test_scale else "")
        _, det = build_detector(backbone, prec, cuda)
        eng = det.eng

        # GroupNorm statistics the convolution library computes in a separate pass (split-K launches, and launches whose
        # epilogue cannot fuse them) call orp_gn_stats_* from C
        def launch(*a, _f=eng._launch, **kw):
            out = _f(*a, **kw)
            if kw.get("stats") is not None and not _lib.tc_last_plan()["gn_fused"]:
                for y in a[1]:
                    note(sig_gn_stats(eng.name, y.shape[0], y.shape[1] * y.shape[2]))
            return out

        def splitk(x, y, tc, L, relu, ks, stats, f16x3, _f=eng._conv_splitk):
            out = _f(x, y, tc, L, relu, ks, stats, f16x3)
            if stats is not None:
                note(sig_gn_stats(eng.name, y.shape[0], y.shape[1] * y.shape[2]))
            return out
        eng._launch, eng._conv_splitk = launch, splitk
        tiles = torch.randint(0, 256, (batch, 1024, 1024, 3), generator=torch.Generator().manual_seed(1), dtype=torch.uint8).to(cuda)
        with torch.no_grad():
            if test_scale:
                data = run_test_pipeline(_config_test_pipeline(backbone), tiles, device=cuda)
                (view,), (vhw,) = data["img"], data["valid_hw"]
                det.forward_dense(view, valid_hw=vhw)
            else:
                det.forward_dense(tiles)
        torch.cuda.synchronize()
        del det, eng, tiles
        torch.cuda.empty_cache()
    pinned = {case_signature(c) for c in CASES}
    print("\n%-6s %-60s %6s  workloads" % ("pinned", "signature", "calls"))
    for sig, e in sorted(seen.items(), key=lambda kv: str(kv[0])):
        print("%-6s %-60s %6d  %s" % ("yes" if sig in pinned else "NO", sig, e["calls"], ", ".join(sorted(e["workloads"]))))
    missing = [s for s in seen if s not in pinned]
    assert not missing, "production launches without a case: %s" % missing


def test_invalid_launches_are_refused(cuda):
    """each refusal comes before any launch; the tensors are large enough for the shapes claimed, so nothing could go out of
    range even if one were not refused"""
    lib, st = _lib.lib(), _st()
    big = torch.zeros(1 << 22, dtype=torch.float16, device=cuda)
    out = torch.full((1 << 22,), 7.0, dtype=torch.float16, device=cuda)
    gamma = torch.ones(2048, device=cuda)
    table = torch.zeros(169 * 24, device=cuda)
    stats = torch.zeros(64 * 32 * 2, dtype=torch.float64, device=cuda)
    p, o = _lib.ptr(big), _lib.ptr(out)
    for fmt in FMTS:
        ln = getattr(lib, "orp_layernorm_%s" % fmt)
        assert ln(p, 1, 4, 4, 12, _lib.ptr(gamma), _lib.ptr(gamma), 1e-5, 4, 4, o, st) == ORP_EINVAL        # C % 8
        assert ln(p, 1, 4, 4, 1544, _lib.ptr(gamma), _lib.ptr(gamma), 1e-5, 4, 4, o, st) == ORP_EINVAL      # C > 1536
        assert ln(p, 1, 4, 4, 96, _lib.ptr(gamma), _lib.ptr(gamma), 1e-5, 3, 4, o, st) == ORP_EINVAL        # Hp < H
        assert ln(p, 1, 4, 4, 96, _lib.ptr(gamma), _lib.ptr(gamma), 1e-5, 4, 3, o, st) == ORP_EINVAL        # Wp < W
        at = getattr(lib, "orp_window_attention_%s" % fmt)
        scale = 32 ** -0.5
        assert at(p, 1, 7, 7, 7, 7, 96, 2, 0, _lib.ptr(table), scale, o, st) == ORP_EINVAL                   # heads * 32 != C
        assert at(p, 1, 7, 7, 7, 7, 96, 3, 7, _lib.ptr(table), scale, o, st) == ORP_EINVAL                   # shift >= 7
        assert at(p, 1, 7, 7, 7, 7, 96, 3, -1, _lib.ptr(table), scale, o, st) == ORP_EINVAL
        assert at(p, 1, 7, 8, 7, 8, 96, 3, 0, _lib.ptr(table), scale, o, st) == ORP_EINVAL                   # Wp % 7
        assert at(p, 1, 8, 7, 8, 7, 96, 3, 0, _lib.ptr(table), scale, o, st) == ORP_EINVAL                   # Hp % 7
        assert getattr(lib, "orp_gn_stats_%s" % fmt)(p, 1, 16, 128, 32, _lib.ptr(stats), st) == ORP_EINVAL  # C != 256
        arr = (_lib.GnProblem * 9)()
        for i in range(9):
            arr[i].x, arr[i].N, arr[i].H, arr[i].W = big.data_ptr(), 1, 2, 2
            arr[i].stats, arr[i].y = stats.data_ptr(), out.data_ptr()
        apply = getattr(lib, "orp_gn_apply_%s_multi" % fmt)
        assert apply(1, arr, 128, 32, _lib.ptr(gamma), _lib.ptr(gamma), 1e-5, 0, st) == ORP_EINVAL          # C != 256
        assert apply(9, arr, 256, 32, _lib.ptr(gamma), _lib.ptr(gamma), 1e-5, 0, st) == ORP_EINVAL          # nprob > 8
    torch.cuda.synchronize()
    assert bool((out == 7.0).all()), "a refused call wrote its output"
