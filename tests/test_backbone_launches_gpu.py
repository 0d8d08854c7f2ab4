"""GPU: every convolution and attention launch of the ResNeXt, HRNet + HRFPN, DCN-stage and GeneralizedAttention graphs at the
benchmark's batch (16 uint8 tiles of 1024^2), and at the test scale (4 tiles through the config's test pipeline to 960^2, with
the valid extents), checked as it happens against fp64 by the checker of tests/test_production_launches_gpu.py.

These graphs reach launches the benchmark workloads never make: HRNet's widths padded to multiples of 8 (24 / 40 / 72 / 144:
Cin below one 64-channel K block or a partly filled last block, Cout padded up inside the N tile), its stride-2 fuse chains with
a 16-bit residual and the fp32-output HRFPN reductions; the attention blocks' Q / KV / proj convolutions; ResNeXt's 1x1
convolutions at its widths and the grouped conv2 inside a real forward; the stride-2 deformable conv2 with and without DCNv2
masks.  For each workload:
- every orp_conv2d / stem / grouped / deformable launch against fp64 on the operands the engine holds, and launched twice more
  into NaN-filled guarded outputs (write-once); every orp_gen_attention launch against the fp64 contract of
  tests/test_gen_attention_gpu.py, and once more into a guarded output;
- no launch outside a checked call, no f16x3 overflow;
- in f16x3, tiles 0 and 15 of the x16 pass within 1e-4 of the family's fp64 graph run on that tile alone;
- every orp_conv2d plan signature pinned by a case of tests/conv_plan_cases.PARITY."""
import time

import pytest
import torch

from orientedreppoints_b200 import gen_attention as ga

import test_production_launches_gpu as tpl
from conv_plan_cases import PARITY, SIG_FIELDS
from test_conv_plans_gpu import PATTERNS, Guarded
from test_gen_attention_gpu import TOL as ATT_TOL, _ref as attention_ref, _tame

pytestmark = pytest.mark.gpu

C3_C5 = (False, True, True, True)


class BackboneChecker(tpl.LaunchChecker):
    """LaunchChecker plus the GeneralizedAttention launches (gen_attention.attend).
    The f16x3 accumulator truncates towards zero: on an H100 each output's error measured 6-8e-7 of its sum of absolute
    products sum |x w|, the same at every pixel, image border or not, and in every image.  Where a channel's products share
    their sign the output comes near that sum and the error near its bound: R-50-GA's layer4.0.c2 (K = 4608) at the 960^2
    test scale measured 9.005e-6 of the image's max on channel 305, at a tolerance of 9.0e-6.  So these graphs' convolutions
    are held to 1.25 times the benchmark workloads' f16x3 bound."""
    conv_margin = 1.25

    def __init__(self, det, name, monkeypatch):
        super().__init__(det, name)
        real = ga.attend

        def counted(*a, **kw):
            self._saw("attention", a, kw)
            return real(*a, **kw)
        self.orig["attend"], self.real_attend = counted, real
        monkeypatch.setattr(ga, "attend", self._attend)

    def _attend(self, eng, q, qc_off, qp_off, kv, k_off, v_off, tables, n, h, w, hk, wk, s, c, heads):
        args = (eng, q, qc_off, qp_off, kv, k_off, v_off, tables, n, h, w, hk, wk, s, c, heads)
        out, _, _ = self._run("attend", *args)
        what = "%s launch %d attention %dx%d -> %dx%d, C %d" % (self.name, self.checked, h, w, hk, wk, c)
        held = lambda t: self.eng.to_float(t).double()                                     # noqa: E731
        qh, kvh = (held(q) if q is not None else None), held(kv)
        px, py = (held(tables[0]).reshape(-1, c), held(tables[1]).reshape(-1, c)) if tables is not None else (None, None)
        got = held(out)
        for j in range(n):
            qj = None if qh is None else qh[j:j + 1].reshape(1, h * w, -1)
            kvj = kvh[j:j + 1].reshape(1, hk * wk, -1)
            ref, energy = attention_ref(None if qc_off is None else qj[..., qc_off:qc_off + c],
                                        None if qp_off is None else qj[..., qp_off:qp_off + c],
                                        None if k_off is None else kvj[..., k_off:k_off + c], kvj[..., v_off:v_off + c],
                                        px, py, h, w, hk, wk, s, heads)
            if self.split:
                tol = ATT_TOL["f16x3"]
            else:                                  # tests/test_gen_attention_gpu.py::test_published_launches_vs_fp64
                tol = 0.02 * max(1.0, float(energy.std()))
            g = got[j].reshape(1, h * w, c)
            assert bool(torch.isfinite(g).all()), "%s: image %d: non-finite output" % (what, j)
            err = float((g - ref).abs().max() / ref.abs().max())
            if err >= tol:
                pix = int((g - ref).abs().amax(2).reshape(-1).argmax())
                raise AssertionError("%s: image %d of %d: rel err %.3e >= %.1e, largest error at (y, x) %s"
                                     % (what, j, n, err, tol, divmod(pix, w)))
            if err > self.worst.get("attention", (-1.0,))[0]:
                self.worst["attention"] = (err, tol, "%s image %d" % (what, j))
        if self.split:
            assert self.eng.overflow_count() == 0, "%s: f16 overflow" % what
        # once more, into a NaN-filled guarded output: bitwise the first result, guards untouched
        guard = Guarded(tuple(out.shape), out.dtype, out.device)
        guard.fill(PATTERNS[0])
        self.replaying, alloc, ga.alloc = True, ga.alloc, (lambda *a: guard.t)
        try:
            self.real_attend(*args)
        finally:
            self.replaying, ga.alloc = False, alloc
        torch.cuda.synchronize()
        assert guard.guards_intact(PATTERNS[0]), "%s: a store landed outside the output" % what
        assert torch.equal(guard.t.view(torch.int16), out.view(torch.int16)), \
            "%s: the re-launch into a NaN-filled buffer differs from the first launch" % what
        self.checked += 1
        return out


# ------------------------------------------------------------------------------------------------------ workloads
def _state(family):
    """(state dict, detector kwargs, fp64 graph: (sd64, img64) -> (outs, feats)) of a family, as its tests build them"""
    from orientedreppoints_b200.weights import (STAGE_BLOCKS, dcn_layout, gen_attention_layout, random_hrnet_state_dict,
                                                random_state_dict)
    if family.startswith("x"):
        depth, groups, bw = {"x101_64x4d": (101, 64, 4), "x50_32x8d": (50, 32, 8)}[family]
        import resnext_ref as xr
        sd = random_state_dict(depth, seed=0, reference_init=False, residual_gain=0.3 if depth == 101 else 1.0, groups=groups,
                               base_width=bw)
        return sd, depth, {}, lambda s, x: xr.forward_dense(s, x, depth, groups)
    if family.startswith("hrnet"):
        import hrnet_ref as hr
        sd = random_hrnet_state_dict(family, seed=0, reference_init=False, residual_gain=0.3)
        return sd, family, {}, lambda s, x: hr.forward_dense(s, x, family, "AVG")
    if family in ("dcn", "dcnv2"):
        import dcn_backbone_ref as dr
        dcn = dict(type="DCN" if family == "dcn" else "DCNv2")
        sd = random_state_dict(50, seed=0, reference_init=False, residual_gain=0.3, dcn=dcn, stage_with_dcn=C3_C5,
                               dcn_offset_scale=1.0)
        lay = dcn_layout(50, dcn, C3_C5)
        return sd, 50, dict(dcn=lay), lambda s, x: dr.forward_dense(s, x, lay, STAGE_BLOCKS[50])
    assert family == "ga"
    import gen_attention_ref as gr
    cfg = dict(gr.PUBLISHED, attention_type="1111")
    sd = _tame(random_state_dict(50, seed=21, reference_init=False, residual_gain=0.5, gen_attention=cfg,
                                 stage_with_gen_attention=gr.PUBLISHED_STAGES, gen_attention_gamma=0.7))
    gal = gen_attention_layout(50, cfg, gr.PUBLISHED_STAGES)
    # tests/gen_attention_ref.py evaluates on the host
    return sd, 50, dict(gen_attention=gal), lambda s, x: gr.forward_dense({k: v.cpu() for k, v in s.items()}, x.cpu(), None, gal)


WORKLOADS = [("x101_64x4d", "f16x3", 16, False), ("x101_64x4d", "bf16", 16, False), ("x101_64x4d", "f16x3", 4, True),
             ("x50_32x8d", "f16x3", 16, False),
             ("hrnetv2p_w18", "f16x3", 16, False), ("hrnetv2p_w18", "bf16", 16, False), ("hrnetv2p_w18", "f16x3", 4, True),
             ("hrnetv2p_w32", "f16x3", 16, False),
             ("dcn", "f16x3", 16, False), ("dcnv2", "f16x3", 16, False),
             ("ga", "f16x3", 16, False), ("ga", "bf16", 16, False), ("ga", "f16x3", 4, True)]


def _tiles_vs_fp64(det, sd, graph64, img, dense, name):
    """tiles 0 and 15 of the eager pass against the family's fp64 graph on that tile alone (tpl._tile_vs_fp64's measure)"""
    outs, feats = dense
    for t in (0, img.shape[0] - 1):
        sdg = {k: v.to(img.device).double() for k, v in sd.items()}
        with torch.no_grad():
            ref_outs, ref_feats = graph64(sdg, tpl._host_normalised64(img[t], det.img_norm_cfg, img.device))
        del sdg
        ref_outs = [[r.to(img.device) for r in o] for o in ref_outs]
        ref_feats = [f.to(img.device) for f in ref_feats]
        errs = {}
        for lvl in range(5):
            errs["feat%d" % lvl] = tpl._rel(tpl._nchw64(det.eng.to_float(feats[lvl][t:t + 1])), ref_feats[lvl])
            for k, nm in enumerate(("cls", "init", "refine")):
                a, b = tpl._nchw64(outs[lvl][k][t:t + 1]), ref_outs[lvl][k]
                assert a.shape == b.shape
                errs["%s%d" % (nm, lvl)] = float((a - b).abs().max()) / max(1.0, float(b.abs().max()))
        worst = max(errs, key=errs.get)
        print("%s tile %d: max rel err %.2e (%s) vs the fp64 graph" % (name, t, errs[worst], worst))
        for k, v in errs.items():
            assert v < tpl.DENSE_TOL, (name, "tile %d" % t, k, v)


def _signatures_pinned(chk):
    """every orp_conv2d / stem plan signature of the pass is pinned by PARITY; the table lists the layers that reach each"""
    pinned = {c[0] for c in PARITY}
    seen = {}
    for sig, layer in zip(chk.sigs, chk.layers):
        e = seen.setdefault(sig, dict(calls=0, layers=[]))
        e["calls"] += 1
        if len(e["layers"]) < 3:
            e["layers"].append(layer)
    print("\n%-6s %-100s %6s  first layers" % ("pinned", " ".join(SIG_FIELDS)[:100], "calls"))
    for sig, e in sorted(seen.items(), key=lambda kv: str(kv[0])):
        print("%-6s %-100s %6d  %s" % ("yes" if sig in pinned else "NO", sig, e["calls"], "; ".join(e["layers"])))
    missing = ["%s (%s)" % (sig, "; ".join(e["layers"])) for sig, e in seen.items() if sig not in pinned]
    assert not missing, "%s: launch plans without a parity case: %s" % (chk.name, missing)


@pytest.mark.parametrize("family,prec,batch,test_scale", WORKLOADS,
                         ids=["%s-%s-x%d%s" % (f, p, n, "-960" if t else "") for f, p, n, t in WORKLOADS])
def test_every_launch_vs_fp64(cuda, monkeypatch, family, prec, batch, test_scale):
    from orientedreppoints_b200.detector import OrientedRepPointsDetector
    t0 = time.time()
    name = "%s %s x%d%s" % (family, prec, batch, " at 960^2" if test_scale else "")
    sd, depth, kw, graph64 = _state(family)
    img, valid = tpl._inputs("r101", batch, test_scale, cuda)      # 960^2: the R-101 config's test pipeline (img_scale 960)
    det = OrientedRepPointsDetector(sd, depth, cuda, prec, test_cfg=dict(score_thr=0.0), **kw)
    chk = BackboneChecker(det, name, monkeypatch)
    if chk.split:
        det.eng.overflow_count()                                      # the counter is global: start from zero
    with torch.no_grad():
        dense = det.forward_dense(img, valid)
    torch.cuda.synchronize()
    line = chk.summary(time.time() - t0)
    print(line)
    assert not chk.escaped, "%s: launches outside a checked call: %s" % (name, chk.escaped)
    assert chk.checked == chk.low and chk.checked > 0, line
    if chk.split:
        assert det.eng.overflow_count() == 0, name
    if chk.split and not test_scale:                                   # north_star's 1e-4 is the f16x3 engine's
        _tiles_vs_fp64(det, sd, graph64, img, dense, name)
    _signatures_pinned(chk)
    print("%s: %.1f s" % (name, time.time() - t0))
    del det, chk, dense
    torch.cuda.empty_cache()
