"""GPU parity tests (run with -m gpu on an H100): the CUDA path through the C-ABI against the
CPU oracle and the committed golden vectors.  Integer/index results bit-exact; fp64 IoU bit-exact;
fp32 'compat32' IoU bit-exact; fp32 'exact64' IoU values within 1e-5 of the fp64 reference."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


# ------------------------------------------------------------------------------- IoU
def test_iou_f64_pairs_bit_exact(cuda, golden, po):
    from orientedreppoints_b200.dota import polyiou
    g = golden("iou_pairs.npz")
    out = polyiou.iou_poly_pairs(g["p"], g["q"])
    assert np.array_equal(out, g["ref64"], equal_nan=True)          # == compiled DOTA_devkit/polyiou.cpp
    assert polyiou.iou_poly(polyiou.VectorDouble([0, 0, 1, 0, 1, 1, 0, 1]),
                            polyiou.VectorDouble([.5, .5, 1.5, .5, 1.5, 1.5, .5, 1.5])) == 0.14285714285714285
    d = po.gen_clustered_boxes(50, 20, seed=21)
    rng = np.random.RandomState(0)
    i, j = rng.randint(0, len(d), 20000), rng.randint(0, len(d), 20000)
    assert np.array_equal(polyiou.iou_poly_pairs(d[i, :8], d[j, :8]), po.iou_poly_f64(d[i, :8], d[j, :8]),
                          equal_nan=True)


def test_quad_iou_matrix_compat32_bit_exact(cuda, golden, po):
    from orientedreppoints_b200.ops import quad_iou_matrix
    g = golden("iou_pairs.npz")
    p, q = g["p"][:400], g["q"][:400]
    m = quad_iou_matrix(_t(p, cuda), _t(q, cuda), mode="compat32").cpu().numpy()
    assert np.array_equal(np.diag(m), g["ref32"][:400], equal_nan=True)   # == compiled rnms_cpu.cpp
    # full matrix against the oracle
    pp = np.repeat(p[:64], 64, 0)
    qq = np.tile(q[:64], (64, 1))
    assert np.array_equal(m[:64, :64].reshape(-1), po.iou_rnms_f32(pp, qq), equal_nan=True)


def test_quad_iou_matrix_exact64_within_1e5(cuda, golden, po):
    from orientedreppoints_b200.ops import quad_iou_matrix
    g = golden("iou_pairs.npz")
    m = quad_iou_matrix(_t(g["p"], cuda), _t(g["q"], cuda), mode="exact64").cpu().numpy()
    d = np.diag(m).astype(np.float64)
    ok = np.isfinite(g["ref64"])
    assert np.abs(d[ok] - g["ref64"][ok]).max() < 1e-5              # north_star asks 1e-4
    # same boxes +16000: the accurate path does not care (the reference fp32 is off by up to 0.5 here)
    mf = quad_iou_matrix(_t(g["p"] + 16000, cuda), _t(g["q"] + 16000, cuda), mode="exact64").cpu().numpy()
    ref_far = po.iou_poly_f64(g["p"] + np.float32(16000), g["q"] + np.float32(16000))
    assert np.abs(np.diag(mf)[ok] - ref_far[ok]).max() < 1e-5


def test_fast_clip_error_envelope(cuda, po):
    """the fp32 clip's self-reported error bound must dominate its true error (checked through
    decisions: every exact64 decision equals the fp64 oracle's on 2M near-threshold-rich pairs)"""
    from orientedreppoints_b200.ops import quad_iou_matrix
    d = po.gen_clustered_boxes(30, 48, seed=5, jitter=2.0)[:, :8]
    m = quad_iou_matrix(_t(d, cuda), _t(d, cuda), mode="exact64").cpu().numpy().astype(np.float64)
    n = len(d)
    ref = po.iou_poly_f64_matrix(d, d)
    ok = np.isfinite(ref)
    assert np.abs(m[ok] - ref[ok]).max() < 1e-5
    assert n * n >= 2_000_000


# ------------------------------------------------------------------------------- NMS
@pytest.mark.parametrize("name", ["nms_1k.npz", "nms_clustered.npz", "nms_1k_offset16000.npz"])
def test_rnms_exact64_equals_fp64_reference(cuda, golden, name):
    from orientedreppoints_b200 import _lib
    from orientedreppoints_b200.ops import rnms, rnms_indices
    g = golden(name)
    d = _t(g["dets"], cuda)
    for thr, key in ((0.1, "keep64_thr01"), (0.3, "keep64_thr03")):
        dets_k, inds = rnms(d, thr)
        assert inds.dtype == torch.int64 and inds.device == d.device
        assert np.array_equal(inds.cpu().numpy(), np.sort(g[key]))            # ascending (rnms_kernel.cu:261-264)
        assert torch.equal(dets_k, d[inds])
        sel = rnms_indices(d, thr, order=_lib.ORP_ORDER_SCORE_DESC)
        assert np.array_equal(sel.cpu().numpy(), g[key])                      # selection order (poly_gpu_nms)


@pytest.mark.parametrize("name", ["nms_1k.npz", "nms_clustered.npz", "nms_1k_offset16000.npz"])
def test_rnms_compat32_equals_fp32_reference(cuda, golden, name):
    """bit-faithful mode reproduces rnms_cpu.cpp even where it is numerically wrong (offset 16000)"""
    from orientedreppoints_b200 import _lib
    from orientedreppoints_b200.ops import rnms_indices
    g = golden(name)
    d = _t(g["dets"], cuda)
    for thr, key in ((0.1, "keep32_thr01"), (0.4, "keep32_thr04")):
        sel = rnms_indices(d, np.float32(thr), mode="compat32", order=_lib.ORP_ORDER_SCORE_DESC)
        assert np.array_equal(sel.cpu().numpy(), g[key])


@pytest.mark.parametrize("n,seed,extent", [(5000, 1, 1024.0), (20000, 2, 1024.0), (20000, 3, 4579.0)])
def test_rnms_large_vs_oracle(cuda, po, n, seed, extent):
    from orientedreppoints_b200 import _lib
    from orientedreppoints_b200.ops import rnms_indices
    d = po.gen_rotated_boxes(n, seed=seed, extent=extent)
    ref = po.nms_poly_f64(d, 0.1, fast=True)                                  # py_cpu_nms_poly_fast semantics
    if n <= 5000:
        assert np.array_equal(ref, po.nms_poly_f64(d, 0.1))                   # == unfiltered fp64 NMS
    sel = rnms_indices(_t(d, cuda), 0.1, order=_lib.ORP_ORDER_SCORE_DESC)
    assert np.array_equal(sel.cpu().numpy(), ref)
    st = _lib.last_nms_stats()
    assert st["n"] == n and st["edges"] > 0 and st["pairs_clipped"] <= st["pairs_aabb"] <= st["pairs_total"]


def test_rnms_clustered_vs_oracle(cuda, po):
    from orientedreppoints_b200 import _lib
    from orientedreppoints_b200.ops import rnms_indices
    d = po.gen_clustered_boxes(400, 25, seed=9)
    for thr in (0.1, 0.4):
        ref = po.nms_poly_f64(d, thr, fast=True)
        sel = rnms_indices(_t(d, cuda), thr, order=_lib.ORP_ORDER_SCORE_DESC)
        assert np.array_equal(sel.cpu().numpy(), ref)


def test_rnms_segments_equal_per_class_runs(cuda, po):
    """segments == what multiclass_rnms's coordinate-offset trick means (bbox_nms.py:156-158)"""
    from orientedreppoints_b200.ops import rnms_indices
    d = po.gen_rotated_boxes(6000, seed=4, extent=700.0)
    lab = np.random.RandomState(0).randint(0, 15, len(d)).astype(np.int32)
    got = rnms_indices(_t(d, cuda), 0.4, segments=_t(lab, cuda)).cpu().numpy()
    exp = []
    for c in range(15):
        idx = np.nonzero(lab == c)[0]
        exp.append(idx[po.nms_poly_f64(d[idx], 0.4)])
    assert np.array_equal(got, np.sort(np.concatenate(exp)))


def test_rnms_edge_cases(cuda, po):
    from orientedreppoints_b200.ops import rnms
    e = torch.zeros((0, 9), device=cuda)
    dets, inds = rnms(e, 0.1)
    assert inds.numel() == 0 and inds.dtype == torch.int64 and dets.shape == (0, 9)
    with pytest.raises(TypeError, match="dets must be cuda tensor"):
        rnms(torch.zeros((3, 9)), 0.1)                                        # nms_wrapper.py:197
    with pytest.raises(TypeError):
        rnms([1, 2, 3], 0.1)
    one = _t(po.gen_rotated_boxes(1, seed=0), cuda)
    assert rnms(one, 0.1)[1].tolist() == [0]
    # identical boxes, equal scores: lower index wins (documented tie-break)
    same = one.repeat(5, 1)
    assert rnms(same, 0.1)[1].tolist() == [0]
    # ragged sizes around the warp/block boundaries
    for n in (31, 32, 33, 63, 64, 65, 255, 257):
        d = po.gen_rotated_boxes(n, seed=n, extent=200.0)
        assert np.array_equal(rnms(_t(d, cuda), 0.1)[1].cpu().numpy(), np.sort(po.nms_poly_f64(d, 0.1)))
    # non-finite rows are kept and never suppress (rnms: NaN > thr is false)
    d = po.gen_rotated_boxes(100, seed=3, extent=100.0)
    d[7, 2] = np.nan
    got = rnms(_t(d, cuda), 0.1)[1].cpu().numpy()
    assert 7 in got


def test_poly_gpu_nms_and_overlaps_host_api(cuda, golden, po):
    from orientedreppoints_b200.dota import poly_nms_gpu as pg
    g = golden("nms_1k.npz")
    keep = pg.poly_gpu_nms(g["dets"], 0.1)
    assert isinstance(keep, list) and np.array_equal(np.array(keep), g["keep64_thr01"])
    assert pg.poly_nms_gpu(np.zeros((0, 9), np.float32), 0.1) == []
    rng = np.random.RandomState(0)
    b = np.stack([rng.uniform(0, 300, 300), rng.uniform(0, 300, 300), rng.uniform(8, 64, 300),
                  rng.uniform(4, 32, 300), rng.uniform(-1.5, 1.5, 300)], 1).astype(np.float32)
    ov = pg.poly_overlaps(b[:170], b[170:])
    assert ov.shape == (170, 130) and ov.dtype == np.float32
    qa, qb = po.rotbox_to_quad_f32(b[:170]), po.rotbox_to_quad_f32(b[170:])
    ref = po.iou_poly_f64_matrix(qa, qb)
    assert np.abs(ov - ref).max() < 1e-4
    assert (ov > 0.05).sum() > 50


# ------------------------------------------------------------------------------- minarearect
def test_minarearect_vs_oracle(cuda, po):
    from orientedreppoints_b200.ops import minaerarect
    rng = np.random.RandomState(0)
    pts = rng.normal(0, 3, (21824, 18)).astype(np.float32)
    pts[:64] = np.round(pts[:64])                     # exact ties / collinear runs
    pts[64:80] = 1.0                                  # fully degenerate sets
    box_o, map_o, hn_o = po.minarearect(pts)
    box_g, map_g = minaerarect(_t(pts, cuda), return_hull_map=True)
    box_g, map_g = box_g.cpu().numpy(), map_g.cpu().numpy()
    assert np.array_equal(map_g, map_o)                                       # point-to-box index map: bit-exact
    # cos and atan2 are evaluated in double and rounded on both sides: bit-identical on every set
    assert np.array_equal(box_g.view(np.uint32), box_o.view(np.uint32)), float(np.abs(box_g - box_o).max())
    # fused affine of orientedreppoints_head.py:748-749
    ctr = rng.uniform(0, 1024, (len(pts), 2)).astype(np.float32)
    fused = minaerarect(_t(pts, cuda), scale=8.0, center=_t(ctr, cuda)).cpu().numpy()
    assert np.array_equal(fused, box_g * np.float32(8.0) + np.tile(ctr, (1, 4)))
    # reference conventions
    out = minaerarect(torch.zeros((0, 18), device=cuda))
    assert out.shape == (0, 8) and out.device.type == "cpu"                   # minarearect_cuda.cpp:7-8
    with pytest.raises(RuntimeError):
        minaerarect(torch.zeros((4, 18)))


def test_box_iou_rotated_known_answers(cuda):
    from orientedreppoints_b200.ops import box_iou_rotated
    b1 = torch.tensor([[.5, .5, 1, 1, 0]], device=cuda)
    b2 = torch.tensor([[1, 1, 1, 1, 0], [.5, .5, 1, 1, np.pi / 4]], device=cuda)
    out = box_iou_rotated(b1, b2).cpu().numpy()
    assert np.allclose(out, [[1 / 7, 0.70710678]], atol=1e-5)                 # SURVEY section 0 probe values


# ------------------------------------------------------------------------------- ResultMerge (SURVEY 8f n1)
def test_result_merge_gpu_vs_restated_reference(cuda, po, tmp_path):
    from orientedreppoints_b200.dota import result_merge as rm
    rng = np.random.RandomState(0)
    lines = []
    for img in ("P0007", "P0003", "P0011"):
        for (tx, ty) in ((0, 0), (824, 0), (0, 824), (824, 824)):
            d = po.gen_rotated_boxes(120, seed=rng.randint(1 << 30), extent=1024.0)
            for r in d:
                lines.append("%s__1__%d___%d %s %s\n" % (img, tx, ty, repr(float(r[8])), " ".join("%.1f" % v for v in r[:8])))
    rng.shuffle(lines)
    # restated mergesingle + nmsbynamedict over the CPU oracle (fp64 IoU on the float32 coordinates the GPU sees)
    names, ids, dets = rm.parse_result_lines(lines)
    exp = []
    for k, name in enumerate(names):
        idx = np.nonzero(ids == k)[0]
        keep = po.nms_poly_f64(dets[idx].astype(np.float32), 0.1, fast=True)
        for i in idx[keep]:
            exp.append(name + ' ' + str(float(dets[i, 8])) + ' ' + ' '.join(map(str, [float(v) for v in dets[i, :8]])))
    got = rm.merge_lines(lines)
    assert got == exp and len(got) > 300
    src = tmp_path / "raw"; dst = tmp_path / "merged"
    src.mkdir()
    (src / "Task1_plane.txt").write_text("".join(lines))
    rm.mergebypoly(str(src), str(dst))
    assert (dst / "Task1_plane.txt").read_text().splitlines() == exp
    assert rm.py_cpu_nms_poly(np.zeros((0, 9)), 0.1) == []
    d = po.gen_rotated_boxes(500, seed=3)
    assert rm.py_cpu_nms_poly(d.astype(np.float64), 0.3) == [int(i) for i in po.nms_poly_f64(d, 0.3)]


def test_box_iou_rotated_vs_compiled_reference(cuda, golden):
    """golden minted from the reference's box_iou_rotated_cpu.cpp (tests/golden/gen_golden_box_iou_rotated.py)"""
    from orientedreppoints_b200.ops import box_iou_rotated
    g = golden("box_iou_rotated.npz")
    out = box_iou_rotated(_t(g["b1"], cuda), _t(g["b2"], cuda)).cpu().numpy()
    assert out.shape == g["iou"].shape and out.dtype == np.float32
    assert np.abs(out - g["iou"]).max() < 1e-4            # north_star tolerance; both are fp32 centre-shifted evaluations
    assert (g["iou"] > 0.05).sum() > 100


def test_convex_iou_matches_oracle_bit_exact(cuda, po):
    """SURVEY 8 n2: orp_convex_iou (fp64 hull + fp64 clipping, float result) == the CPU oracle's sequence, bit for bit,
    through the reference-shaped python mirror (mmdet/ops/iou/iou_wrapper.py:21-30)"""
    from orientedreppoints_b200.ops import convex_iou, convex_overlaps
    rng = np.random.RandomState(3)
    n, k = 700, 40
    pts = (rng.rand(n, 9, 2) * 60 + rng.rand(n, 1, 2) * 100).astype(np.float32)
    # degenerate sets: duplicated points, collinear triples, axis-aligned grids (exact ties in the gift wrapping)
    pts[:50, 3:] = pts[:50, :1]
    pts[50:100, 2] = (pts[50:100, 0] + pts[50:100, 1]) / 2
    gx, gy = np.meshgrid(np.arange(3, dtype=np.float32), np.arange(3, dtype=np.float32))
    pts[100:150] = (np.stack([gx.ravel(), gy.ravel()], 1)[None] * 8 + rng.randint(0, 100, size=(50, 1, 2))).astype(np.float32)
    quads = po.gen_rotated_boxes(k, seed=4, extent=160.0, wmin=10, wmax=80)[:, :8].astype(np.float32)
    ref = po.convex_iou(pts.reshape(n, 18), quads)
    got = convex_iou(torch.from_numpy(pts.reshape(n, 18)).to(cuda), torch.from_numpy(quads).to(cuda))
    assert got.shape == (n, k) and got.is_cuda
    g = got.cpu().numpy()
    assert np.array_equal(g.view(np.uint32), ref.view(np.uint32)), float(np.abs(g - ref).max())
    assert torch.equal(convex_overlaps(torch.from_numpy(quads).to(cuda), torch.from_numpy(pts.reshape(n, 18)).to(cuda)), got.t())
    with pytest.raises(TypeError):
        convex_iou(torch.zeros(1, 18), torch.zeros(1, 8))
    assert convex_iou(torch.zeros(0, 18, device=cuda), torch.from_numpy(quads).to(cuda)).shape == (0, k)


def test_soft_rnms_equals_reference(cuda, golden):
    """soft_rnms (nms_wrapper.py:120-175 / rnms_cpu.cpp:165-320) against vectors minted by the reference's own compiled
    soft_rnms (tests/golden/gen_golden_soft_rnms.py): kept set, ORDER and decayed scores, for the three methods"""
    from orientedreppoints_b200.ops import soft_rnms
    g = golden("soft_rnms.npz")
    for name in ("rand600", "clustered"):
        d = g[name + "_dets"]
        for method in ("original", "linear", "gaussian"):
            for thr in (0.3, 0.5):
                ref = g["%s_%s_thr%02d" % (name, method, int(thr * 10))]
                new_dets, inds = soft_rnms(d, thr, method=method, sigma=0.5, min_score=1e-3)
                assert new_dets.dtype == d.dtype and inds.dtype == np.int64
                assert np.array_equal(inds, ref[:, 9].astype(np.int64)), (name, method, thr)
                assert np.array_equal(new_dets[:, :8], ref[:, :8])
                if method == "gaussian":                       # expf of libm vs numpy: last-bit differences allowed
                    assert np.allclose(new_dets[:, 8], ref[:, 8], rtol=2e-6, atol=0)
                else:
                    assert np.array_equal(new_dets[:, 8], ref[:, 8])
    t = torch.from_numpy(g["rand600_dets"]).to(cuda)
    nd, ind = soft_rnms(t, 0.3, method="linear")
    assert nd.is_cuda and ind.dtype == torch.long and np.array_equal(ind.cpu().numpy(), g["rand600_linear_thr03"][:, 9].astype(np.int64))
    with pytest.raises(ValueError):
        soft_rnms(g["rand600_dets"], 0.3, method="nope")
