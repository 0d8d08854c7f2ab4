"""GPU: rotated NMS at the sizes the hot path and BASELINE.json configs[2] name - 80 160 candidates in 15 class segments
(one 1024x1024 tile), 100 000 and 200 000 proposals - keep lists bit-exact against the CPU oracle's restatement of the
reference's py_cpu_nms_poly_fast (ResultMerge_multi_process.py:60-121; pinned to the reference's compiled polyiou).
These run `orp_rnms` through rnms_indices, not poly_gpu_nms: the unsegmented 100k / 200k sets are cut into y strips, the
tile-load case (segments without a known bound) is not.  tests/test_nms_plans_gpu.py covers poly_gpu_nms and the other plans."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _run(cuda, d, thr, segments=None):
    from orientedreppoints_b200 import _lib
    from orientedreppoints_b200.ops import rnms_indices
    seg = None if segments is None else torch.from_numpy(segments).to(cuda)
    sel = rnms_indices(torch.from_numpy(d).to(cuda), thr, segments=seg, union_mode=_lib.ORP_UNION_NAN_SUPPRESSES,
                       order=_lib.ORP_ORDER_SCORE_DESC)
    torch.cuda.synchronize()
    return sel.cpu().numpy(), _lib.last_nms_stats()


@pytest.mark.parametrize("n,dense", [(100000, True), (100000, False), (200000, True)])
def test_nms_sweep_sizes_bit_exact(cuda, po, n, dense):
    from orientedreppoints_b200.synth import const_density_extent, gen_rotated_boxes
    d = gen_rotated_boxes(n, seed=7, extent=1024.0 if dense else const_density_extent(n))
    got, st = _run(cuda, d, 0.1)
    ref = po.nms_poly_f64(d, 0.1, fast=True)
    print("n=%d dense=%s kept=%d stats=%s" % (n, dense, len(ref), st))
    assert st["overflow"] == 0
    assert np.array_equal(got, ref)                          # indices AND order
    # the lazy evaluation clips only against kept boxes
    assert st["pairs_clipped"] <= st["edges"]


def test_nms_tile_load_segments_bit_exact(cuda, po):
    """the tile's real load: 15 classes x 5344 candidates, suppression only inside a class"""
    from orientedreppoints_b200.synth import gen_rotated_boxes
    parts, segs = [], []
    for c in range(15):
        parts.append(gen_rotated_boxes(5344, seed=100 + c, extent=1024.0))
        segs.append(np.full(5344, c, np.int32))
    d = np.concatenate(parts)
    # interleave the classes so that segments are not contiguous in the input (as multiclass_rnms feeds them)
    perm = np.random.RandomState(0).permutation(d.shape[0])
    d, seg = d[perm], np.concatenate(segs)[perm]
    # scores must stay unique across the whole set for an order-exact comparison
    d[:, 8] = (np.argsort(np.argsort(d[:, 8])) + 1).astype(np.float32) / np.float32(d.shape[0] + 1)
    got, st = _run(cuda, d, 0.4, segments=seg)
    keep = []
    for c in range(15):
        ids = np.nonzero(seg == c)[0]
        keep.append(ids[po.nms_poly_f64(d[ids], 0.4, fast=True)])
    ref = np.concatenate(keep)
    ref = ref[np.argsort(-d[ref, 8], kind="stable")]
    print("tile load: kept=%d stats=%s" % (len(ref), st))
    assert st["overflow"] == 0
    assert np.array_equal(got, ref)
