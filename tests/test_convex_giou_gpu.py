"""GPU: orp_convex_giou (csrc/convex_iou.cu), ops.convex_giou and the GIoULoss of losses.py.

- The C entry point equals the reference's own devrIoU (tests/golden/convex_giou_ref.npz) bit for bit, all 19 floats, NaN
  where NaN, at launch sizes around a warp and past the grid-stride cap, with inputs at a non-zero storage offset, into
  outputs pre-filled with two NaN patterns inside guard regions (_twice of test_geometry_ops_gpu.py).
- The loss and pred.grad equal a plain torch restatement of mmdet/models/losses/iou_loss.py:69-128 applied to the golden's
  (giou, grad) bit for bit, for every reduction, weight kind and loss_weight; the loss's forward makes no host sync."""
import os

import numpy as np
import pytest
import torch

from orientedreppoints_b200 import _lib

from test_geometry_ops_gpu import _same, _stream, _t, _twice

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def g():
    d = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "convex_giou_ref.npz"))
    return {k: d[k] for k in d}


def _giou(dev, pts, quads):
    n = len(pts)
    L = _lib.lib()
    # inputs at a non-zero storage offset
    x = _t(np.concatenate([np.zeros((1, 18), np.float32), pts]), dev)[1:]
    y = _t(np.concatenate([np.zeros((3, 8), np.float32), quads]), dev)[3:]
    assert x.storage_offset() > 0 and y.storage_offset() > 0
    return _twice(dev, [((n, 19), torch.float32)],
                  lambda o: L.orp_convex_giou(_lib.ptr(x), _lib.ptr(y), n, _lib.ptr(o), _stream()), "orp_convex_giou")[0]


def test_convex_giou_reference_bits(cuda, g):
    got = _giou(cuda, g["pts"], g["quads"])
    bad = ~np.all((got.view(np.int32) == g["out"].view(np.int32)) | (np.isnan(got) & np.isnan(g["out"])), 1)
    assert not bad.any(), "%d rows differ, kinds %s" % (bad.sum(), sorted(set(g["kind"][bad].tolist())))


@pytest.mark.parametrize("n", [1, 31, 32, 33, 65])
def test_convex_giou_launch_sizes(cuda, g, n):
    idx = np.random.RandomState(n).permutation(len(g["pts"]))[:n]
    assert _same(_giou(cuda, g["pts"][idx], g["quads"][idx]), g["out"][idx])


def test_convex_giou_past_the_grid_cap(cuda, g):
    """the launch is capped at 132 SMs x 32 blocks x 128 threads; every row past it comes from the grid-stride loop"""
    n = 132 * 32 * 128 + 1000
    idx = np.arange(n) % len(g["pts"])
    assert _same(_giou(cuda, g["pts"][idx], g["quads"][idx]), g["out"][idx])


def test_convex_giou_nonfinite_rows(cuda, g):
    """the reference never returns on NaN input; the device writes a NaN row for any non-finite coordinate"""
    pts, quads = g["pts"][:8].copy(), g["quads"][:8].copy()
    pts[0, 3] = np.nan
    pts[1, 0] = np.inf
    quads[2, 7] = -np.inf
    quads[3, 0] = np.nan
    got = _giou(cuda, pts, quads)
    assert np.isnan(got[:4]).all()
    assert _same(got[4:], g["out"][4:8])


def test_errors_and_empty_launches(cuda):
    L = _lib.lib()
    buf = torch.zeros(64, device=cuda)
    p, s = _lib.ptr(buf), _stream()
    assert L.orp_convex_giou(p, p, -1, p, s) == -1
    for args in [(None, p, 1, p), (p, None, 1, p), (p, p, 1, None)]:
        assert L.orp_convex_giou(*args, s) == -1
    _lib.reset_launch_count()
    assert L.orp_convex_giou(None, None, 0, None, s) == 0
    assert _lib.launch_count() == 0
    from orientedreppoints_b200.ops import convex_giou
    gi, gr = convex_giou(torch.zeros(0, 18, device=cuda), torch.zeros(0, 8, device=cuda))
    assert gi.shape == (0,) and gr.shape == (0, 18) and gi.device == cuda and gr.device == cuda
    assert _lib.launch_count() == 0


def test_python_op_returns_views_of_the_rows(cuda, g):
    from orientedreppoints_b200.ops import convex_giou
    pts = torch.from_numpy(g["pts"][:300]).to(cuda)
    quads = torch.from_numpy(g["quads"][:300]).to(cuda)
    gi, gr = convex_giou(pts, quads)
    assert gi.shape == (300,) and gr.shape == (300, 18) and gi.dtype == gr.dtype == torch.float32
    assert gi.data_ptr() == gr.data_ptr() + 18 * 4 and gr.stride() == (19, 1) and gi.stride() == (19,)
    assert _same(gr.cpu().numpy(), g["out"][:300, :18]) and _same(gi.cpu().numpy(), g["out"][:300, 18])


def _restated(pred, giou, grad, weight, reduction, loss_weight):
    """iou_loss.py:69-128 in plain torch on given (giou, grad): GIoULossFuction.forward, its stored gradient and the
    second loss_weight of GIoULoss.forward"""
    if weight is not None and not torch.any(weight > 0):
        return (pred * weight.unsqueeze(-1)).sum(), None
    loss = 1 - giou
    if weight is not None:
        loss = loss * weight
        grad = grad * weight.reshape(-1, 1)
    if reduction == 'sum':
        loss = loss.sum()
    elif reduction == 'mean':
        loss = loss.mean()
    grad = grad.clone()
    unvaild_inds = torch.nonzero((grad > 1).sum(1))[:, 0]
    grad[unvaild_inds] = 1e-6
    return loss_weight * loss, -grad / grad.size(0) * loss_weight


@pytest.mark.parametrize("loss_weight", [0.375, 1.0])
@pytest.mark.parametrize("wkind", ["none", "positive", "zero", "large"])
@pytest.mark.parametrize("reduction", ["none", "mean", "sum"])
def test_giou_loss_matches_the_reference_function(cuda, g, reduction, wkind, loss_weight):
    from orientedreppoints_b200.losses import GIoULoss
    sel = np.isin(g["kind"], ("realistic", "disjoint", "contains", "inside")) & np.isfinite(g["out"]).all(1)
    n = 777
    pts, quads, out = g["pts"][sel][:n], g["quads"][sel][:n], g["out"][sel][:n]
    gen = torch.Generator().manual_seed(n)
    weight = {"none": None, "positive": torch.rand(n, generator=gen) + 0.05, "zero": torch.zeros(n),
              "large": torch.rand(n, generator=gen) * 4e4}[wkind]
    weight = None if weight is None else weight.to(cuda)
    pred = torch.from_numpy(pts).to(cuda).requires_grad_(True)
    target = torch.from_numpy(quads).to(cuda)
    o = torch.from_numpy(out).to(cuda)
    exp_loss, exp_grad = _restated(pred.detach(), o[:, 18], o[:, :18], weight, reduction, loss_weight)
    if wkind == "large":
        assert bool(((o[:, :18] * weight[:, None]) > 1).any(1).any()), "the > 1 row filter does not fire"
    loss = GIoULoss(reduction=reduction, loss_weight=loss_weight)(pred, target, weight, avg_factor=123.0)
    assert loss.dtype == exp_loss.dtype and loss.shape == exp_loss.shape
    assert torch.equal(loss.detach().view(torch.int32), exp_loss.view(torch.int32))
    # backward ignores the incoming gradient: any upstream scale gives the stored gradient
    (loss.sum() * 3.0).backward()
    if exp_grad is None:
        assert torch.equal(pred.grad, torch.zeros_like(pred))
    else:
        assert torch.equal(pred.grad.view(torch.int32), exp_grad.view(torch.int32))


def test_giou_loss_function_makes_no_host_sync(cuda, g):
    from orientedreppoints_b200.losses import convex_giou_loss
    pred = torch.from_numpy(g["pts"][:512]).to(cuda)
    target = torch.from_numpy(g["quads"][:512]).to(cuda)
    weight = torch.rand(512, device=cuda) * 10
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = convex_giou_loss(pred, target, weight, "mean", None, 0.375)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert loss.shape == () and bool(torch.isfinite(loss))
