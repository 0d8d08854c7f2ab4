"""Host-side mirror of mmdet/ops/box_iou_rotated (box_iou_rotated.h:20-38) over liborp_b200.so."""
import torch

from .. import _lib


def _check_rows(name, t, width):
    """the kernels read `width` floats per row: any other shape would read past the buffer"""
    if t.dim() != 2 or t.shape[1] != width:
        raise ValueError("%s: expected a [N, %d] tensor, got %s" % (name, width, list(t.shape)))


def box_iou_rotated(boxes1, boxes2):
    """boxes [N,5], [M,5] = (cx, cy, w, h, theta in radians) -> IoU [N,M] float32 (CUDA only)."""
    _check_rows("box_iou_rotated boxes1", boxes1, 5)
    _check_rows("box_iou_rotated boxes2", boxes2, 5)
    if not (boxes1.is_cuda and boxes2.is_cuda):
        raise RuntimeError("box_iou_rotated: this build has no CPU path; tensors must be CUDA")
    b1 = boxes1.float().contiguous()
    b2 = boxes2.float().contiguous()
    n, m = b1.shape[0], b2.shape[0]
    out = torch.empty((n, m), dtype=torch.float32, device=b1.device)
    if n and m:
        with torch.cuda.device(b1.device):
            rc = _lib.lib().orp_box_iou_rotated(_lib.ptr(b1), n, _lib.ptr(b2), m, _lib.ptr(out),
                                                _lib.current_stream_ptr())
        _lib.check(rc, "orp_box_iou_rotated")
    return out


def quad_iou_matrix(quads_a, quads_b, mode="exact64", union_mode=_lib.ORP_UNION_NAN_KEEPS):
    """N x K IoU of 8-coordinate quadrilaterals (the rnms/poly_nms IoU as a matrix)."""
    _check_rows("quad_iou_matrix quads_a", quads_a, 8)
    _check_rows("quad_iou_matrix quads_b", quads_b, 8)
    a = quads_a.float().contiguous()
    b = quads_b.float().contiguous()
    n, k = a.shape[0], b.shape[0]
    out = torch.empty((n, k), dtype=torch.float32, device=a.device)
    if n and k:
        m = {"exact64": _lib.ORP_NMS_EXACT64, "compat32": _lib.ORP_NMS_COMPAT32}[mode]
        with torch.cuda.device(a.device):
            rc = _lib.lib().orp_quad_iou_matrix(_lib.ptr(a), n, _lib.ptr(b), k, m, union_mode, _lib.ptr(out),
                                                _lib.current_stream_ptr())
        _lib.check(rc, "orp_quad_iou_matrix")
    return out
