"""poly2rbox_single_v3 (DOTA_devkit/dota_poly2rbox.py:128-190), the quad -> rotated box conversion of the mAOE, on the
device (orp_poly2rbox_v3).

    poly2rbox_v3(quads)            [n, 8] -> fp64 [n, 5] (x_ctr, y_ctr, w, h, angle) on the GPU, one call
    poly2rbox_single_v3(poly)      the reference's 5-tuple of Python floats for one quad

The arithmetic is the reference's: float32 edges and ratio, angles in [-pi/4, 3pi/4) from the float32 differences
widened to double.  Centres and sizes are numpy's bits; angles come from CUDA's atan2 (within 2 ulp of numpy's), with
numpy's branch decisions except where |angle1| and |angle2| are within ~45 ulp: there the exact angles decide
(DESIGN.md section 2, deviation 11).
"""
import numpy as np
import torch

from .. import _lib


def poly2rbox_v3(quads, device=None):
    """rotated boxes of quads [n, 8] (torch tensor or array-like; x1 y1 ... x4 y4) -> fp64 tensor [n, 5] on the device
    of `quads` when it is a CUDA tensor, else on `device` (default: the current CUDA device)"""
    if isinstance(quads, torch.Tensor) and quads.is_cuda:
        dev = quads.device
    else:
        dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    q = torch.as_tensor(np.asarray(quads) if not isinstance(quads, torch.Tensor) else quads)
    q = q.to(device=dev, dtype=torch.float64).reshape(-1, 8).contiguous()
    out = torch.empty((q.shape[0], 5), dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        rc = _lib.lib().orp_poly2rbox_v3(_lib.ptr(q), int(q.shape[0]), _lib.ptr(out), _lib.current_stream_ptr())
    _lib.check(rc, "orp_poly2rbox_v3")
    return out


def poly2rbox_single_v3(poly):
    """(x_ctr, y_ctr, w, h, angle) of one quad [x1, y1, ..., x4, y4], as the reference returns it"""
    return tuple(float(v) for v in poly2rbox_v3(np.asarray(poly, np.float64)[:8]).cpu().numpy()[0])
