"""Golden vectors for the FPN_CARAFE neck: the reference's OWN mmdet/models/necks/fpn_carafe.py (FPN_CARAFE), mmdet/ops/upsample.py
and mmdet/ops/carafe/carafe.py (CARAFEPack), imported FROM the reference tree with gen_golden_dense.install_stubs() and executed
on the CPU in float64.  CARAFEPack's `carafe` (a CUDA extension) is bound to the reference's own CARAFENAIVEForward kernel
compiled as host C++ (oracle/build_ref_carafe.py), run in float64.
Stored per case: the first OUT_CHANNELS channels of the five output levels (float32), and the reference neck's parameter names
and shapes, for the CPU tests' tree comparison.  Weights come from weights._draw_fpn_carafe (randomised norms and biases,
carafe_gain > 0 so that the softmax is peaked), loaded strict=True with the reference's key names; the inputs (the backbone's
stride-8, -16 and -32 outputs) are regenerated from the seeds stored here.

    python tests/golden/gen_golden_fpn_carafe.py   # needs the reference source tree; writes tests/golden/fpn_carafe_ref.npz
"""
import ctypes
import importlib
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import gen_golden_dense                                                              # noqa: E402
from fpn_carafe_ref import CASES, OUT_CHANNELS, inputs, neck_cfg, weights            # noqa: E402
from oracle import build_ref_carafe                                                   # noqa: E402


def naive_carafe_host():
    """carafe(features, masks, k, G, s) through the reference's CARAFENAIVEForward compiled as host C++, float64"""
    lib = ctypes.CDLL(build_ref_carafe.build())
    fn = lib.ref_carafe_naive_forward_f64
    fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 7 + [ctypes.c_void_p]

    def carafe(features, masks, k, group, scale):
        f, m = features.double().contiguous(), masks.double().contiguous()
        n, c, h, w = f.shape
        assert m.shape == (n, k * k * group, h * scale, w * scale)
        out = torch.zeros((n, c, h * scale, w * scale), dtype=torch.float64)
        fn(f.data_ptr(), m.data_ptr(), n, c, h, w, k, group, scale, out.data_ptr())
        return out
    return carafe


def install():
    gen_golden_dense.install_stubs()
    ref = gen_golden_dense.REF
    for name in ("carafe_cuda", "carafe_naive_cuda"):
        sys.modules["mmdet.ops.carafe." + name] = types.ModuleType(name)
    gen_golden_dense._pkg("mmdet.ops.carafe", os.path.join(ref, "mmdet", "ops", "carafe"))
    cm = importlib.import_module("mmdet.ops.carafe.carafe")                          # REAL CARAFEPack
    cm.carafe = naive_carafe_host()
    pkg = sys.modules["mmdet.ops.carafe"]
    pkg.CARAFEPack = cm.CARAFEPack
    ops = sys.modules["mmdet.ops"]
    ops.build_upsample_layer = importlib.import_module("mmdet.ops.upsample").build_upsample_layer      # REAL
    return importlib.import_module("mmdet.models.necks.fpn_carafe").FPN_CARAFE


def main():
    FPN_CARAFE = install()
    out = {}
    for case in CASES:
        sd = {k[len("neck."):]: v.double() for k, v in weights(case).items()}        # float32 draws, as the tests make them
        torch.set_default_dtype(torch.float64)
        tag = case["tag"]
        cfg = neck_cfg(case)
        cfg.pop("type")
        m = FPN_CARAFE(**cfg).double().eval()
        m.load_state_dict(sd, strict=True)
        torch.set_default_dtype(torch.float32)
        feats = inputs(case)
        unused = [torch.zeros((1, c, 1, 1)) for c in cfg["in_channels"][:cfg["start_level"]]]     # below start_level: not read
        with torch.no_grad():
            levels = m(unused + feats)
        for i, lv in enumerate(levels):
            out["%s/level%d" % (tag, i)] = lv[:, :OUT_CHANNELS].float().numpy()
        names = list(m.state_dict().keys())
        out["%s/keys" % tag] = np.array(names)
        out["%s/shapes" % tag] = np.array([",".join(str(d) for d in v.shape) for v in m.state_dict().values()])
    np.savez_compressed(os.path.join(HERE, "fpn_carafe_ref.npz"), **out)
    print("wrote", len(out), "arrays")


if __name__ == "__main__":
    main()
