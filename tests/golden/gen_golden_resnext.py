"""Golden vectors for the ResNeXt backbones: the reference's OWN mmdet/models/backbones/resnext.py (ResNeXt, its Bottleneck,
and the resnet.py it builds on), imported FROM /root/reference with gen_golden_dense.install_stubs() and executed on the CPU in
float64, loaded (strict=True: the reference's key names) with the state dict `orientedreppoints_b200.weights.random_state_dict`
draws for the same (depth, groups, base_width).  Weights are regenerated from the seeds stored here, not stored.

    python tests/golden/gen_golden_resnext.py     # needs the reference source tree; writes tests/golden/resnext_ref.npz
"""
import importlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import gen_golden_dense                                                              # noqa: E402
from orientedreppoints_b200.weights import random_state_dict                        # noqa: E402

# (tag, depth, groups, base_width, seed, residual_gain, H, W)
CASES = [("x50_32x4d", 50, 32, 4, 20, 1.0, 32, 64), ("x101_64x4d", 101, 64, 4, 21, 0.3, 32, 32),
         ("x50_32x8d", 50, 32, 8, 22, 1.0, 64, 32)]


def main():
    gen_golden_dense.install_stubs()
    ResNeXt = importlib.import_module("mmdet.models.backbones.resnext").ResNeXt
    out = {}
    for tag, depth, groups, base_width, seed, gain, h, w in CASES:
        sd = random_state_dict(depth, seed=seed, reference_init=False, residual_gain=gain, groups=groups, base_width=base_width)
        bb = {k[len("backbone."):]: v for k, v in sd.items() if k.startswith("backbone.")}
        model = ResNeXt(groups=groups, base_width=base_width, depth=depth, num_stages=4, out_indices=(0, 1, 2, 3),
                        frozen_stages=1, norm_cfg=dict(type='BN', requires_grad=True), style='pytorch')
        res = model.load_state_dict(bb, strict=True)                                  # the reference's own key names
        assert not res.missing_keys and not res.unexpected_keys
        model.double()
        model.eval()                                                                  # (ResNet.train returns None here)
        img = torch.randn(1, 3, h, w, generator=torch.Generator().manual_seed(seed + 10), dtype=torch.float64)
        with torch.no_grad():
            feats = model(img)
        out[tag + "_meta"] = np.array([depth, groups, base_width, seed, int(gain * 10), h, w], dtype=np.int64)
        out[tag + "_img"] = img.numpy()
        for l, f in enumerate(feats):
            out["%s_c%d" % (tag, l + 2)] = f.numpy().astype(np.float32)
        print(tag, [tuple(f.shape) for f in feats], [float(f.abs().max()) for f in feats])
    np.savez_compressed(os.path.join(HERE, "resnext_ref.npz"), **out)
    print("wrote resnext_ref.npz")


if __name__ == "__main__":
    main()
