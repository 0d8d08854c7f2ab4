"""Golden vectors for the HRNet backbones and the HRFPN neck: the reference's OWN mmdet/models/backbones/hrnet.py (with the
resnet.py blocks it imports) and necks/hrfpn.py, imported FROM the reference tree with gen_golden_dense.install_stubs() (plus
mmcv.cnn.caffe2_xavier_init, which hrfpn.py imports) and executed on the CPU in float64, loaded (strict=True: the reference's
key names) with the state dicts `orientedreppoints_b200.weights.random_hrnet_state_dict` draws.  Weights are regenerated
from the seeds stored here, not stored, and so are the inputs (numpy's RandomState, whose streams do not change).  HRFPN has
64 output channels here, which keeps the file small; the restatement it pins reads the width from the weights.  The file also
holds the parameter keys of HRNet + HRFPN(256) for every published width: the four share one key list, stored once, with one
shape list per width.

    python tests/golden/gen_golden_hrnet.py     # needs the reference source tree; writes hrnet_ref.npz
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
from orientedreppoints_b200.hrnet import ARCHS                                      # noqa: E402
from orientedreppoints_b200.weights import random_hrnet_state_dict                  # noqa: E402

FEAT = 64
# (tag, arch, seed, residual_gain, H, W); 96 x 96 gives a 24 x 24 reduced map: partial windows at pool 16 (and 8 is exact)
CASES = [("w18_64x128", "hrnetv2p_w18", 30, 0.3, 64, 128), ("w32_64x64", "hrnetv2p_w32", 31, 0.3, 64, 64),
         ("w18_96x96", "hrnetv2p_w18", 32, 0.3, 96, 96)]


def main():
    gen_golden_dense.install_stubs()
    sys.modules["mmcv.cnn"].caffe2_xavier_init = lambda *a, **k: None
    HRNet = importlib.import_module("mmdet.models.backbones.hrnet").HRNet
    HRFPN = importlib.import_module("mmdet.models.necks.hrfpn").HRFPN
    out = {}
    for name, arch in ARCHS.items():
        for part, m in (("backbone", HRNet(arch.extra())), ("neck", HRFPN(list(arch.out_widths), 256, stride=2))):
            sd = m.state_dict()
            keys = "\n".join(sd)
            assert out.setdefault("keys_" + part, np.array(keys)) == keys      # one key list for every width
            out["%s_shapes_%s" % (name, part)] = np.array(";".join(",".join(map(str, v.shape)) for v in sd.values()))
    for tag, arch, seed, gain, h, w in CASES:
        sd = random_hrnet_state_dict(arch, seed=seed, reference_init=False, residual_gain=gain, feat=FEAT)
        bb = HRNet(ARCHS[arch].extra())
        res = bb.load_state_dict({k[len("backbone."):]: v for k, v in sd.items() if k.startswith("backbone.")}, strict=False)
        assert not res.missing_keys and all(k.endswith("num_batches_tracked") for k in res.unexpected_keys), res
        bb.double().eval()
        img = torch.from_numpy(np.random.RandomState(seed + 10).standard_normal((1, 3, h, w)))
        with torch.no_grad():
            feats = bb(img)
        out[tag + "_meta"] = np.array([seed, int(round(gain * 10)), h, w], dtype=np.int64)
        out[tag + "_arch"] = np.array(arch)
        for l, f in enumerate(feats):
            out["%s_y%d" % (tag, l)] = f.numpy().astype(np.float32)
        for pooling in ("AVG", "MAX"):
            nk = HRFPN(list(ARCHS[arch].out_widths), FEAT, pooling_type=pooling, stride=2)
            nk.load_state_dict({k[len("neck."):]: v for k, v in sd.items() if k.startswith("neck.")}, strict=True)
            nk.double().eval()
            with torch.no_grad():
                levels = nk([f.clone() for f in feats])
            for l, f in enumerate(levels):
                if l > 0 or pooling == "AVG":                                   # level 0 is not pooled
                    out["%s_%sp%d" % (tag, pooling + "_" if l else "", l)] = f.numpy().astype(np.float32)
        print(tag, [tuple(f.shape) for f in feats], [float(f.abs().max()) for f in feats], [tuple(f.shape) for f in levels])
    np.savez_compressed(os.path.join(HERE, "hrnet_ref.npz"), **out)
    print("wrote hrnet_ref.npz")


if __name__ == "__main__":
    main()
