"""mmdet/apis/inference.py:16-87: init_detector / inference_detector.

    model = init_detector('configs/dota/orientedrepoints_r101_demo.py', 'epoch_40.pth', device='cuda:0')
    result = inference_detector(model, img)      # img: decoded uint8 HWC (BGR, as cv2 reads it)

`inference_detector` runs the config's test pipeline (data.test.pipeline, LoadImage in place of the file loader) on the
device (datasets/pipelines.py), then the detector with rescale=True: one view -> simple_test, several (MultiScaleFlipAug
with several scales or flip) -> aug_test.  Detections come back in the coordinates of the input image."""
import importlib.util
import os
import types

import numpy as np
import torch

from .datasets.pipelines import run_test_pipeline
from .models import build_detector


class Config(dict):
    """the module-level names of a config file as a dict with attribute access (the mmcv.Config surface this needs)"""

    def __getattr__(self, k):
        try:
            v = self[k]
        except KeyError:
            raise AttributeError(k)
        return Config(v) if isinstance(v, dict) and not isinstance(v, Config) else v

    @classmethod
    def fromfile(cls, path):
        spec = importlib.util.spec_from_file_location("_orp_cfg_%s" % os.path.basename(path).replace(".", "_"), path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return cls.from_module(mod)

    @classmethod
    def from_module(cls, mod):
        return cls({k: v for k, v in vars(mod).items() if not k.startswith("_") and not isinstance(v, types.ModuleType)})


def init_detector(config, checkpoint=None, device='cuda:0', precision='f16x3'):
    """config: a config file path, a Config / dict, or a config module.  checkpoint: a .pth file holding the reference's
    state_dict (or {'state_dict': ...}); None keeps the reference's initialisation."""
    if isinstance(config, str):
        config = Config.fromfile(config)
    elif isinstance(config, types.ModuleType):
        config = Config.from_module(config)
    elif isinstance(config, dict):
        config = Config(config)
    else:
        raise TypeError('config must be a filename, a dict or a config module, but got {}'.format(type(config)))
    model_cfg = dict(config['model'], pretrained=None, precision=precision)
    model = build_detector(model_cfg, test_cfg=config.get('test_cfg'))
    if checkpoint is not None:
        ck = torch.load(checkpoint, map_location='cpu')
        sd = ck.get('state_dict', ck) if isinstance(ck, dict) else ck
        model.load_state_dict(sd, strict=True)
        meta = ck.get('meta', {}) if isinstance(ck, dict) else {}
        if 'CLASSES' in meta:
            model.CLASSES = meta['CLASSES']
    model.cfg = config
    model.eval()
    eng = model.engine(torch.device(device))
    if 'img_norm_cfg' in config:
        c = config['img_norm_cfg']
        eng.img_norm_cfg = dict(mean=list(c['mean']), std=list(c['std']), to_rgb=c.get('to_rgb', True))
    return model


def _engine_of(model):
    return model.engine() if hasattr(model, 'engine') else model


def inference_detector(model, img):
    """img: a decoded uint8 HWC image (ndarray or tensor), or a batch [N,H,W,C] of images sharing one shape.  Returns
    rbbox2result lists (15 arrays [k, 9] of 8 corner coordinates + score, input-image coordinates) for one image, a list
    of them for a batch."""
    cfg = model.cfg
    eng = _engine_of(model)
    batched = (img.ndim if isinstance(img, np.ndarray) else img.dim()) == 4
    data = run_test_pipeline(cfg['data']['test']['pipeline'], img, device=eng.device)
    views, metas, valids = data['img'], data['img_meta'], data['valid_hw']
    norm = metas[0][0].get('img_norm_cfg')
    if norm is not None:
        eng.img_norm_cfg = dict(mean=[float(v) for v in norm['mean']], std=[float(v) for v in norm['std']], to_rgb=bool(norm['to_rgb']))
    with torch.no_grad():
        if len(views) == 1:
            results = eng.simple_test(views[0], metas[0], rescale=True, valid_hw=valids[0])
        else:
            n = views[0].shape[0]
            results = [eng.aug_test([v[i:i + 1] for v in views], [[m[i]] for m in metas], rescale=True,
                                    valid_hws=[v[i:i + 1] for v in valids]) for i in range(n)]
    return results if batched else results[0]
