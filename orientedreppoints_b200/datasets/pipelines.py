"""Test-time data pipeline of the configs (configs/dota/*.py test_pipeline) on the device.

Mirrors mmdet/datasets/pipelines/test_aug.py (MultiScaleFlipAug) and transforms.py (RotateResize / Resize with
keep_ratio, RotateRandomFlip / RandomFlip, Normalize, Pad) plus formating.py (ImageToTensor, Collect), built from the
config dicts through the registry.  The input is a device uint8 HWC batch of images sharing one shape; every view comes
out as
    img       uint8 [N, Hp, Wp, C]: resized (cv2.resize INTER_LINEAR, bit for bit), mirrored when the view flips,
              zero outside the resized extent
    valid_hw  int32 [N, 2] on the device: the resized extent (img_shape) of every image
    img_meta  list of N dicts: ori_shape, img_shape, pad_shape, scale_factor, flip, flip_direction, img_norm_cfg
Normalize is deferred into the detector's input transform (the fused uint8 stems / Swin patch gather, or
detector.normalize), which also reproduces Pad-after-Normalize: the padded region enters the network as exactly 0.0.

Resize, flip and pad are one launch of `orp_resize_u8`; its coefficient tables are computed here in float32 the way cv2
computes them and cached on the device per (source, destination) shape, so a CUDA graph can capture the launch.
What the configs do not use raises NotImplementedError naming the transform."""
import copy

import numpy as np
import torch

from .. import _lib
from ..utils.registry import Registry, build_from_cfg

PIPELINES = Registry('pipeline')
INTER_RESIZE_COEF_SCALE = 2048


# ----------------------------------------------------------------------------------------------- sizes and tables
def rescale_size(old_size, scale):
    """mmcv.rescale_size for a tuple scale: ((new_w, new_h), scale_factor).  old_size is (w, h)."""
    w, h = old_size
    if not (isinstance(scale, tuple) and len(scale) == 2):
        raise NotImplementedError("Resize: scale %r (only a (long edge, short edge) tuple is used by the configs)" % (scale,))
    sf = min(max(scale) / max(h, w), min(scale) / min(h, w))
    return (int(w * float(sf) + 0.5), int(h * float(sf) + 0.5)), sf


def resize_tables(n_src, n_dst, clamp):
    """cv2.resize INTER_LINEAR coefficients of one axis for uint8 images, int32 [n_dst, 4] = (i0, i1, w0, w1):
    f = (float)((d + 0.5) * (1 / (n_dst / n_src)) - 0.5), i = floor(f), f -= i, w = rint((1 - f, f) * 2048) in float32.
    clamp=True (columns): i < 0 -> (0, f = 0); i >= n_src - 1 -> (n_src - 1, f = 0).  clamp=False (rows): the weights keep
    f, only the two source rows are clamped into [0, n_src - 1] when read."""
    scale = 1.0 / (n_dst / n_src)
    f = ((np.arange(n_dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    i = np.floor(f).astype(np.int64)
    f = (f - i.astype(np.float32)).astype(np.float32)
    if clamp:
        lo, hi = i < 0, i >= n_src - 1
        i[lo], f[lo] = 0, 0
        i[hi], f[hi] = n_src - 1, 0
    w0 = np.rint((np.float32(1) - f) * np.float32(INTER_RESIZE_COEF_SCALE)).astype(np.int32)
    w1 = np.rint(f * np.float32(INTER_RESIZE_COEF_SCALE)).astype(np.int32)
    i0, i1 = np.clip(i, 0, n_src - 1), np.clip(i + 1, 0, n_src - 1)
    return np.stack([i0, i1, w0, w1], axis=1).astype(np.int32)


def resize_u8_numpy(img, dsize, flip=False):
    """the kernel's integer arithmetic on the host tables, in numpy: uint8 HWC img -> dsize = (w, h), then mirrored when
    flip (cv2.resize(img, dsize, interpolation=cv2.INTER_LINEAR), then [:, ::-1])"""
    h, w = img.shape[:2]
    xt, yt = resize_tables(w, dsize[0], True), resize_tables(h, dsize[1], False)
    s = img.reshape(h, w, -1).astype(np.int64)
    hor = s[:, xt[:, 0]] * xt[None, :, 2, None] + s[:, xt[:, 1]] * xt[None, :, 3, None]
    v = (((yt[:, 2, None, None] * (hor[yt[:, 0]] >> 4)) >> 16) + ((yt[:, 3, None, None] * (hor[yt[:, 1]] >> 4)) >> 16) + 2) >> 2
    out = np.clip(v, 0, 255).astype(np.uint8)
    if flip:
        out = out[:, ::-1]
    return np.ascontiguousarray(out).reshape((dsize[1], dsize[0]) + img.shape[2:])


_TABLES = {}


def device_tables(device, src_hw, dst_hw):
    """(xtab, ytab) int32 device tensors for a (src h, w) -> (dst h, w) resize, made once per shape and device (a graph
    capture reuses them)"""
    key = (str(device), tuple(src_hw), tuple(dst_hw))
    t = _TABLES.get(key)
    if t is None:
        xt = torch.from_numpy(resize_tables(src_hw[1], dst_hw[1], True)).to(device)
        yt = torch.from_numpy(resize_tables(src_hw[0], dst_hw[0], False)).to(device)
        t = _TABLES[key] = (xt, yt)
    return t


def resize_u8(img, dst_hw, pad_hw=None, flip=False, out=None):
    """device uint8 [N,H,W,C] -> [N,Hp,Wp,C]: cv2-exact bilinear resize to dst_hw, mirrored when flip, zero outside dst_hw"""
    n, h, w, c = img.shape
    hd, wd = dst_hw
    hp, wp = pad_hw if pad_hw is not None else dst_hw
    img = img.contiguous()
    if out is None:
        out = torch.empty((n, hp, wp, c), dtype=torch.uint8, device=img.device)
    assert out.shape == (n, hp, wp, c) and out.dtype == torch.uint8 and out.is_contiguous()
    xt, yt = device_tables(img.device, (h, w), (hd, wd))
    with torch.cuda.device(img.device):
        _lib.check(_lib.lib().orp_resize_u8(_lib.ptr(img), n, h, w, c, _lib.ptr(out), hd, wd, hp, wp, int(bool(flip)), _lib.ptr(xt),
                                            _lib.ptr(yt), _lib.current_stream_ptr()), "orp_resize_u8")
    return out


# ----------------------------------------------------------------------------------------------- transforms
class Compose(object):
    """mmdet/datasets/pipelines/compose.py"""

    def __init__(self, transforms):
        self.transforms = [build_from_cfg(t, PIPELINES) if isinstance(t, dict) else t for t in transforms]

    def __call__(self, data):
        for t in self.transforms:
            data = t(data)
            if data is None:
                return None
        return data


@PIPELINES.register_module
class LoadImage(object):
    """mmdet/apis/inference.py LoadImage for an image already decoded: an HWC uint8 ndarray / tensor, or a batch
    [N,H,W,C] of images sharing one shape, moved to `device` once"""

    def __init__(self, device=None):
        self.device = device

    def __call__(self, results):
        img = results['img']
        if isinstance(img, str):
            raise NotImplementedError("LoadImage: file names (decode the image first; the pipeline starts from pixels)")
        if isinstance(img, np.ndarray):
            img = torch.from_numpy(np.ascontiguousarray(img))
        if img.dtype != torch.uint8:
            raise ValueError("LoadImage: a uint8 image is expected, got %s" % img.dtype)
        if img.dim() == 2:
            img = img[:, :, None]
        results['batched'] = img.dim() == 4
        if img.dim() == 3:
            img = img[None]
        dev = self.device if self.device is not None else (img.device if img.is_cuda else torch.device("cuda", torch.cuda.current_device()))
        results['img'] = img.to(dev).contiguous()
        results['filename'] = None
        results['img_shape'] = results['ori_shape'] = tuple(img.shape[1:])
        return results


def _check_resize_args(name, img_scale, multiscale_mode, ratio_range, keep_ratio):
    if not keep_ratio:
        raise NotImplementedError("%s(keep_ratio=False): the rotated-box head needs one scale factor (a 4-vector is not supported)" % name)
    if ratio_range is not None:
        raise NotImplementedError("%s(ratio_range=%r): random ratio sampling is a training transform" % (name, ratio_range))
    if img_scale is not None:
        scales = img_scale if isinstance(img_scale, list) else [img_scale]
        assert all(isinstance(s, tuple) for s in scales)
        return scales
    return None


@PIPELINES.register_module
class RotateResize(object):
    """transforms.py:84-200 with keep_ratio=True: mmcv.imrescale(img, scale) = cv2 INTER_LINEAR to rescale_size(); the
    resize itself runs in ImageToTensor together with flip and pad (one launch)"""

    def __init__(self, img_scale=None, multiscale_mode='range', ratio_range=None, keep_ratio=True, clamp_rbbox=True):
        self.img_scale = _check_resize_args(type(self).__name__, img_scale, multiscale_mode, ratio_range, keep_ratio)
        self.multiscale_mode, self.ratio_range, self.keep_ratio = multiscale_mode, ratio_range, keep_ratio

    def __call__(self, results):
        if 'scale' not in results:
            if self.img_scale is None or len(self.img_scale) != 1:
                raise NotImplementedError("%s: random scale sampling (%s over %r) is a training transform"
                                          % (type(self).__name__, self.multiscale_mode, self.img_scale))
            results['scale'] = self.img_scale[0]
        h, w = results['img_shape'][:2]
        (nw, nh), sf = rescale_size((w, h), results['scale'])
        results['img_shape'] = results['pad_shape'] = (nh, nw) + tuple(results['img_shape'][2:])
        results['scale_factor'] = sf
        results['keep_ratio'] = True
        return results


@PIPELINES.register_module
class Resize(RotateResize):
    """transforms.py:273-440 (the axis-aligned twin; the image path is the same)"""

    def __init__(self, img_scale=None, multiscale_mode='range', ratio_range=None, keep_ratio=True):
        super().__init__(img_scale, multiscale_mode, ratio_range, keep_ratio)


@PIPELINES.register_module
class RotateRandomFlip(object):
    """transforms.py:202-270: the view's 'flip' flag (set by MultiScaleFlipAug) mirrors the resized image horizontally"""

    def __init__(self, flip_ratio=None, direction=['horizontal']):
        dirs = direction if isinstance(direction, (list, tuple)) else [direction]
        if any(d != 'horizontal' for d in dirs):
            raise NotImplementedError("%s(direction=%r): only horizontal flipping is supported" % (type(self).__name__, direction))
        self.flip_ratio, self.direction = flip_ratio, direction

    def __call__(self, results):
        if 'flip' not in results:
            if self.flip_ratio:
                raise NotImplementedError("%s(flip_ratio=%r): random flipping is a training transform" % (type(self).__name__, self.flip_ratio))
            results['flip'] = False
        if results.get('flip_direction', 'horizontal') != 'horizontal':
            raise NotImplementedError("%s: only horizontal flipping is supported" % type(self).__name__)
        results['flip_direction'] = 'horizontal'
        return results


@PIPELINES.register_module
class RandomFlip(RotateRandomFlip):
    """transforms.py:443-519"""

    def __init__(self, flip_ratio=None, direction='horizontal'):
        super().__init__(flip_ratio, direction)


@PIPELINES.register_module
class Normalize(object):
    """transforms.py:583-611: recorded in img_norm_cfg and applied inside the detector's input transform"""

    def __init__(self, mean, std, to_rgb=True):
        self.mean = np.array(mean, dtype=np.float32)
        self.std = np.array(std, dtype=np.float32)
        self.to_rgb = to_rgb

    def __call__(self, results):
        results['img_norm_cfg'] = dict(mean=self.mean, std=self.std, to_rgb=self.to_rgb)
        return results


@PIPELINES.register_module
class Pad(object):
    """transforms.py:522-580 (pad_val 0 after Normalize): only the padded shape is decided here"""

    def __init__(self, size=None, size_divisor=None, pad_val=0):
        assert size is not None or size_divisor is not None
        assert size is None or size_divisor is None
        if pad_val != 0:
            raise NotImplementedError("Pad(pad_val=%r): only zero padding is supported" % (pad_val,))
        self.size, self.size_divisor = size, size_divisor

    def __call__(self, results):
        h, w = results['img_shape'][:2]
        if self.size is not None:
            ph, pw = self.size
            assert ph >= h and pw >= w, "Pad: size %r is smaller than the image %r" % (self.size, (h, w))
        else:
            d = self.size_divisor
            ph, pw = -(-h // d) * d, -(-w // d) * d
        results['pad_shape'] = (ph, pw) + tuple(results['img_shape'][2:])
        results['pad_fixed_size'] = self.size
        results['pad_size_divisor'] = self.size_divisor
        return results


def _materialise(results):
    """resize + flip + pad of the view as one orp_resize_u8 launch (identity views are copied only when padding)"""
    if results.get('materialised'):
        return results
    img = results['img']
    n = img.shape[0]
    hd, wd = results['img_shape'][:2]
    hp, wp = results.get('pad_shape', results['img_shape'])[:2]
    flip = bool(results.get('flip', False))
    if (hd, wd) == tuple(img.shape[1:3]) and (hp, wp) == (hd, wd) and not flip:
        out = img                                              # identity view (e.g. R-50 on a 1024^2 tile): no launch
    else:
        out = resize_u8(img, (hd, wd), (hp, wp), flip)
    results['img'] = out
    results['valid_hw'] = torch.tensor([[hd, wd]] * n, dtype=torch.int32).to(img.device)
    results['materialised'] = True
    return results


@PIPELINES.register_module
class ImageToTensor(object):
    """formating.py ImageToTensor: the view's uint8 HWC batch is materialised on the device (the HWC -> CHW transpose
    and the float conversion happen inside the network's input transform)"""

    def __init__(self, keys):
        if list(keys) != ['img']:
            raise NotImplementedError("ImageToTensor(keys=%r): only 'img' is supported" % (keys,))
        self.keys = keys

    def __call__(self, results):
        return _materialise(results)


@PIPELINES.register_module
class Collect(object):
    """formating.py Collect: {'img', 'valid_hw', 'img_meta': one dict per image}"""

    def __init__(self, keys, meta_keys=('filename', 'ori_shape', 'img_shape', 'pad_shape', 'scale_factor', 'flip', 'flip_direction',
                                        'img_norm_cfg')):
        if list(keys) != ['img']:
            raise NotImplementedError("Collect(keys=%r): only 'img' is supported at test time" % (keys,))
        self.keys, self.meta_keys = keys, meta_keys

    def __call__(self, results):
        results = _materialise(results)
        meta = {k: results[k] for k in self.meta_keys if k in results}
        n = results['img'].shape[0]
        return {'img': results['img'], 'valid_hw': results['valid_hw'], 'img_meta': [copy.deepcopy(meta) for _ in range(n)]}


@PIPELINES.register_module
class MultiScaleFlipAug(object):
    """test_aug.py:8-32: one view per (scale, flip); the result is a dict of per-view lists"""

    def __init__(self, transforms, img_scale, flip=False):
        self.transforms = Compose(transforms)
        self.img_scale = img_scale if isinstance(img_scale, list) else [img_scale]
        assert all(isinstance(s, tuple) for s in self.img_scale)
        self.flip = flip

    def __call__(self, results):
        aug = []
        for scale in self.img_scale:
            for flip in ([False, True] if self.flip else [False]):
                r = results.copy()
                r['scale'], r['flip'] = scale, flip
                aug.append(self.transforms(r))
        return {k: [d[k] for d in aug] for k in aug[0]}


def build_test_pipeline(pipeline_cfg, device=None):
    """a config's test_pipeline -> Compose whose input is dict(img=<decoded uint8 image or batch>), as inference_detector
    builds it (mmdet/apis/inference.py:79: LoadImage replaces the file loader)"""
    cfgs = list(pipeline_cfg)
    if cfgs and isinstance(cfgs[0], dict) and cfgs[0].get('type') in ('LoadImageFromFile', 'LoadImage'):
        cfgs = cfgs[1:]
    return Compose([LoadImage(device)] + cfgs)


def run_test_pipeline(pipeline_cfg, img, device=None):
    """dict(img=[view], valid_hw=[view], img_meta=[view]): per view the padded uint8 batch, its valid extents and one
    meta dict per image; a pipeline without MultiScaleFlipAug gives one view"""
    data = build_test_pipeline(pipeline_cfg, device)(dict(img=img))
    if not isinstance(data['img'], list):
        data = {k: [v] for k, v in data.items()}
    return data
