"""OrientedRepPointsDetector inference (simple_test path) over liborp_b200.so.

Mirrors mmdet/models/detectors/orientedreppoints_detector.py:37-46:
    x = extract_feat(img)            # single_stage.py:44-50: backbone -> neck
    outs = bbox_head(x)              # orientedreppoints_head.py:173: forward_single per level
    bbox_list = bbox_head.get_bboxes(*outs, img_meta, test_cfg, rescale)
    rbbox2result(...)                # core/bbox/transforms.py:356-375

Host code is Python; every layer is a kernel of this repository called through the C ABI
(include/orp_b200.h) on torch-owned device memory and the current torch stream.  Activations are NHWC.
Three arithmetic engines: 'f16x3' (wgmma tensor cores on fp16 hi/lo operand pairs, three MMAs per product,
fp32 accumulation - fp32-faithful, the parity AND benchmark arithmetic), 'bf16' (wgmma, single-pass bf16
operands - 3x the rate, ~1e-2 accuracy) and 'fp32' (CUDA-core FMAs).  There is no PyTorch/cuDNN fallback for any layer.
"""
import numpy as np
import torch

from . import _lib
from .weights import STAGE_BLOCKS, fold_bn

STRIDES = (8, 16, 32, 64, 128)


class ConvLayer:
    """weights of one convolution in kernel layout [Cout, KH, KW, Cin] (+ optional bias)"""

    def __init__(self, w_nchw, bias, stride, pad, device, pad_cin_to=None):
        w = w_nchw.permute(0, 2, 3, 1).contiguous()                   # [Cout, KH, KW, Cin]
        self.w_raw = w.float().cpu()                                  # unpadded, for the tensor-core operand prep
        if pad_cin_to is not None and w.shape[3] < pad_cin_to:
            w = torch.cat([w, w.new_zeros(*w.shape[:3], pad_cin_to - w.shape[3])], 3).contiguous()
        self.cout, self.kh, self.kw, self.cin = w.shape
        self.w = w.to(device=device, dtype=torch.float32).contiguous()
        self.bias = None if bias is None else bias.to(device=device, dtype=torch.float32).contiguous()
        self.stride, self.pad = stride, pad
        self.tc = None    # tensor-core operand cache (dense_tc), filled lazily by the bf16 engine


class Norm:
    def __init__(self, sd, prefix, device):
        self.gamma = sd[prefix + ".weight"].to(device=device, dtype=torch.float32).contiguous()
        self.beta = sd[prefix + ".bias"].to(device=device, dtype=torch.float32).contiguous()


class EngineF32:
    """fp32 CUDA-core kernels (csrc/dense_f32.cu)"""
    name = "fp32"
    act_dtype = torch.float32

    def __init__(self, device):
        self.device = device
        self.lib = _lib.lib()

    def prepare_input(self, img_nchw):
        n, c, h, w = img_nchw.shape
        x = torch.zeros((n, h, w, 4), dtype=torch.float32, device=self.device)
        x[..., :c] = img_nchw.to(self.device, torch.float32).permute(0, 2, 3, 1)
        return x

    def conv(self, x, L, relu=False, residual=None, want_stats=False, out_f32=False):
        """out_f32: accepted for the tensor-core engines' interface; every output of this engine is fp32"""
        n, h, w, cin = x.shape
        assert cin == L.cin, (cin, L.cin)
        ho = (h + 2 * L.pad - L.kh) // L.stride + 1
        wo = (w + 2 * L.pad - L.kw) // L.stride + 1
        y = torch.empty((n, ho, wo, L.cout), dtype=torch.float32, device=self.device)
        stats = torch.zeros((n, 32, 2), dtype=torch.float64, device=self.device) if want_stats else None
        rc = self.lib.orp_conv2d_f32(_lib.ptr(x), n, h, w, cin, _lib.ptr(L.w), L.cout, L.kh, L.kw, L.stride, L.pad,
                                     _lib.ptr(L.bias), _lib.ptr(residual), int(relu), _lib.ptr(y), _lib.ptr(stats), 32,
                                     _lib.current_stream_ptr())
        _lib.check(rc, "orp_conv2d_f32")
        return (y, stats) if want_stats else y

    def gn(self, x, stats, norm, relu=False, up=None):
        n, h, w, c = x.shape
        y = torch.empty_like(x)
        rc = self.lib.orp_gn_apply_f32(_lib.ptr(x), n, h, w, c, _lib.ptr(stats), 32, _lib.ptr(norm.gamma),
                                       _lib.ptr(norm.beta), 1e-5, int(relu), _lib.ptr(up), _lib.ptr(y),
                                       _lib.current_stream_ptr())
        _lib.check(rc, "orp_gn_apply_f32")
        return y

    def conv_gn(self, x, L, norm, relu=False, up=None):
        y, st = self.conv(x, L, want_stats=True)
        return self.gn(y, st, norm, relu=relu, up=up)

    # multi-level forms (the head's weights are shared by the five FPN levels)
    def conv_multi(self, xs, L, relu=False, residual=None, out_f32=False, residual_f32=None):
        res = residual if residual is not None else residual_f32
        return [self.conv(x, L, relu=relu, residual=None if res is None else res[i]) for i, x in enumerate(xs)]

    def conv_gn_multi(self, xs, L, norm, relu=False):
        return [self.conv_gn(x, L, norm, relu=relu) for x in xs]

    def deform_conv_multi(self, xs, offsets, L, relu=False):
        return [self.deform_conv(x, o, L, relu=relu) for x, o in zip(xs, offsets)]

    def stem(self, x, L):
        return self.conv(x, L, relu=True)

    def maxpool(self, x):
        n, h, w, c = x.shape
        ho, wo = (h + 2 - 3) // 2 + 1, (w + 2 - 3) // 2 + 1
        y = torch.empty((n, ho, wo, c), dtype=torch.float32, device=self.device)
        rc = self.lib.orp_maxpool3x3s2_f32(_lib.ptr(x), n, h, w, c, _lib.ptr(y), _lib.current_stream_ptr())
        _lib.check(rc, "orp_maxpool3x3s2_f32")
        return y

    def deform_conv(self, x, offset, L, relu=False, mask=None):
        n, h, w, cin = x.shape
        ho, wo = (h + 2 * L.pad - L.kh) // L.stride + 1, (w + 2 * L.pad - L.kw) // L.stride + 1
        y = torch.empty((n, ho, wo, L.cout), dtype=torch.float32, device=self.device)
        rc = self.lib.orp_deform_conv2d_f32(_lib.ptr(x), n, h, w, cin, _lib.ptr(offset), _lib.ptr(mask), _lib.ptr(L.w),
                                            L.cout, L.kh, L.kw, L.stride, L.pad, 1, _lib.ptr(L.bias), int(relu),
                                            _lib.ptr(y), _lib.current_stream_ptr())
        _lib.check(rc, "orp_deform_conv2d_f32")
        return y


class OrientedRepPointsDetector:
    """R-50 / R-101 or Swin-T/S/B/L + FPN(GN) + OrientedRepPointsHead, inference only."""

    def __init__(self, state_dict, depth=50, device="cuda", precision="fp32", test_cfg=None, dcn=None):
        """depth: 50 / 101 (ResNet), or a Swin backbone - "swin_tiny" (Swin-T, window 7), any key of swin.ARCHS
        ("swin_small", "swin_base_w12", ...) or a swin.SwinArch.
        dcn: the ResNet's deformable conv2 layers per stage and block, None / 'DCN' / 'DCNv2' (models.ResNet.dcn_layout,
        weights.dcn_layout); None: every conv2 is a plain convolution"""
        from .swin import arch_of
        self.device = torch.device(device)
        if self.device.type == "cuda" and self.device.index is None:      # 'cuda' -> the current device, with its index
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.depth = depth
        self.swin_arch = arch_of(depth)                    # None for a ResNet
        self.dcn = dcn
        self.test_cfg = dict(nms_pre=2000, min_bbox_size=0, score_thr=0.05, nms=dict(type='rnms', iou_thr=0.4),
                             max_per_img=2000)                         # configs/dota/orientedrepoints_r50_demo.py:62-67
        if test_cfg:
            self.test_cfg.update(test_cfg)
        # configs/dota/orientedrepoints_r50_demo.py:72-73; used when simple_test() is given decoded uint8 HWC tiles
        self.img_norm_cfg = dict(mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375], to_rgb=True)
        if precision == "fp32":
            self.eng = EngineF32(self.device)
        elif precision == "bf16":
            from .engine_tc import EngineTC
            self.eng = EngineTC(self.device)
        elif precision == "f16x3":
            from .engine_tc import EngineTCSplit
            self.eng = EngineTCSplit(self.device)
        else:
            raise ValueError("precision must be 'f16x3' (tensor cores, fp32-faithful), 'bf16' (tensor cores) or 'fp32' (CUDA cores)")
        self._load(state_dict)
        base = np.arange(-1, 2).astype(np.float64)
        off = np.stack([np.repeat(base, 3), np.tile(base, 3)], axis=1).reshape(-1)        # head :78-88 (dy,dx)
        self.dcn_base_offset = torch.tensor(off, dtype=torch.float32, device=self.device).view(1, 1, 1, 18)
        import ctypes
        self._dcn_base_host = (ctypes.c_float * 18)(*[float(v) for v in off])

    # ------------------------------------------------------------------ weights
    def _load(self, sd):
        d = self.device
        if self.swin_arch is not None:
            if self.dcn is not None:
                raise ValueError("dcn describes the deformable layers of a ResNet backbone; the Swin backbone has none")
            return self._load_swin(sd)

        def folded(conv, bn, stride, pad, pad_cin_to=None):
            w, b = fold_bn(sd[conv + ".weight"].float(), sd[bn + ".weight"].float(), sd[bn + ".bias"].float(),
                           sd[bn + ".running_mean"].float(), sd[bn + ".running_var"].float())
            return ConvLayer(w, b, stride, pad, d, pad_cin_to)

        layout = self.dcn if self.dcn is not None else tuple((None,) * n for n in STAGE_BLOCKS[self.depth])
        if tuple(len(s) for s in layout) != STAGE_BLOCKS[self.depth] or \
                any(k not in (None, 'DCN', 'DCNv2') for s in layout for k in s):
            raise ValueError("dcn must give None, 'DCN' or 'DCNv2' for each of the %s blocks of R-%d" % (STAGE_BLOCKS[self.depth], self.depth))
        self.stem = folded("backbone.conv1", "backbone.bn1", 2, 3, pad_cin_to=4)
        self.blocks = []
        for li, nblk in enumerate(STAGE_BLOCKS[self.depth]):
            stage = []
            for b in range(nblk):
                p = "backbone.layer%d.%d" % (li + 1, b)
                s = 2 if (b == 0 and li > 0) else 1
                blk = dict(c1=folded(p + ".conv1", p + ".bn1", 1, 0), c2=folded(p + ".conv2", p + ".bn2", s, 1),
                           c3=folded(p + ".conv3", p + ".bn3", 1, 0),
                           ds=folded(p + ".downsample.0", p + ".downsample.1", s, 0) if b == 0 else None)
                blk["dcn"] = layout[li][b]
                blk["off"] = self._offset_conv(sd, p + ".conv2", blk["dcn"], 64 << li, s)
                stage.append(blk)
            self.blocks.append(stage)
        self.lat = [(ConvLayer(sd["neck.lateral_convs.%d.conv.weight" % i].float(), None, 1, 0, d),
                     Norm(sd, "neck.lateral_convs.%d.gn" % i, d)) for i in range(3)]
        self.fpn = [(ConvLayer(sd["neck.fpn_convs.%d.conv.weight" % i].float(), None, 2 if i >= 3 else 1, 1, d),
                     Norm(sd, "neck.fpn_convs.%d.gn" % i, d)) for i in range(5)]
        self._load_head(sd)

    def _offset_conv(self, sd, conv2, kind, planes, stride):
        """the conv_offset of a deformable conv2 (deform_conv.py:258-323, 377-446): a plain 3x3 convolution with bias into
        2 * 9 (DCN) or 3 * 9 (DCNv2) channels; None for a plain conv2.  The state dict must hold exactly the layers `kind`
        names, in their shapes"""
        has = conv2 + ".conv_offset.weight" in sd
        if kind is None:
            if has:
                raise ValueError("%s has a conv_offset but dcn names a plain convolution there" % conv2)
            return None
        co = 27 if kind == 'DCNv2' else 18
        if not has or tuple(sd[conv2 + ".conv_offset.weight"].shape) != (co, planes, 3, 3) or \
                tuple(sd[conv2 + ".conv_offset.bias"].shape) != (co,) or tuple(sd[conv2 + ".weight"].shape) != (planes, planes, 3, 3):
            raise ValueError("%s is %s: it needs weight [%d,%d,3,3] and conv_offset weight [%d,%d,3,3] / bias [%d]"
                             % (conv2, kind, planes, planes, co, planes, co))
        return ConvLayer(sd[conv2 + ".conv_offset.weight"].float(), sd[conv2 + ".conv_offset.bias"].float(), stride, 1,
                         self.device)

    def _conv2(self, x, blk):
        """a block's 3x3 convolution + folded bn2 + ReLU.  Deformable (DCN / DCNv2): the offset convolution writes fp32 NHWC
        [N,Ho,Wo,18|27]; for DCNv2 one kernel splits that into the offsets (channels 0..17) and the sigmoid mask (18..26),
        ModulatedDeformConvPack.forward; the deformable convolution then samples x with them"""
        e = self.eng
        if blk["dcn"] is None:
            return e.conv(x, blk["c2"], relu=True)
        om = e.conv(x, blk["off"], out_f32=True)
        if blk["dcn"] == 'DCN':
            return e.deform_conv(x, om, blk["c2"], relu=True)
        n, ho, wo, _ = om.shape
        off = torch.empty((n, ho, wo, 18), dtype=torch.float32, device=self.device)
        mask = torch.empty((n, ho, wo, 9), dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib().orp_dcnv2_offset_mask(_lib.ptr(om), n * ho * wo, _lib.ptr(off), _lib.ptr(mask),
                                                    _lib.current_stream_ptr()), "orp_dcnv2_offset_mask")
        return e.deform_conv(x, off, blk["c2"], relu=True, mask=mask)

    def _load_head(self, sd):
        d = self.device
        h = "bbox_head."
        self.cls_convs = [(ConvLayer(sd[h + "cls_convs.%d.conv.weight" % i].float(), None, 1, 1, d),
                           Norm(sd, h + "cls_convs.%d.gn" % i, d)) for i in range(3)]
        self.reg_convs = [(ConvLayer(sd[h + "reg_convs.%d.conv.weight" % i].float(), None, 1, 1, d),
                           Norm(sd, h + "reg_convs.%d.gn" % i, d)) for i in range(3)]
        r = h + "reppoints_"
        self.cls_dcn = ConvLayer(sd[r + "cls_conv.weight"].float(), None, 1, 1, d)
        self.cls_out = ConvLayer(sd[r + "cls_out.weight"].float(), sd[r + "cls_out.bias"].float(), 1, 0, d)
        self.init_conv = ConvLayer(sd[r + "pts_init_conv.weight"].float(), sd[r + "pts_init_conv.bias"].float(), 1, 1, d)
        self.init_out = ConvLayer(sd[r + "pts_init_out.weight"].float(), sd[r + "pts_init_out.bias"].float(), 1, 0, d)
        self.ref_dcn = ConvLayer(sd[r + "pts_refine_conv.weight"].float(), None, 1, 1, d)
        self.ref_out = ConvLayer(sd[r + "pts_refine_out.weight"].float(), sd[r + "pts_refine_out.bias"].float(), 1, 0, d)

    def _load_swin(self, sd):
        """Swin + FPN(in [2E,4E,8E], start_level 0, no extra convs: P6/P7 = stride-2 subsampling, fpn.py:163-165)"""
        from .swin import Swin
        d = self.device
        if self.eng.name not in ("bf16", "f16x3"):
            raise ValueError("the Swin backbones run on the tensor-core engines ('f16x3' or 'bf16')")
        self.swin = Swin(sd, d, self.eng, self.swin_arch)
        self.lat = [(ConvLayer(sd["neck.lateral_convs.%d.conv.weight" % i].float(), None, 1, 0, d),
                     Norm(sd, "neck.lateral_convs.%d.gn" % i, d)) for i in range(3)]
        self.fpn = [(ConvLayer(sd["neck.fpn_convs.%d.conv.weight" % i].float(), None, 1, 1, d),
                     Norm(sd, "neck.fpn_convs.%d.gn" % i, d)) for i in range(3)]
        self._load_head(sd)

    # ------------------------------------------------------------------ dense graph
    def normalize(self, img, valid_hw=None):
        """decoded uint8 HWC tiles [N,H,W,3] -> the pipeline's Normalize + ImageToTensor on the device
        (mmdet/datasets/pipelines/transforms.py:Normalize, formating.py:ImageToTensor); float NCHW input passes through.
        valid_hw (device int32 [N,2]): per-image extent of the image inside the padded batch; outside it the result is
        exactly 0.0 (Pad after Normalize)"""
        if img.dtype != torch.uint8:
            return img
        c = self.img_norm_cfg
        x = img.to(self.device).float()
        if c["to_rgb"]:
            x = x.flip(-1)
        key = (tuple(c["mean"]), tuple(c["std"]))
        if getattr(self, "_norm_key", None) != key:                   # device constants, made once (not inside a graph capture)
            self._norm_mean = torch.tensor(c["mean"], dtype=torch.float32).to(self.device)
            self._norm_stdinv = torch.tensor([1.0 / v for v in c["std"]], dtype=torch.float64).float().to(self.device)
            self._norm_key = key
        x = (x - self._norm_mean) * self._norm_stdinv
        if valid_hw is not None:
            n, h, w = x.shape[:3]
            vh = valid_hw.to(self.device)
            inside = (torch.arange(h, device=self.device).view(1, h, 1) < vh[:, 0].view(n, 1, 1)) & \
                     (torch.arange(w, device=self.device).view(1, 1, w) < vh[:, 1].view(n, 1, 1))
            x = torch.where(inside.unsqueeze(-1), x, torch.zeros((), dtype=x.dtype, device=self.device))
        return x.permute(0, 3, 1, 2).contiguous()

    def extract_feat(self, img, valid_hw=None):
        """valid_hw: optional device int32 [N,2] extents of uint8 images padded by the test pipeline"""
        e = self.eng
        if self.swin_arch is not None:
            # decoded uint8 tiles: Normalize + ImageToTensor (+ the zero padding outside valid_hw) are fused into the patch gather
            c3, c4, c5 = self.swin.forward(img, self.img_norm_cfg, valid_hw)
            l2 = e.conv_gn(c5, *self.lat[2])
            l1 = e.conv_gn(c4, *self.lat[1], up=l2)
            l0 = e.conv_gn(c3, *self.lat[0], up=l1)
            outs = [e.conv_gn(l0, *self.fpn[0]), e.conv_gn(l1, *self.fpn[1]), e.conv_gn(l2, *self.fpn[2])]
            outs.append(self.swin.subsample2(outs[-1]))
            outs.append(self.swin.subsample2(outs[-1]))
            return outs
        if img.dtype == torch.uint8 and hasattr(e, "stem_u8") and img.shape[1] % 2 == 0 and img.shape[2] % 2 == 0:
            x = e.maxpool(e.stem_u8(img, self.stem, self.img_norm_cfg, valid_hw))   # Normalize (+ Pad) fused into the stem input
        else:
            x = e.prepare_input(self.normalize(img, valid_hw))
            x = e.maxpool(e.stem(x, self.stem))
        feats = []
        for stage in self.blocks:
            for blk in stage:
                idt = x if blk["ds"] is None else e.conv(x, blk["ds"])
                o = e.conv(x, blk["c1"], relu=True)
                o = self._conv2(o, blk)
                x = e.conv(o, blk["c3"], relu=True, residual=idt)
            feats.append(x)
        c3, c4, c5 = feats[1], feats[2], feats[3]
        l2 = e.conv_gn(c5, *self.lat[2])
        l1 = e.conv_gn(c4, *self.lat[1], up=l2)
        l0 = e.conv_gn(c3, *self.lat[0], up=l1)
        outs = [e.conv_gn(l0, *self.fpn[0]), e.conv_gn(l1, *self.fpn[1]), e.conv_gn(l2, *self.fpn[2])]
        outs.append(e.conv_gn(c5, *self.fpn[3]))
        outs.append(e.conv_gn(outs[-1], *self.fpn[4]))
        return outs

    def head(self, feats, gradient_mul=0.3):
        """forward_single (orientedreppoints_head.py:148-171) for all levels at once: the weights are shared,
        so every layer is ONE launch over the five levels.  Returns per level (cls, init, refine), fp32 NHWC."""
        e = self.eng
        cf, pf = list(feats), list(feats)
        for (lc, nc), (lr, nr) in zip(self.cls_convs, self.reg_convs):
            cf = e.conv_gn_multi(cf, lc, nc, relu=True)
            pf = e.conv_gn_multi(pf, lr, nr, relu=True)
        init = e.conv_multi(e.conv_multi(pf, self.init_conv, relu=True), self.init_out, out_f32=True)   # [N,H,W,18]
        # head :162-163, evaluated in fp32 exactly as written there - one launch for the five levels
        import ctypes
        offsets = [torch.empty_like(t) for t in init]
        n = len(init)
        pa = (ctypes.c_void_p * n)(*[t.data_ptr() for t in init])
        po = (ctypes.c_void_p * n)(*[t.data_ptr() for t in offsets])
        ne = (ctypes.c_longlong * n)(*[t.numel() for t in init])
        _lib.check(_lib.lib().orp_dcn_offsets_multi(n, pa, po, ne, float(gradient_mul), self._dcn_base_host, _lib.current_stream_ptr()),
                   "orp_dcn_offsets_multi")
        cls = e.conv_multi(e.deform_conv_multi(cf, offsets, self.cls_dcn, relu=True), self.cls_out, out_f32=True)
        ref = e.conv_multi(e.deform_conv_multi(pf, offsets, self.ref_dcn, relu=True), self.ref_out, out_f32=True,
                           residual_f32=init)
        return [(c.float(), i, r.float()) for c, i, r in zip(cls, init, ref)]

    def forward_dense(self, img, valid_hw=None):
        # every launch goes to the current stream of the current device: make that this detector's device
        with torch.cuda.device(self.device):
            if img.device != self.device:
                img = img.to(self.device)
            feats = self.extract_feat(img, valid_hw)
            return self.head(feats), feats

    # ------------------------------------------------------------------ CUDA graph of the dense graph
    def capture(self, img_shape, dtype=torch.float32, padded=False):
        """Capture backbone + FPN + head for a fixed input shape into ONE CUDA graph (static buffers): the
        ~180 kernel launches of a step become a single graph launch, which removes the host-side launch
        cost that otherwise dominates a one-tile step.  simple_test() replays it when the shape matches.
        padded=True captures the test-pipeline form (uint8 input with per-image valid extents): the extents are a static
        device buffer of the graph like the image, so one capture serves every extent of that input shape."""
        shape = tuple(img_shape)
        torch.cuda.set_device(self.device)
        self._g_img = torch.zeros(shape, dtype=dtype, device=self.device)
        self._g_valid = None
        if padded:
            self._g_valid = torch.tensor([list(shape[1:3])] * shape[0], dtype=torch.int32).to(self.device)
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):
            for _ in range(2):                                      # warm-up: lazy weight prep, func attributes
                self._forward_dense_opt(self._g_img, self._g_valid)
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        self._graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self._graph):
            self._g_out = self._forward_dense_opt(self._g_img, self._g_valid)
        self._g_shape = (shape, dtype) if not padded else (shape, dtype, "valid_hw")
        return self

    def _forward_dense_opt(self, img, valid_hw):
        return self.forward_dense(img) if valid_hw is None else self.forward_dense(img, valid_hw)

    def _graph_key(self, img, valid_hw):
        key = (tuple(img.shape), img.dtype)
        return key if valid_hw is None else key + ("valid_hw",)

    def forward_dense_graph(self, img, valid_hw=None):
        with torch.cuda.device(self.device):
            self._g_img.copy_(img, non_blocking=True)
            if valid_hw is not None:
                self._g_valid.copy_(valid_hw, non_blocking=True)
            self._graph.replay()
        return self._g_out

    # ------------------------------------------------------------------ simple_test
    def simple_test(self, img, img_metas=None, rescale=False, return_tensors=False, valid_hw=None):
        """valid_hw: device int32 [N,2] extents of a uint8 batch padded by the test pipeline (datasets/pipelines.py);
        pixels outside them enter the network as 0.0"""
        with torch.cuda.device(self.device):
            return self._simple_test(img, img_metas, rescale, return_tensors, valid_hw)

    def _simple_test(self, img, img_metas, rescale, return_tensors, valid_hw=None):
        from .core.get_bboxes import get_bboxes
        if getattr(self, "_g_shape", None) == self._graph_key(img, valid_hw):
            outs, _ = self.forward_dense_graph(img, valid_hw)
        else:
            outs, _ = self._forward_dense_opt(img, valid_hw)
        n = img.shape[0]
        if img_metas is None:
            img_metas = [dict(scale_factor=1.0) for _ in range(n)]
        nms_cfg = self.test_cfg['nms']
        if getattr(self, "fused_post", True) and nms_cfg.get('type', 'rnms') == 'rnms' and nms_cfg.get('mode', 'exact64') == 'exact64':
            from .core.get_bboxes import get_bboxes_fused
            dets, labels, counts = get_bboxes_fused([o[0] for o in outs], [o[2] for o in outs], STRIDES, img_metas,
                                                    self.test_cfg, rescale)
            if return_tensors == "padded":
                return dets, labels, counts
            cnt = counts.tolist()                                      # the one host sync of a step
            if any(c < 0 for c in cnt):
                raise _lib.OrpError("rotated NMS candidate list overflowed its buffer (orp_head_postprocess): results invalid")
            results = [(dets[i, :cnt[i]], labels[i, :cnt[i]]) for i in range(n)]
        else:
            results = get_bboxes([o[0] for o in outs], [o[2] for o in outs], STRIDES, img_metas, self.test_cfg, rescale)
        if return_tensors:
            return results
        from .core.transforms import rbbox2result
        return [rbbox2result(d, l, 16) for d, l in results]

    # ------------------------------------------------------------------ aug_test (multi-scale / flip merge)
    @staticmethod
    def rbbox_flip(rbboxes, img_shape, direction='horizontal'):
        """orientedreppoints_detector.py:48-73: x -> w - x - 1 (or y -> h - y - 1) on every vertex"""
        assert rbboxes.shape[-1] % 8 == 0
        flipped = rbboxes.clone()
        if direction == 'horizontal':
            flipped[..., 0::2] = img_shape[1] - rbboxes[..., 0::2] - 1
        elif direction == 'vertical':
            flipped[..., 1::2] = img_shape[0] - rbboxes[..., 1::2] - 1
        else:
            raise ValueError('Invalid flipping direction "{}"'.format(direction))
        return flipped

    def merge_aug_results(self, aug_bboxes, aug_scores, img_metas):
        """orientedreppoints_detector.py:81-110: map every view's boxes back (un-flip, / scale_factor), concatenate"""
        recovered = []
        for bboxes, info in zip(aug_bboxes, img_metas):
            m = info[0]
            b = self.rbbox_flip(bboxes, m['img_shape']) if m['flip'] else bboxes
            recovered.append(b / m['scale_factor'])
        bboxes = torch.cat(recovered, dim=0)
        if aug_scores is None:
            return bboxes
        return bboxes, torch.cat(aug_scores, dim=0)

    def aug_test(self, imgs, img_metas, rescale=False, valid_hws=None, return_tensors=False):
        """orientedreppoints_detector.py:112-144 for N >= 1 images.  imgs: list of views, each the N images of that view
        (float NCHW [N,3,H,W] or uint8 HWC [N,H,W,3]); img_metas: per view the list of N dicts (img_shape, scale_factor,
        flip); valid_hws: optional list of per-view device int32 [N,2] extents (views padded by the test pipeline).
        One dense pass per view over the whole batch; the raw candidates of all views of an image (get_bboxes(nms=False),
        head :778-779) are mapped back, concatenated and go through ONE multiclass_rnms - in one device pipeline
        (get_bboxes_aug_fused) when fused_post is on and the NMS is 'rnms' in the default arithmetic, else op by op.
        Returns the rbbox2result list ([k, 9] arrays: box | score) of the image for N == 1, a list of them for N > 1;
        return_tensors="padded" (fused pipeline only): the device triple (dets [N,max_per_img,27] with box | score in
        columns 18..26, labels, counts) without a host read."""
        with torch.cuda.device(self.device):
            return self._aug_test(imgs, img_metas, rescale, valid_hws, return_tensors)

    def _aug_test(self, imgs, img_metas, rescale, valid_hws, return_tensors):
        from .core.transforms import rbbox2result
        n = imgs[0].shape[0]
        if len(img_metas) != len(imgs) or any(v.shape[0] != n for v in imgs) or any(len(m) != n for m in img_metas):
            raise ValueError("aug_test: every view needs the same %d images and their metas" % n)
        dense = [self._forward_dense_opt(img, None if valid_hws is None else valid_hws[k])[0] for k, img in enumerate(imgs)]
        cls, ref = [[o[0] for o in outs] for outs in dense], [[o[2] for o in outs] for outs in dense]
        nms_cfg = self.test_cfg['nms']
        if getattr(self, "fused_post", True) and nms_cfg.get('type', 'rnms') == 'rnms' and nms_cfg.get('mode', 'exact64') == 'exact64':
            from .core.get_bboxes import get_bboxes_aug_fused
            dets, labels, counts = get_bboxes_aug_fused(cls, ref, STRIDES, img_metas, self.test_cfg, rescale)
            if return_tensors == "padded":
                return dets, labels, counts
            cnt = counts.tolist()                                      # the one host sync of a call
            if any(c < 0 for c in cnt):
                raise _lib.OrpError("rotated NMS candidate list overflowed its buffer (orp_head_postprocess_aug): results invalid")
            results = [(dets[i, :cnt[i], 18:], labels[i, :cnt[i]]) for i in range(n)]
        else:
            if return_tensors == "padded":
                raise ValueError("aug_test: return_tensors='padded' is the output of the fused post-processing "
                                 "(fused_post on, nms type 'rnms' in the default arithmetic)")
            results = [self._aug_merge_eager([[c[i:i + 1] for c in v] for v in cls], [[p[i:i + 1] for p in v] for v in ref],
                                             [[m[i]] for m in img_metas], rescale) for i in range(n)]
        out = [rbbox2result(d, l, 16) for d, l in results]
        return out[0] if n == 1 else out

    def _aug_merge_eager(self, cls, ref, img_metas, rescale):
        """the op-by-op merge of ONE image's views: (dets [k, 9] box | score, labels [k])"""
        from .core.bbox_nms import multiclass_rnms
        from .core.get_bboxes import get_bboxes
        aug_bboxes, aug_scores = [], []
        for c, p, meta in zip(cls, ref, img_metas):
            b, sc = get_bboxes(c, p, STRIDES, meta, self.test_cfg, False, nms=False)[0]
            aug_bboxes.append(b)
            aug_scores.append(sc)
        merged_bboxes, merged_scores = self.merge_aug_results(aug_bboxes, aug_scores, img_metas)
        det_bboxes, det_labels = multiclass_rnms(merged_bboxes, merged_scores, self.test_cfg['score_thr'],
                                                 self.test_cfg['nms'], self.test_cfg['max_per_img'])
        if not rescale:
            det_bboxes = det_bboxes.clone()
            det_bboxes[:, :8] *= img_metas[0][0]['scale_factor']
        return det_bboxes, det_labels
